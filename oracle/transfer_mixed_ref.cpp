// TEST INFRASTRUCTURE.  The drop-in for pools that mix particle types (INTEGRATION.md §2): this file includes
// oracle/transfer_ref.cpp unchanged — the same reference sources, stand-in headers and MPM<3> / AsyncMPM<3> harness — and adds
// reft_substep_via_mpmb_mixed, which hands a pool of several registered types to libmpmb with one material group per distinct
// (type, parameters) and the per-kind plastic-scalar offsets of MpmbAosLayout.  AsyncMPM's substep() calls come here through
// oracle/async_route_mixed.h.  Built into oracle/_ref/libtransfer_mixed_ref.so by oracle/pyoracle_mixed.py, only where the
// reference tree exists.
#include "transfer_ref.cpp"

#include <vector>

namespace {
// the engine's parameter vector of a reference particle (MpmbMaterialKind numbering), read from the object itself
bool particle_params(int kind, MPMParticle<3> *p, float prm[8]) {
  for (int k = 0; k < 8; k++) prm[k] = 0;
  switch (kind) {
    case 0: prm[0] = static_cast<LinearParticle<3> *>(p)->mu; prm[1] = static_cast<LinearParticle<3> *>(p)->lambda; return true;
    case 1: prm[0] = static_cast<JellyParticle<3> *>(p)->mu; prm[1] = static_cast<JellyParticle<3> *>(p)->lambda; return true;
    case 2: { auto *q = static_cast<SnowParticle<3> *>(p); prm[0] = q->mu_0; prm[1] = q->lambda_0; prm[2] = q->hardening; prm[3] = q->theta_c;
              prm[4] = q->theta_s; prm[5] = q->min_Jp; prm[6] = q->max_Jp; return true; }
    case 3: { auto *q = static_cast<WaterParticle<3> *>(p); prm[0] = q->k; prm[1] = q->gamma; return true; }
    case 4: { auto *q = static_cast<SandParticle<3> *>(p); prm[0] = q->mu_0; prm[1] = q->lambda_0; prm[2] = q->alpha; prm[3] = q->cohesion;
              prm[4] = q->beta; return true; }
    case 5: prm[0] = static_cast<ElasticParticle<3> *>(p)->mu_0; prm[1] = static_cast<ElasticParticle<3> *>(p)->lambda_0; return true;
    case 6: { auto *q = static_cast<VonMisesParticle<3> *>(p); prm[0] = q->mu_0; prm[1] = q->lambda_0; prm[2] = q->yield_stress; return true; }
    case 7: { auto *q = static_cast<ViscoParticle<3> *>(p); prm[0] = q->mu_0; prm[1] = q->lambda_0; prm[2] = q->visco_nu; prm[3] = q->visco_kappa;
              prm[4] = q->dt; return true; }
  }
  return false;
}

struct GroupKey {
  int kind;
  float prm[8];
  bool operator==(const GroupKey &o) const { return kind == o.kind && std::memcmp(prm, o.prm, sizeof(prm)) == 0; }
};
}  // namespace

extern "C" {
// offsetof() of the plastic scalars in the order of MpmbAosLayout::off_scalar_by_kind: SnowParticle::Jp, WaterParticle::j,
// SandParticle::logJp, ViscoParticle::visco_tau
void reft_aos_scalar_offsets(int32_t *out) {
  out[0] = (int32_t)offsetof(SnowParticle<3>, Jp);
  out[1] = (int32_t)offsetof(WaterParticle<3>, j);
  out[2] = (int32_t)offsetof(SandParticle<3>, logJp);
  out[3] = (int32_t)offsetof(ViscoParticle<3>, visco_tau);
}

// reft_substep_via_mpmb for a pool of any mix of the registered types: one group per distinct (type, parameters) over
// `particles`, as INTEGRATION.md §2 builds it, each group's parameters read from its first particle, group[k] passed to
// mpmb_upload_aos, and the scalar offsets per kind.  A pool of one (type, parameters) takes reft_substep_via_mpmb itself: the
// same calls and the same single-offset layout.  Rigid bodies are routed only with single-type pools.  Returns survivors, or
// a negative status.
int64_t reft_substep_via_mpmb_mixed(void *hp, const char *lib_path, int n, char *err, int err_len) {
  Harness *h = static_cast<Harness *>(hp);
  Solver &m = h->m;
  auto fail = [&](const char *msg, int code) -> int64_t { if (err && err_len > 0) { std::strncpy(err, msg, err_len - 1); err[err_len - 1] = 0; } return code; };
  std::vector<GroupKey> keys;
  std::vector<int32_t> group;
  group.reserve(m.particles.size());
  bool rigid = false;
  for (auto ptr : m.particles) {
    MPMParticle<3> *p = m.allocator[ptr];
    if (p->is_rigid()) { rigid = true; continue; }
    GroupKey k{h->kind[p->id], {}};
    if (!particle_params(k.kind, p, k.prm)) return fail("unknown particle type", -103);
    size_t g = 0;
    while (g < keys.size() && !(keys[g] == k)) g++;
    if (g == keys.size()) keys.push_back(k);
    group.push_back((int32_t)g);
  }
  if (keys.size() <= 1) return reft_substep_via_mpmb(hp, lib_path, n, err, err_len);
  if (rigid) return fail("pools of several particle types are routed without rigid bodies only", -105);
  if (keys.size() > MPMB_MAX_GROUPS) return fail("more distinct (type, parameters) than material groups", -106);
  void *lib = dlopen(lib_path, RTLD_NOW | RTLD_LOCAL);
  if (!lib) return fail(dlerror(), -100);
#define SYM(name) auto name##_ = reinterpret_cast<decltype(&name)>(dlsym(lib, #name)); if (!name##_) return fail("missing symbol " #name, -101)
  SYM(mpmb_create); SYM(mpmb_destroy); SYM(mpmb_last_error); SYM(mpmb_set_material); SYM(mpmb_set_planes); SYM(mpmb_upload_aos);
  SYM(mpmb_substep); SYM(mpmb_download_aos); SYM(mpmb_set_delta_t);
#undef SYM
  MpmbConfig c{};
  for (int d = 0; d < 3; d++) { c.res[d] = m.res[d]; c.gravity[d] = m.gravity[d]; }
  c.dx = m.delta_x; c.dt = m.base_delta_t;
  c.particle_gravity = m.particle_gravity;
  c.clean_boundary = m.config_backup.get("clean_boundary", true);
  c.device = 0; c.world = 1;
  // a routed solver keeps one engine across calls (and shares it with reft_substep_via_mpmb), as there
  const bool keep = !h->route_lib.empty();
  MpmbHandle e = keep ? h->route_engine : nullptr;
  if (!e) {
    if (mpmb_create_(&c, &e) != MPMB_OK) return fail(mpmb_last_error_(nullptr), -102);
  } else if (mpmb_set_delta_t_(e, m.base_delta_t) != MPMB_OK) {
    return fail(mpmb_last_error_(e), -104);
  }
  if (keep) { h->route_engine = e; h->route_destroy = mpmb_destroy_; }
  using P3 = MPMParticle<3>;
  MpmbAosLayout L{};
  L.stride = (int32_t)sizeof(ParticleContainer<3>);
  L.off_pos = (int32_t)offsetof(P3, pos);
  L.off_v_and_m = (int32_t)offsetof(P3, v_and_m);
  L.off_dg_e = (int32_t)offsetof(P3, dg_e);
  L.off_apic_b = (int32_t)offsetof(P3, apic_b);
  L.col_pitch = (int32_t)sizeof(VectorND<3, real>);
  L.off_vol = (int32_t)offsetof(P3, vol);
  L.off_scalar = -1;
  reft_aos_scalar_offsets(L.off_scalar_by_kind);
  // every group's material before the upload: mpmb_upload_aos takes its snapshot of the group kinds
  int rc = MPMB_OK;
  for (size_t g = 0; rc == MPMB_OK && g < keys.size(); g++) rc = mpmb_set_material_(e, (int32_t)g, keys[g].kind, keys[g].prm, 8);
  if (rc == MPMB_OK && m.levelset.levelset0 && !m.levelset.levelset0->planes.empty()) {
    std::vector<float> pl;
    for (auto &q : m.levelset.levelset0->planes) for (int k = 0; k < 4; k++) pl.push_back(q[k]);
    rc = mpmb_set_planes_(e, (int32_t)m.levelset.levelset0->planes.size(), pl.data(), m.levelset.levelset0->friction);
  }
  const int64_t n_up = (int64_t)m.particles.size();
  if (rc == MPMB_OK) rc = mpmb_upload_aos_(e, n_up, m.allocator.pool.data(), (int64_t)m.allocator.pool.size(), m.particles.data(), &L, group.data());
  if (rc == MPMB_OK) rc = mpmb_substep_(e, n);
  int64_t alive = 0;
  if (rc == MPMB_OK) rc = mpmb_download_aos_(e, m.allocator.pool.data(), (int64_t)m.allocator.pool.size(), m.particles.data(), n_up, &L, &alive);
  if (rc != MPMB_OK) {
    fail(mpmb_last_error_(e), rc);
    if (!keep) mpmb_destroy_(e);
    return rc;
  }
  m.particles.resize((size_t)alive);                      // == what clear_boundary_particles leaves (src/mpm.cpp:583-633)
  m.current_t += n * m.base_delta_t;
  m.substep_counter += n;
  if (!keep) mpmb_destroy_(e);
  return alive;
}
}

namespace taichi {
// harness_substep of transfer_ref.cpp with the mixed-pool route: AsyncMPM's level sets may hold several particle types
void harness_substep_mixed(MPM<3> *m) {
  auto it = harness_registry().find(m);
  Harness *h = it == harness_registry().end() ? nullptr : it->second;
  if (!h || h->route_lib.empty()) { m->substep(); return; }
  char err[512] = {0};
  const int64_t rc = reft_substep_via_mpmb_mixed(h, h->route_lib.c_str(), 1, err, (int)sizeof(err));
  if (rc < 0) h->route_error = err;
  h->routed_substeps++;
}
}  // namespace taichi
