// TEST INFRASTRUCTURE.  The 2-D drop-in, executed (INTEGRATION.md §2, §6): this file includes oracle/transfer2d_ref.cpp
// unchanged — the reference's MPM<2> compiled in place from its own translation units, with the stand-in core headers — and
// adds reft2_aos_layout and reft2_substep_via_mpmb, which hand the MPM<2> object's own AoS particle pool (ParticleContainer<2>
// slots) to libmpmb through mpmb_upload_aos / mpmb_download_aos on a 2-D handle.  Built into
// oracle/_ref/libtransfer2d_aos_ref.so by oracle/pyoracle2d_aos.py, only where the reference tree exists.
#include "transfer2d_ref.cpp"

#include <vector>

namespace {
// the engine's parameter vector of a reference particle (MpmbMaterialKind numbering), read from the object itself
bool particle_params2(int kind, MPMParticle<2> *p, float prm[8]) {
  for (int k = 0; k < 8; k++) prm[k] = 0;
  switch (kind) {
    case 0: prm[0] = static_cast<LinearParticle<2> *>(p)->mu; prm[1] = static_cast<LinearParticle<2> *>(p)->lambda; return true;
    case 1: prm[0] = static_cast<JellyParticle<2> *>(p)->mu; prm[1] = static_cast<JellyParticle<2> *>(p)->lambda; return true;
    case 2: { auto *q = static_cast<SnowParticle<2> *>(p); prm[0] = q->mu_0; prm[1] = q->lambda_0; prm[2] = q->hardening; prm[3] = q->theta_c;
              prm[4] = q->theta_s; prm[5] = q->min_Jp; prm[6] = q->max_Jp; return true; }
    case 3: { auto *q = static_cast<WaterParticle<2> *>(p); prm[0] = q->k; prm[1] = q->gamma; return true; }
    case 4: { auto *q = static_cast<SandParticle<2> *>(p); prm[0] = q->mu_0; prm[1] = q->lambda_0; prm[2] = q->alpha; prm[3] = q->cohesion;
              prm[4] = q->beta; return true; }
    case 5: prm[0] = static_cast<ElasticParticle<2> *>(p)->mu_0; prm[1] = static_cast<ElasticParticle<2> *>(p)->lambda_0; return true;
    case 6: { auto *q = static_cast<VonMisesParticle<2> *>(p); prm[0] = q->mu_0; prm[1] = q->lambda_0; prm[2] = q->yield_stress; return true; }
    case 7: { auto *q = static_cast<ViscoParticle<2> *>(p); prm[0] = q->mu_0; prm[1] = q->lambda_0; prm[2] = q->visco_nu; prm[3] = q->visco_kappa;
              prm[4] = q->dt; return true; }
  }
  return false;
}

struct GroupKey2 {
  int kind;
  float prm[8];
  bool operator==(const GroupKey2 &o) const { return kind == o.kind && std::memcmp(prm, o.prm, sizeof(prm)) == 0; }
};
}  // namespace

extern "C" {
// offsetof() / sizeof() on the reference's own 2-D particle classes: the MpmbAosLayout of its ParticleContainer<2> pool, as
// int32 out[12] in the struct's field order.  kind >= 0: the single-offset layout of that particle type (scalar -1 for the
// types without one); kind = -1: the per-kind layout of a pool that mixes types (off_scalar = -1, off_scalar_by_kind =
// SnowParticle<2>::Jp, WaterParticle<2>::j, SandParticle<2>::logJp, ViscoParticle<2>::visco_tau).
void reft2_aos_layout(int kind, int32_t *out) {
  using P2 = MPMParticle<2>;
  const int32_t scalar[4] = {(int32_t)offsetof(SnowParticle<2>, Jp), (int32_t)offsetof(WaterParticle<2>, j), (int32_t)offsetof(SandParticle<2>, logJp),
                             (int32_t)offsetof(ViscoParticle<2>, visco_tau)};
  out[0] = (int32_t)sizeof(ParticleContainer<2>);
  out[1] = (int32_t)offsetof(P2, pos);
  out[2] = (int32_t)offsetof(P2, v_and_m);
  out[3] = (int32_t)offsetof(P2, dg_e);
  out[4] = (int32_t)offsetof(P2, apic_b);
  out[5] = (int32_t)sizeof(VectorND<2, real>);   // one column of MatrixND<2>
  out[6] = (int32_t)offsetof(P2, vol);
  out[7] = kind == 2 ? scalar[0] : kind == 3 ? scalar[1] : kind == 4 ? scalar[2] : kind == 7 ? scalar[3] : -1;
  for (int k = 0; k < 4; k++) out[8 + k] = kind == -1 ? scalar[k] : 0;
}

// n substeps of the MPM<2> object on libmpmb (lib_path: libmpmb.so or its SIMT-emulator build, loaded with dlopen): a 2-D
// handle from the solver's fields, one material group per distinct (type, parameters) with each group's parameters read
// from its first particle, the planes of levelset0, mpmb_upload_aos of allocator.pool / particles, mpmb_substep,
// mpmb_download_aos back into both, particles.resize(survivors).  A pool of one (type, parameters) takes the single-offset
// layout of its type, a mixed pool the per-kind one.  Returns survivors, or a negative status.
int64_t reft2_substep_via_mpmb(void *hp, const char *lib_path, int n, char *err, int err_len) {
  Harness2 *h = static_cast<Harness2 *>(hp);
  Solver2 &m = h->m;
  auto fail = [&](const char *msg, int code) -> int64_t { if (err && err_len > 0) { std::strncpy(err, msg, err_len - 1); err[err_len - 1] = 0; } return code; };
  if (m.particles.empty()) return 0;
  std::vector<GroupKey2> keys;
  std::vector<int32_t> group;
  group.reserve(m.particles.size());
  for (auto ptr : m.particles) {
    MPMParticle<2> *p = m.allocator[ptr];
    GroupKey2 k{h->kind[p->id], {}};
    if (!particle_params2(k.kind, p, k.prm)) return fail("unknown particle type", -103);
    size_t g = 0;
    while (g < keys.size() && !(keys[g] == k)) g++;
    if (g == keys.size()) keys.push_back(k);
    group.push_back((int32_t)g);
  }
  if (keys.size() > MPMB_MAX_GROUPS) return fail("more distinct (type, parameters) than material groups", -106);
  void *lib = dlopen(lib_path, RTLD_NOW | RTLD_LOCAL);
  if (!lib) return fail(dlerror(), -100);
#define SYM(name) auto name##_ = reinterpret_cast<decltype(&name)>(dlsym(lib, #name)); if (!name##_) return fail("missing symbol " #name, -101)
  SYM(mpmb_create); SYM(mpmb_destroy); SYM(mpmb_last_error); SYM(mpmb_set_material); SYM(mpmb_set_planes); SYM(mpmb_upload_aos);
  SYM(mpmb_substep); SYM(mpmb_download_aos);
#undef SYM
  MpmbConfig c{};
  for (int d = 0; d < 2; d++) { c.res[d] = m.res[d]; c.gravity[d] = m.gravity[d]; }
  c.dim = 2;
  c.dx = m.delta_x; c.dt = m.base_delta_t;
  c.particle_gravity = m.particle_gravity;
  c.clean_boundary = m.config_backup.get("clean_boundary", true);
  c.apic_damping = m.apic_damping;
  c.rpic_damping = m.rpic_damping;
  c.device = 0; c.world = 1;
  MpmbHandle e = nullptr;
  if (mpmb_create_(&c, &e) != MPMB_OK) return fail(mpmb_last_error_(nullptr), -102);
  MpmbAosLayout L{};
  reft2_aos_layout(keys.size() == 1 ? keys[0].kind : -1, &L.stride);
  // every group's material before the upload: mpmb_upload_aos takes its snapshot of the group kinds
  int rc = MPMB_OK;
  for (size_t g = 0; rc == MPMB_OK && g < keys.size(); g++) rc = mpmb_set_material_(e, (int32_t)g, keys[g].kind, keys[g].prm, 8);
  if (rc == MPMB_OK && m.levelset.levelset0 && !m.levelset.levelset0->planes.empty()) {
    std::vector<float> pl;   // (n_x, n_y, d) -> (n_x, n_y, 0, d)
    for (auto &q : m.levelset.levelset0->planes) { pl.push_back(q[0]); pl.push_back(q[1]); pl.push_back(0.0f); pl.push_back(q[2]); }
    rc = mpmb_set_planes_(e, (int32_t)m.levelset.levelset0->planes.size(), pl.data(), m.levelset.levelset0->friction);
  }
  const int64_t n_up = (int64_t)m.particles.size();
  if (rc == MPMB_OK) rc = mpmb_upload_aos_(e, n_up, m.allocator.pool.data(), (int64_t)m.allocator.pool.size(), m.particles.data(), &L, group.data());
  if (rc == MPMB_OK) rc = mpmb_substep_(e, n);
  int64_t alive = 0;
  if (rc == MPMB_OK) rc = mpmb_download_aos_(e, m.allocator.pool.data(), (int64_t)m.allocator.pool.size(), m.particles.data(), n_up, &L, &alive);
  if (rc != MPMB_OK) {
    fail(mpmb_last_error_(e), rc);
    mpmb_destroy_(e);
    return rc;
  }
  mpmb_destroy_(e);
  m.particles.resize((size_t)alive);                      // == what clear_boundary_particles leaves (src/mpm.cpp:583-633)
  m.current_t += n * m.base_delta_t;
  m.substep_counter += n;
  return alive;
}
}
