// TEST INFRASTRUCTURE.  The reference's 2-D solver MPM<2> (src/mpm.cpp:983-988) from its own translation units, compiled
// where they lie: this file includes oracle/transfer_ref.cpp unchanged — the same reference sources (transfer.cpp, mpm.cpp,
// visualize.cpp, particles.cpp, ...), the same stand-in core headers and its MPM<3> harness — and adds the reft2_* entry points
// that drive an MPM<2> object.  Built into oracle/_ref/libtransfer2d_ref.so by oracle/pyoracle2d.py, only where the reference
// tree exists.
#include "transfer_ref.cpp"

namespace taichi {
// the one member of the 2-D solver that lives outside this build (src/mpm_rigid_body.cpp) and that the MPM<3> harness does not
// stub: add_particles' rigid branch, never reached without rigid bodies
template <> void MPM<2>::add_rigid_particle(Config) {}
}  // namespace taichi

// ================================================================================================ MPM<2>
// The reference's 2-D solver, MPM<2> (src/mpm.cpp:983-988), from the same translation units: its own
// sort_particles_and_populate_grid, rasterize_optimized (= rasterize(dt, true), src/transfer.cpp:280-284), the grid update,
// resample_optimized (= resample(), :697-701), clear_boundary_particles and substep().  Particle arrays are dim-packed:
// x, v [n][2]; F, b [n][4] column-major (m[c * 2 + r]); planes (n_x, n_y, d) in grid units.
namespace {
using Solver2 = MPM<2>;
struct Harness2 {
  Solver2 m;
  std::vector<int> kind;
};
MatrixND<2, real> load2(const float *a) {
  MatrixND<2, real> r;
  for (int c = 0; c < 2; c++) for (int q = 0; q < 2; q++) r[c][q] = a[c * 2 + q];
  return r;
}
void store2(const MatrixND<2, real> &a, float *o) {
  for (int c = 0; c < 2; c++) for (int q = 0; q < 2; q++) o[c * 2 + q] = a[c][q];
}
}  // namespace

extern "C" {
void *reft2_create(const int *res, float dx, float dt, const float *gravity, int particle_gravity, int clean_boundary, float apic_damping,
                   float rpic_damping) {
  Harness2 *h = new Harness2();
  Solver2 &m = h->m;
  m.res = VectorND<2, int>(res[0], res[1]);
  m.delta_x = dx;
  m.inv_delta_x = 1.0f / dx;
  m.base_delta_t = dt;
  m.gravity = VectorND<2, real>(gravity[0], gravity[1]);
  m.particle_gravity = particle_gravity != 0;
  m.apic = true;
  m.apic_damping = apic_damping;
  m.rpic_damping = rpic_damping;
  m.affine_damping = m.penalty = 0;
  m.pushing_force = 20000.0f;
  m.cutting_counter = m.plasticity_counter = 0;
  m.reorder_interval = 1000;                               // src/mpm.cpp:45
  m.config_backup.set("clean_boundary", clean_boundary != 0);
  m.spgrid_size = 4096;                                   // src/mpm.cpp:50-54
  while (m.spgrid_size / 2 > (m.res.max() + 1)) m.spgrid_size /= 2;
  m.grid = std::make_unique<Solver2::SparseGrid>(m.spgrid_size, m.spgrid_size);
  m.page_map = std::make_unique<Solver2::PageMap>(*m.grid);
  m.rigid_page_map = std::make_unique<Solver2::PageMap>(*m.grid);
  m.fat_page_map = std::make_unique<Solver2::PageMap>(*m.grid);
  m.levelset.levelset0 = std::make_shared<LevelSet<2>>();  // no planes: phi = +inf everywhere
  return h;
}
void reft2_destroy(void *hp) { delete static_cast<Harness2 *>(hp); }
// threads of the stand-in's parallel loops, as reft_set_threads: 1 = serial (the pins); more only to time
void reft2_set_threads(void *hp, int n) {
  static_cast<Harness2 *>(hp)->m.num_threads = n < 1 ? 1 : n;
  stub_num_threads() = n < 1 ? 1 : n;
#if defined(_OPENMP)
  omp_set_num_threads(n < 1 ? 1 : n);
#endif
}
// n particles of one kind (the oracle's numbering and parameter vectors); particle k gets id k in the order of the calls
int64_t reft2_add_particles(void *hp, int kind, const float *params, int64_t n, const float *x, const float *v, const float *mass,
                            const float *vol, const float *F, const float *b, const float *ps) {
  Harness2 *h = static_cast<Harness2 *>(hp);
  static const char *names[8] = {"linear", "jelly", "snow", "water", "sand", "elastic", "von_mises", "visco"};
  if (kind < 0 || kind > 7) return -1;
  for (int64_t i = 0; i < n; i++) {
    auto alloc = h->m.allocator.allocate_particle(names[kind]);
    MPMParticle<2> *p = alloc.second;
    Config cfg;
    switch (kind) {
      case 0: p->initialize(cfg); static_cast<LinearParticle<2> *>(p)->mu = params[0]; static_cast<LinearParticle<2> *>(p)->lambda = params[1]; break;
      case 1: p->initialize(cfg); static_cast<JellyParticle<2> *>(p)->mu = params[0]; static_cast<JellyParticle<2> *>(p)->lambda = params[1]; break;
      case 2:
        cfg.set("mu_0", params[0]).set("lambda_0", params[1]).set("hardening", params[2]).set("theta_c", params[3]).set("theta_s", params[4])
            .set("min_Jp", params[5]).set("max_Jp", params[6]).set("Jp", ps[i]);
        p->initialize(cfg);
        break;
      case 3: cfg.set("k", params[0]).set("gamma", params[1]); p->initialize(cfg); static_cast<WaterParticle<2> *>(p)->j = ps[i]; break;
      case 4:
        cfg.set("mu_0", params[0]).set("lambda_0", params[1]).set("cohesion", params[3]).set("beta", params[4]);
        p->initialize(cfg);
        static_cast<SandParticle<2> *>(p)->alpha = params[2];
        static_cast<SandParticle<2> *>(p)->logJp = ps[i];
        break;
      case 5: p->initialize(cfg); static_cast<ElasticParticle<2> *>(p)->mu_0 = params[0]; static_cast<ElasticParticle<2> *>(p)->lambda_0 = params[1]; break;
      case 6:
        cfg.set("yield_stress", params[2]);
        p->initialize(cfg);
        static_cast<VonMisesParticle<2> *>(p)->mu_0 = params[0];
        static_cast<VonMisesParticle<2> *>(p)->lambda_0 = params[1];
        break;
      case 7:
        cfg.set("nu", params[2]).set("kappa", params[3]).set("base_delta_t", params[4]).set("tau", ps[i]);
        p->initialize(cfg);
        static_cast<ViscoParticle<2> *>(p)->mu_0 = params[0];
        static_cast<ViscoParticle<2> *>(p)->lambda_0 = params[1];
        break;
    }
    p->pos = VectorND<2, real>(x[2 * i], x[2 * i + 1]);
    p->set_mass(mass[i]);
    p->set_velocity(VectorND<2, real>(v[2 * i], v[2 * i + 1]));
    p->vol = vol[i];
    p->dg_e = load2(F + 4 * i);
    p->apic_b = load2(b + 4 * i);
    h->m.particles.push_back(alloc.first);
    h->kind.push_back(kind);
  }
  return n;
}
// static level set of half-planes, grid units: phi(X) = n.X + d (planes3[k] = n_x, n_y, d)
void reft2_set_planes(void *hp, int n, const float *planes3, float friction) {
  Solver2 &m = static_cast<Harness2 *>(hp)->m;
  auto ls = std::make_shared<LevelSet<2>>();
  ls->friction = friction;
  for (int k = 0; k < n; k++) ls->planes.push_back(VectorND<3, real>(planes3[3 * k], planes3[3 * k + 1], planes3[3 * k + 2]));
  m.levelset.levelset0 = ls;
}
// stage 1: sort_particles_and_populate_grid + rasterize_optimized; 2: the grid update of substep() (src/mpm.cpp:519-540);
// 3: resample_optimized and, with clean_boundary, clear_boundary_particles
void reft2_stage(void *hp, int stage) {
  Solver2 &m = static_cast<Harness2 *>(hp)->m;
  if (stage == 1) { m.sort_particles_and_populate_grid(); m.rasterize_optimized(m.base_delta_t); }
  if (stage == 2) {
    VectorND<2, real> inc = m.gravity * m.base_delta_t;
    if (m.particle_gravity) inc = VectorND<2, real>(0.0f);
    m.normalize_grid_and_apply_external_force(inc);
    m.apply_grid_boundary_conditions(m.levelset, m.current_t);
  }
  if (stage == 3) {
    m.resample_optimized();
    if (m.config_backup.get("clean_boundary", true)) m.clear_boundary_particles();
    m.current_t += m.base_delta_t;
    m.substep_counter += 1;
  }
}
// dense [res0+1][res1+1][4] = (p_x | v_x, p_y | v_y, 0, m) of the nodes of the fat blocks
void reft2_get_grid(void *hp, float *out) {
  Solver2 &m = static_cast<Harness2 *>(hp)->m;
  using Mask2 = Solver2::SparseMask;
  const int nx = m.res[0] + 1, ny = m.res[1] + 1;
  auto fat = m.fat_page_map->Get_Blocks();
  std::memset(out, 0, sizeof(float) * 4 * size_t(nx) * ny);
  auto grid_array = m.grid->Get_Array();
  for (int b = 0; b < (int)fat.second; b++) {
    auto c = Mask2::LinearToCoord(fat.first[b]);
    for (int i = 0; i < (1 << Mask2::block_xbits); i++)
      for (int j = 0; j < (1 << Mask2::block_ybits); j++) {
        int X = c[0] + i, Y = c[1] + j;
        if (X >= nx || Y >= ny) continue;
        const GridState<2> &g = grid_array(std::array<int, 2>{X, Y});
        float *o = out + 4 * (size_t(X) * ny + Y);
        o[0] = g.velocity_and_mass[0];
        o[1] = g.velocity_and_mass[1];
        o[3] = g.velocity_and_mass[2];
      }
  }
}
// n whole substeps by MPM<2>::substep() itself.  Returns the number of live particles.
int64_t reft2_substep(void *hp, int n) {
  Solver2 &m = static_cast<Harness2 *>(hp)->m;
  for (int i = 0; i < n; i++) m.substep();
  return (int64_t)m.particles.size();
}
int64_t reft2_num_particles(void *hp) { return (int64_t)static_cast<Harness2 *>(hp)->m.particles.size(); }
// state by id (= order of reft2_add_particles); alive[id] = 1 for the particles still in MPM::particles
void reft2_get_particles(void *hp, float *x, float *v, float *F, float *b, float *ps, uint8_t *alive) {
  Harness2 *h = static_cast<Harness2 *>(hp);
  Solver2 &m = h->m;
  std::memset(alive, 0, h->kind.size());
  for (auto ptr : m.particles) {
    MPMParticle<2> *p = m.allocator[ptr];
    const int id = p->id;
    alive[id] = 1;
    for (int d = 0; d < 2; d++) { x[2 * id + d] = p->pos[d]; v[2 * id + d] = p->get_velocity()[d]; }
    store2(p->dg_e, F + 4 * id);
    store2(p->apic_b, b + 4 * id);
    switch (h->kind[id]) {
      case 2: ps[id] = static_cast<SnowParticle<2> *>(p)->Jp; break;
      case 3: ps[id] = static_cast<WaterParticle<2> *>(p)->j; break;
      case 4: ps[id] = static_cast<SandParticle<2> *>(p)->logJp; break;
      case 7: ps[id] = static_cast<ViscoParticle<2> *>(p)->visco_tau; break;
      default: ps[id] = 0;
    }
  }
}
// frame dump by MPM<2>::write_partio itself (src/visualize.cpp:16-100)
void reft2_write_partio(void *hp, const char *file_name) { static_cast<Harness2 *>(hp)->m.write_partio(file_name); }
}
