// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product.
//
// The 2-D restatement (MPM<2>) next to the 3-D one: this translation unit includes oracle/mpm_oracle.cpp unchanged — its
// 3x3 helpers, B-spline weights, material numbering and exports come along — and adds the 2-D substep and its C entry points.
// Built into oracle/liboracle2d.so by oracle/pyoracle2d.py; only tests/, bench_2d.py's CPU baseline and the golden generator
// load it.
#include "mpm_oracle.cpp"

namespace {
// ================================================================================
// MPM<2> (src/mpm.cpp:983-988): the substep with the scalar transfers MPM<2> runs — rasterize(dt, true) and resample()
// (src/transfer.cpp:193-284, 585-701; MLSMPM defined, :27) — the dimension-generic grid update and boundary condition
// (src/mpm.cpp:277-372) and deletion (src/mpm.h:269-276, src/mpm.cpp:583-633), with the constitutive models of
// src/particles.cpp at dim = 2.  No rigid bodies: the colour test never fires and near_boundary() stays false.
// 2x2 matrices are column-major: m[c*2+r].  The SVD is F = U diag(s) V^T with proper rotations U, V (det F < 0 gives the
// smaller singular value a negative sign), from the eigen-system of E = F F^T - I formed as G + G^T + G G^T (G = F - I).
// PARITY STATUS: pinned against the reference's own MPM<2> compiled in place (oracle/transfer2d_ref.cpp, reft2_*): stage by
// stage and as whole substeps, all eight materials (tests/test_oracle_ref_mpm2d.py, golden vectors tests/golden/mpm2d_ref.npz).
// ================================================================================
template <class R> struct Scene2 {
  int res[2];
  R dx, inv_dx, dt;
  R gravity[2];
  int particle_gravity, clean_boundary;
  R apic_damping, rpic_damping;
  const int32_t *mat_kind;
  const R *mat_params;
  const R *sdf;  // [nx][ny][4] = (n_x, n_y, 0, phi) in grid units, or null
  R friction;
  int nx() const { return res[0] + 1; }
  int ny() const { return res[1] + 1; }
  size_t node(int i, int j) const { return size_t(i) * ny() + j; }
  size_t n_nodes() const { return size_t(nx()) * ny(); }
};
template <class R> struct Particles2 {
  int64_t n;
  R *x, *v, *F, *b;  // [n][2], [n][2], [n][4], [n][4]
  const R *mass, *vol;
  R *ps;
  const int32_t *group;
};

template <class R> inline R &at2(R *m, int r, int c) { return m[c * 2 + r]; }
template <class R> inline R at2(const R *m, int r, int c) { return m[c * 2 + r]; }
template <class R> inline void mul2(const R *a, const R *b, R *out) {
  R t[4];
  for (int c = 0; c < 2; c++)
    for (int r = 0; r < 2; r++) at2(t, r, c) = at2(a, r, 0) * at2(b, 0, c) + at2(a, r, 1) * at2(b, 1, c);
  std::memcpy(out, t, sizeof(t));
}
template <class R> inline void transpose2(const R *a, R *out) {
  R t[4] = {a[0], a[2], a[1], a[3]};
  std::memcpy(out, t, sizeof(t));
}
template <class R> inline R det2(const R *a) { return a[0] * a[3] - a[2] * a[1]; }
// F = U diag(s) V^T
template <class R> void svd2c(const R *F, R *U, R *s, R *V) {
  const R g00 = F[0] - 1, g10 = F[1], g01 = F[2], g11 = F[3] - 1;
  const R a = 2 * g00 + (g00 * g00 + g01 * g01), d = 2 * g11 + (g10 * g10 + g11 * g11), b = (g01 + g10) + (g00 * g10 + g01 * g11);
  const R m = (a + d) / 2, h = (a - d) / 2, r = std::sqrt(h * h + b * b), det = a * d - b * b;
  R e1, e2;
  if (m >= 0) { e1 = m + r; e2 = e1 != 0 ? det / e1 : R(0); }
  else { e2 = m - r; e1 = det / e2; }
  const R phi = r > 0 ? std::atan2(b, h) / 2 : R(0);
  const R c = std::cos(phi), sn = std::sin(phi);
  U[0] = c; U[1] = sn; U[2] = -sn; U[3] = c;
  s[0] = std::sqrt(R(1) + e1);
  s[1] = (det2(F) < 0 ? R(-1) : R(1)) * std::sqrt(std::max(R(1) + e2, R(0)));
  for (int k = 0; k < 2; k++) {  // column k of V = F^T u_k / s_k
    const R u0 = at2(U, 0, k), u1 = at2(U, 1, k);
    R w0 = at2(F, 0, 0) * u0 + at2(F, 1, 0) * u1, w1 = at2(F, 0, 1) * u0 + at2(F, 1, 1) * u1;
    if (s[k] != 0) { w0 /= s[k]; w1 /= s[k]; }
    at2(V, 0, k) = w0; at2(V, 1, k) = w1;
  }
  if (s[1] == 0) { at2(V, 0, 1) = -at2(V, 1, 0); at2(V, 1, 1) = at2(V, 0, 0); }
}
// U diag(d) V^T
template <class R> inline void usv2(const R *U, const R *d, const R *V, R *out) {
  R US[4] = {U[0] * d[0], U[1] * d[0], U[2] * d[1], U[3] * d[1]}, Vt[4];
  transpose2(V, Vt);
  mul2(US, Vt, out);
}
// fixed corotated: 2 mu (F - R) + lambda (J - 1) J F^-T, R = U V^T (src/particles.cpp:207-214, 391-398)
template <class R> void piola_fc2(const R *F, R mu, R lambda, R *P) {
  R U[4], s[2], V[4], one[2] = {1, 1}, Rm[4];
  svd2c(F, U, s, V);
  usv2(U, one, V, Rm);
  const R j = det2(F);
  const R FinvT[4] = {F[3] / j, -F[2] / j, -F[1] / j, F[0] / j};
  for (int k = 0; k < 4; k++) P[k] = 2 * mu * (F[k] - Rm[k]) + lambda * (j - 1) * j * FinvT[k];
}
template <class R> void calculate_force2(int kind, const R *prm, const R *F, R ps, R vol, R *out) {
  R P[4], Ft[4], PFt[4];
  transpose2(F, Ft);
  switch (kind) {
    case MAT_LINEAR: {  // src/particles.cpp:329-337: mu (F + F^T - 2) + lambda (tr F - dim)
      const R tr = F[0] + F[3];
      for (int c = 0; c < 2; c++)
        for (int r = 0; r < 2; r++) at2(P, r, c) = prm[0] * (at2(F, r, c) + at2(F, c, r) - (r == c ? R(2) : R(0))) + (r == c ? prm[1] * (tr - R(2)) : R(0));
      break;
    }
    case MAT_WATER: {  // src/particles.cpp:463-467
      const R p = prm[0] * (std::pow(ps, -prm[1]) - R(1));
      out[0] = -vol * ps * (-p); out[1] = 0; out[2] = 0; out[3] = -vol * ps * (-p);
      return;
    }
    case MAT_SAND:
    case MAT_ELASTIC:
    case MAT_VON_MISES: {  // src/particles.cpp:628-637 (703-712, 800-809): -vol U center V^T F^T
      R U[4], s[2], V[4], center[2];
      svd2c(F, U, s, V);
      const R l0 = std::log(s[0]), l1 = std::log(s[1]);
      center[0] = R(2) * prm[0] * (R(1) / s[0]) * l0 + prm[1] * (l0 + l1) * (R(1) / s[0]);
      center[1] = R(2) * prm[0] * (R(1) / s[1]) * l1 + prm[1] * (l0 + l1) * (R(1) / s[1]);
      usv2(U, center, V, P);
      break;
    }
    case MAT_SNOW: {  // src/particles.cpp:244-252: Lame parameters * exp(h (1 - Jp))
      const R e = std::exp(prm[2] * (R(1) - ps));
      piola_fc2(F, prm[0] * e, prm[1] * e, P);
      break;
    }
    default:  // JELLY, VISCO (mu_0, lambda_0)
      piola_fc2(F, prm[0], prm[1], P);
  }
  mul2(P, Ft, PFt);
  for (int k = 0; k < 4; k++) out[k] = -vol * PFt[k];
}
// SandParticle::project (src/particles.cpp:599-626), d = 2
template <class R> void sand_project2(const R *prm, const R *sigma, R &logJp, R *out) {
  const R d = 2, mu0 = prm[0], lambda0 = prm[1], alpha = prm[2], cohesion = prm[3], beta = prm[4];
  R eps[2];
  for (int i = 0; i < 2; i++) eps[i] = std::log(std::max(std::abs(sigma[i]), R(1e-4))) - cohesion;
  const R eps_sum = eps[0] + eps[1], tr = eps_sum + logJp;
  const R hat[2] = {eps[0] - tr / d, eps[1] - tr / d};
  const R hat_n = std::sqrt(hat[0] * hat[0] + hat[1] * hat[1]);
  if (tr >= 0) {
    out[0] = out[1] = std::exp(cohesion);
    logJp = beta * eps_sum + logJp;
  } else {
    logJp = 0;
    const R dgamma = hat_n + (d * lambda0 + R(2) * mu0) / (R(2) * mu0) * tr * alpha;
    for (int i = 0; i < 2; i++) out[i] = dgamma <= 0 ? std::exp(eps[i] + cohesion) : std::exp(eps[i] - dgamma / hat_n * hat[i] + cohesion);
  }
}
template <class R> void visco_exponent2(R dt, const R *m, R *out, int depth = 0) {  // src/particles.cpp:89-102
  R s[4], h[4], r[4];
  for (int i = 0; i < 4; i++) { s[i] = m[i] * dt; h[i] = s[i] * R(0.5); }
  h[0] += 1; h[3] += 1;
  mul2(h, s, r);
  r[0] += 1; r[3] += 1;
  if (det2(r) > 0 || depth >= 16) { std::memcpy(out, r, sizeof(r)); return; }
  R t[4];
  visco_exponent2(dt / R(2), m, t, depth + 1);
  mul2(t, t, out);
}
template <class R> void plasticity2(int kind, const R *prm, const R *cdg, R *F, R &ps) {
  if (kind == MAT_WATER) {  // src/particles.cpp:469-478: j *= tr(cdg) - (dim - 1)
    ps *= (cdg[0] + cdg[3]) - R(1);
    if (ps < R(0.1)) ps = R(0.1);
    return;
  }
  if (kind == MAT_VISCO) {  // src/particles.cpp:104-137
    const R mu0 = prm[0], lambda0 = prm[1], nu = prm[2], kappa = prm[3], dt = prm[4];
    R m[4] = {(cdg[0] - 1) / dt, cdg[1] / dt, cdg[2] / dt, (cdg[3] - 1) / dt}, ex[4], Fh[4];
    visco_exponent2(dt, m, ex);
    mul2(ex, F, Fh);
    R U[4], sg[2], V[4], P[4];
    svd2c(Fh, U, sg, V);
    piola_fc2(F, mu0, lambda0, P);
    const R pnorm = std::sqrt(P[0] * P[0] + P[1] * P[1] + P[2] * P[2] + P[3] * P[3]);
    R gamma = 0;
    if (pnorm > R(1e-5)) gamma = std::min(std::max(dt * nu * (pnorm - ps) / pnorm, R(0)), R(1));
    const R det = sg[0] * sg[1];
    R scale = 1;
    if (std::abs(det) > R(1e-5)) scale = R(1) / std::pow(det, R(1) / R(2));
    R sn[2];
    for (int d = 0; d < 2; d++) {
      const R mid = std::pow(sg[d] * scale, gamma), mid_inv = std::abs(mid) > R(1e-5) ? R(1) / mid : R(1);
      sn[d] = std::min(std::max(sg[d] * mid_inv, R(0.1)), R(10));
    }
    usv2(U, sn, V, F);
    ps += kappa * gamma * pnorm;
    return;
  }
  R Fn[4];
  mul2(cdg, F, Fn);
  if (kind == MAT_LINEAR || kind == MAT_JELLY || kind == MAT_ELASTIC) { std::memcpy(F, Fn, sizeof(Fn)); return; }
  R U[4], s[2], V[4], sn[2];
  svd2c(Fn, U, s, V);
  if (kind == MAT_VON_MISES) {  // src/particles.cpp:714-734
    const R e0 = std::log(s[0]), e1 = std::log(s[1]), tr = e0 + e1;
    const R h0 = e0 - tr / R(2), h1 = e1 - tr / R(2), n2 = h0 * h0 + h1 * h1;
    const R dgamma = n2 - prm[2] / (R(2) * prm[0]);
    if (dgamma <= 0) { std::memcpy(F, Fn, sizeof(Fn)); return; }
    sn[0] = std::exp(e0 - (dgamma / n2) * h0);
    sn[1] = std::exp(e1 - (dgamma / n2) * h1);
  } else if (kind == MAT_SNOW) {  // src/particles.cpp:222-242
    R det_orig = 1, det_new = 1;
    for (int i = 0; i < 2; i++) {
      det_orig *= s[i];
      sn[i] = std::min(std::max(s[i], R(1) - prm[3]), R(1) + prm[4]);
      det_new *= sn[i];
    }
    R jp = ps * det_orig / det_new;
    if (!(jp <= prm[6])) jp = prm[6];
    if (!(jp >= prm[5])) jp = prm[5];
    ps = jp;
  } else {  // MAT_SAND, src/particles.cpp:639-647
    sand_project2(prm, s, ps, sn);
  }
  usv2(U, sn, V, F);
}
template <class R> void friction_project2(const R *vel, const R *n, R friction, R *out) {  // src/mpm_fwd.h:25-57, base 0
  if (friction == R(-1)) { out[0] = out[1] = 0; return; }
  const bool slip = friction <= R(-2);
  if (slip) friction = -friction - R(2);
  const R nn = n[0] * vel[0] + n[1] * vel[1];
  const R t[2] = {vel[0] - nn * n[0], vel[1] - nn * n[1]};
  const R tn = std::sqrt(t[0] * t[0] + t[1] * t[1]);
  const R scale = std::max(tn + std::min(nn, R(0)) * friction, R(0)) / std::max(R(1e-30), tn);
  const R keep = std::max(R(0), nn * R(!slip));
  for (int d = 0; d < 2; d++) out[d] = scale * t[d] + keep * n[d];
}
// stencil start int(X - 0.5) and MPMKernel<2,2> weights (src/kernel.h:122-134, src/transfer.cpp:188-190)
template <class R> inline void weights2(const Scene2<R> &sc, const R *x, int *base, R (*w)[3], R *X) {
  for (int d = 0; d < 2; d++) {
    X[d] = x[d] * sc.inv_dx;
    base[d] = int(X[d] - R(0.5));
    R dw[3];
    quadratic_kernel_axis(X[d], w[d], dw);
  }
}
template <class R> inline bool on_grid2(const Scene2<R> &sc, const R *x) {
  if (!std::isfinite(x[0]) || !std::isfinite(x[1])) return false;
  for (int d = 0; d < 2; d++) {
    const int b = int(x[d] * sc.inv_dx - R(0.5));
    if (b < 0 || b + 2 > sc.res[d]) return false;
  }
  return true;
}
template <class R> void substep2(const Scene2<R> &sc, Particles2<R> &P, uint8_t *alive, R *grid_out, R *grid_rast_out) {
  std::vector<R> local;
  R *grid = grid_out;
  if (!grid) { local.assign(sc.n_nodes() * 4, R(0)); grid = local.data(); }
  else std::fill(grid, grid + sc.n_nodes() * 4, R(0));
  // whatever clean_boundary says, a particle whose stencil leaves the node grid is not rasterised (the engine deletes it at
  // upload; the reference would write past res into its SPGrid)
  for (int64_t i = 0; i < P.n; i++)
    if (alive[i] && !on_grid2(sc, P.x + 2 * i)) alive[i] = 0;
  // P2G (src/transfer.cpp:193-278)
  for (int64_t i = 0; i < P.n; i++) {
    if (!alive[i]) continue;
    R *v = P.v + 2 * i;
    if (sc.particle_gravity) for (int d = 0; d < 2; d++) v[d] = v[d] + sc.gravity[d] * sc.dt;
    int base[2]; R w[2][3], X[2];
    weights2(sc, P.x + 2 * i, base, w, X);
    const R mass = P.mass[i];
    const int g = P.group[i];
    R force[4], A[4], Fd[4];
    calculate_force2(sc.mat_kind[g], sc.mat_params + g * kMatParams, P.F + 4 * i, P.ps[i], P.vol[i], force);
    for (int k = 0; k < 4; k++) { A[k] = P.b[4 * i + k] * (R(4) * mass); Fd[k] = sc.dt * force[k]; }
    for (int a = 0; a < 3; a++)
      for (int c = 0; c < 3; c++) {
        const R dpos[2] = {X[0] - R(base[0] + a), X[1] - R(base[1] + c)};
        const R wt = w[0][a] * w[1][c];
        R *gn = grid + 4 * sc.node(base[0] + a, base[1] + c);
        for (int r = 0; r < 2; r++) {
          const R ad = at2(A, r, 0) * dpos[0] + at2(A, r, 1) * dpos[1];
          const R fd = at2(Fd, r, 0) * dpos[0] + at2(Fd, r, 1) * dpos[1];
          gn[r] += wt * ((mass * v[r] + ad) + (-fd * R(4) * sc.inv_dx));
        }
        gn[3] += wt * mass;
      }
  }
  if (grid_rast_out) std::memcpy(grid_rast_out, grid, sizeof(R) * sc.n_nodes() * 4);
  // grid update (src/mpm.cpp:277-372)
  R incr[2] = {0, 0};
  if (!sc.particle_gravity) for (int d = 0; d < 2; d++) incr[d] = sc.gravity[d] * sc.dt;
  const size_t nn = sc.n_nodes();
#pragma omp parallel for schedule(static)
  for (size_t nd = 0; nd < nn; nd++) {
    R *gn = grid + 4 * nd;
    const R mass = gn[3];
    if (mass > 0) for (int d = 0; d < 2; d++) gn[d] = gn[d] / mass + incr[d];
    if (sc.sdf && mass != R(0)) {
      const R *s = sc.sdf + 4 * nd;
      if (s[3] < R(-3) || R(0) < s[3]) continue;
      R out[2];
      friction_project2(gn, s, sc.friction, out);
      gn[0] = out[0]; gn[1] = out[1];
    }
  }
  // G2P (src/transfer.cpp:585-687)
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < P.n; i++) {
    if (!alive[i]) continue;
    int base[2]; R w[2][3], X[2];
    weights2(sc, P.x + 2 * i, base, w, X);
    R v[2] = {0, 0}, b[4] = {0, 0, 0, 0};
    for (int a = 0; a < 3; a++)
      for (int c = 0; c < 3; c++) {
        const R dpos[2] = {X[0] - R(base[0] + a), X[1] - R(base[1] + c)};
        const R wt = w[0][a] * w[1][c];
        const R *gn = grid + 4 * sc.node(base[0] + a, base[1] + c);
        for (int r = 0; r < 2; r++) {
          v[r] += wt * gn[r];
          for (int cc = 0; cc < 2; cc++) at2(b, r, cc) += wt * gn[r] * dpos[cc];
        }
      }
    // damp_affine_momemtum (src/mpm.h:465-469)
    const R so = (b[1] + b[2]) / 2;
    const R kr = R(1) - sc.rpic_damping, ka = R(1) - sc.apic_damping;
    R *pb = P.b + 4 * i;
    pb[0] = kr * b[0]; pb[3] = kr * b[3];
    pb[1] = kr * so + ka * (b[1] - so); pb[2] = kr * so + ka * (b[2] - so);
    P.v[2 * i] = v[0]; P.v[2 * i + 1] = v[1];
    R cdg[4];
    for (int k = 0; k < 4; k++) cdg[k] = sc.dt * (b[k] * (R(-4) * sc.inv_dx));
    cdg[0] += 1; cdg[3] += 1;
    const int g = P.group[i];
    plasticity2(sc.mat_kind[g], sc.mat_params + g * kMatParams, cdg, P.F + 4 * i, P.ps[i]);
    R *x = P.x + 2 * i;
    for (int d = 0; d < 2; d++) x[d] = x[d] + sc.dt * v[d];
    const bool finite = std::isfinite(x[0]) && std::isfinite(x[1]) && std::isfinite(v[0]) && std::isfinite(v[1]);
    for (int d = 0; d < 2; d++) x[d] = std::min(std::max(x[d] * sc.inv_dx, R(0)), R(sc.res[d]) - R(1e-6)) * sc.dx;  // position correction
    bool dead = !finite;
    if (sc.clean_boundary) {  // near_boundary: within 7 cells of a face
      const R X0 = x[0] * sc.inv_dx, X1 = x[1] * sc.inv_dx;
      dead = dead || std::min(X0, X1) < R(7) || std::max(X0 - R(sc.res[0]), X1 - R(sc.res[1])) > R(-7);
    } else {
      dead = dead || !on_grid2(sc, x);
    }
    if (dead) alive[i] = 0;
  }
}

}  // namespace

// MPM<2>: one substep (grids [res0+1][res1+1][4] = (p_x, p_y, 0, m) after P2G / (v_x, v_y, 0, m) after the update, either
// may be null; x, v [n][2], F, b [n][4] column-major) and the 2x2 material functions
#define DEFINE_2D_FOR(R, SUF)                                                                                                  \
  ORACLE_API void oracle_substep2d_##SUF(const int *res, R dx, R dt, const R *gravity, int particle_gravity, int clean_boundary, \
                                         R apic_damping, R rpic_damping, const int32_t *mat_kind, const R *mat_params,       \
                                         const R *sdf, R friction, int64_t n, R *x, R *v, R *F, R *b, const R *mass,          \
                                         const R *vol, R *ps, const int32_t *group, uint8_t *alive, R *grid_rast, R *grid_vel) { \
    Scene2<R> sc;                                                                                                              \
    for (int d = 0; d < 2; d++) { sc.res[d] = res[d]; sc.gravity[d] = gravity[d]; }                                            \
    sc.dx = dx; sc.inv_dx = R(1) / dx; sc.dt = dt;                                                                             \
    sc.particle_gravity = particle_gravity; sc.clean_boundary = clean_boundary;                                                \
    sc.apic_damping = apic_damping; sc.rpic_damping = rpic_damping;                                                            \
    sc.mat_kind = mat_kind; sc.mat_params = mat_params; sc.sdf = sdf; sc.friction = friction;                                  \
    Particles2<R> P{n, x, v, F, b, mass, vol, ps, group};                                                                      \
    substep2<R>(sc, P, alive, grid_vel, grid_rast);                                                                            \
  }                                                                                                                            \
  ORACLE_API void oracle_calculate_force2d_##SUF(int kind, const R *prm, const R *F, R ps, R vol, R *out) {                    \
    calculate_force2<R>(kind, prm, F, ps, vol, out);                                                                           \
  }                                                                                                                            \
  ORACLE_API void oracle_plasticity2d_##SUF(int kind, const R *prm, const R *cdg, R *F, R *ps) {                               \
    plasticity2<R>(kind, prm, cdg, F, *ps);                                                                                    \
  }
DEFINE_2D_FOR(float, f32)
DEFINE_2D_FOR(double, f64)
