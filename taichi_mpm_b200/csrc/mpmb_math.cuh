// Device math for the MLS-MPM substep kernels (sm_90a).
//
// All isotropic constitutive updates of the reference (src/particles.cpp) are evaluated from ONE
// decomposition: the eigen-system of the small-strain-exact tensor E = F F^T - I, built from
// G = F - I as E = G + G^T + G G^T so that the small quantity is formed without cancellation.
// With F = U S V^T:  E = U (S^2 - I) U^T, hence
//   * every Kirchhoff stress  P F^T = U diag(tau_i(sigma)) U^T          (calculate_force)
//   * every return map        U S' V^T = U diag(sigma'_i/sigma_i) U^T F (plasticity)
// needs U and e_i = sigma_i^2 - 1 only — no V, no second factorisation, and ln(sigma) =
// 0.5*log1p(e) keeps full relative precision at the 1e-4 strains sand lives at.
// The reference calls svd()/polar_decomp() of the (un-vendored) taichi core at
// src/particles.cpp:212,227,394,630,642; results here are compared against the fp64 oracle
// through convention-invariant quantities only.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

// out-of-line device function (host builds of this header — tests/host_math, tests/simt — take the GNU spelling:
// libstdc++ uses the bare word __noinline__ inside attributes, so it cannot be a macro there)
#ifdef __CUDACC__
#define MPMB_NOINLINE_DEVICE __device__ __noinline__
#else
#define MPMB_NOINLINE_DEVICE __attribute__((noinline)) inline
#endif

namespace mpmb {

enum { MAT_LINEAR = 0, MAT_JELLY = 1, MAT_SNOW = 2, MAT_WATER = 3, MAT_SAND = 4, MAT_ELASTIC = 5, MAT_VON_MISES = 6, MAT_VISCO = 7 };
// Hencky stress tau_i = 2 mu ln s_i + lambda sum ln s: sand, elastic and von Mises share calculate_force word for word
// (src/particles.cpp:628-637, 800-809, 703-712)
__device__ __forceinline__ bool is_hencky(int kind) { return kind == MAT_SAND || kind == MAT_ELASTIC || kind == MAT_VON_MISES; }

struct Mat3 {  // column-major: m[c*3+r]
  float m[9];
  __device__ __forceinline__ float &operator()(int r, int c) { return m[c * 3 + r]; }
  __device__ __forceinline__ float operator()(int r, int c) const { return m[c * 3 + r]; }
};

struct Sym3 {  // symmetric 3x3
  float xx, yy, zz, xy, xz, yz;
};

// MUFU.RSQ without the denormal pre-scaling sequence rsqrtf() expands to.
__device__ __forceinline__ float rsqrt_fast(float x) {
  float y;
#ifndef MPMB_HOST_MATH
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
#else  // tests/host_math compiles this header with g++ (no GPU): IEEE value instead of MUFU.RSQ
  y = 1.0f / sqrtf(x);
#endif
  return y;
}

// One cyclic Jacobi rotation annihilating a_pq; (app,aqq,apq) the 2x2 pivot, (arp,arq) the
// remaining off-diagonals, v*p/v*q the eigenvector columns p and q.
// Half-angle form with two MUFU.RSQ and no division:
//   d = aqq-app, b = 2 apq, h = sqrt(d^2+b^2):  cos 2t = |d|/h, sin 2t = |b|/h (smaller angle)
//   c = sqrt((1+cos 2t)/2),  s = sgn(d b) sin 2t / (2c),  tan t = s/c.
__device__ __forceinline__ void jacobi_rotate(float &app, float &aqq, float &apq, float &arp, float &arq, float &v0p,
                                              float &v1p, float &v2p, float &v0q, float &v1q, float &v2q) {
  const float d = aqq - app;
  const float b = 2.0f * apq;
  const float h2 = fmaf(d, d, b * b);
  const float inv_h = h2 > 1e-36f ? rsqrt_fast(h2) : 0.0f;
  const float c2 = fmaf(0.5f * fabsf(d), inv_h, 0.5f);  // in [0.5,1]; h2 == 0 -> 0.5 with s = 0 below (A already diagonal here)
  float rc = rsqrt_fast(c2);
  rc = rc * fmaf(-0.5f * c2, rc * rc, 1.5f);  // one Newton step: c,s orthonormal to fp32 round-off
  float c = c2 * rc;
  float s = copysignf(0.5f, d) * b * inv_h * rc;
  if (!(h2 > 1e-36f)) { c = 1.0f; s = 0.0f; rc = 1.0f; }
  const float t = s * rc;
  app = fmaf(-t, apq, app);
  aqq = fmaf(t, apq, aqq);
  apq = 0.0f;
  const float n_rp = fmaf(c, arp, -s * arq);
  const float n_rq = fmaf(s, arp, c * arq);
  arp = n_rp;
  arq = n_rq;
  const float t0 = fmaf(c, v0p, -s * v0q), t1 = fmaf(c, v1p, -s * v1q), t2 = fmaf(c, v2p, -s * v2q);
  v0q = fmaf(s, v0p, c * v0q);
  v1q = fmaf(s, v1p, c * v1q);
  v2q = fmaf(s, v2p, c * v2q);
  v0p = t0;
  v1p = t1;
  v2p = t2;
}

// Eigen-decomposition A = U diag(e) U^T by cyclic Jacobi.  Convergence is cubic: 3 sweeps leave
// off/norm < 1e-7 for 99% of random symmetric matrices (max 2e-5 over 2e5 samples); lanes still
// above 3e-7 take a fourth sweep, which reaches fp32 round-off for every sample.
template <int SWEEPS>
__device__ __forceinline__ void eig_sym3(Sym3 A, Mat3 &U, float e[3]) {
  float u00 = 1.f, u10 = 0.f, u20 = 0.f, u01 = 0.f, u11 = 1.f, u21 = 0.f, u02 = 0.f, u12 = 0.f, u22 = 1.f;
#pragma unroll
  for (int s = 0; s < SWEEPS; s++) {
    // (p,q,r) = (0,1,2): pivot xy, others xz (r=2 with p=0), yz (r=2 with q=1)
    jacobi_rotate(A.xx, A.yy, A.xy, A.xz, A.yz, u00, u10, u20, u01, u11, u21);
    // (0,2,1): pivot xz, others xy (r=1 with p=0), yz (r=1 with q=2)
    jacobi_rotate(A.xx, A.zz, A.xz, A.xy, A.yz, u00, u10, u20, u02, u12, u22);
    // (1,2,0): pivot yz, others xy (r=0 with p=1), xz (r=0 with q=2)
    jacobi_rotate(A.yy, A.zz, A.yz, A.xy, A.xz, u01, u11, u21, u02, u12, u22);
  }
  {
    const float off2 = fmaf(A.xy, A.xy, fmaf(A.xz, A.xz, A.yz * A.yz));
    const float nrm2 = fmaf(A.xx, A.xx, fmaf(A.yy, A.yy, A.zz * A.zz));
    if (off2 > 1e-13f * nrm2) {
      jacobi_rotate(A.xx, A.yy, A.xy, A.xz, A.yz, u00, u10, u20, u01, u11, u21);
      jacobi_rotate(A.xx, A.zz, A.xz, A.xy, A.yz, u00, u10, u20, u02, u12, u22);
      jacobi_rotate(A.yy, A.zz, A.yz, A.xy, A.xz, u01, u11, u21, u02, u12, u22);
    }
  }
  U.m[0] = u00; U.m[1] = u10; U.m[2] = u20;
  U.m[3] = u01; U.m[4] = u11; U.m[5] = u21;
  U.m[6] = u02; U.m[7] = u12; U.m[8] = u22;
  e[0] = A.xx; e[1] = A.yy; e[2] = A.zz;
}

// log1p with full relative precision for the small strains that dominate (|x| < 1/16: degree-7
// Taylor polynomial, error < 3e-11); library log1pf elsewhere.
__device__ __forceinline__ float log1p_strain(float x) {
  if (fabsf(x) < 0.0625f) {
    float p = fmaf(x, 1.0f / 7.0f, -1.0f / 6.0f);
    p = fmaf(p, x, 0.2f);
    p = fmaf(p, x, -0.25f);
    p = fmaf(p, x, 1.0f / 3.0f);
    p = fmaf(p, x, -0.5f);
    p = fmaf(p, x, 1.0f);
    return p * x;
  }
  return log1pf(x);
}

// E = F F^T - I from G = F - I (no cancellation for F ~ I).
__device__ __forceinline__ Sym3 left_strain(const Mat3 &F) {
  float g00 = F.m[0] - 1.f, g10 = F.m[1], g20 = F.m[2];
  float g01 = F.m[3], g11 = F.m[4] - 1.f, g21 = F.m[5];
  float g02 = F.m[6], g12 = F.m[7], g22 = F.m[8] - 1.f;
  Sym3 E;
  // (G G^T)_rs = sum_c G_rc G_sc
  E.xx = fmaf(g00, g00, fmaf(g01, g01, g02 * g02)) + 2.f * g00;
  E.yy = fmaf(g10, g10, fmaf(g11, g11, g12 * g12)) + 2.f * g11;
  E.zz = fmaf(g20, g20, fmaf(g21, g21, g22 * g22)) + 2.f * g22;
  E.xy = fmaf(g00, g10, fmaf(g01, g11, g02 * g12)) + (g01 + g10);
  E.xz = fmaf(g00, g20, fmaf(g01, g21, g02 * g22)) + (g02 + g20);
  E.yz = fmaf(g10, g20, fmaf(g11, g21, g12 * g22)) + (g12 + g21);
  return E;
}

// M = U diag(d) U^T
__device__ __forceinline__ Sym3 sym_from_eig(const Mat3 &U, const float d[3]) {
  Sym3 M;
  M.xx = fmaf(d[0] * U.m[0], U.m[0], fmaf(d[1] * U.m[3], U.m[3], d[2] * U.m[6] * U.m[6]));
  M.yy = fmaf(d[0] * U.m[1], U.m[1], fmaf(d[1] * U.m[4], U.m[4], d[2] * U.m[7] * U.m[7]));
  M.zz = fmaf(d[0] * U.m[2], U.m[2], fmaf(d[1] * U.m[5], U.m[5], d[2] * U.m[8] * U.m[8]));
  M.xy = fmaf(d[0] * U.m[0], U.m[1], fmaf(d[1] * U.m[3], U.m[4], d[2] * U.m[6] * U.m[7]));
  M.xz = fmaf(d[0] * U.m[0], U.m[2], fmaf(d[1] * U.m[3], U.m[5], d[2] * U.m[6] * U.m[8]));
  M.yz = fmaf(d[0] * U.m[1], U.m[2], fmaf(d[1] * U.m[4], U.m[5], d[2] * U.m[7] * U.m[8]));
  return M;
}

// out = S * F (S symmetric)
__device__ __forceinline__ Mat3 sym_mul(const Sym3 &S, const Mat3 &F) {
  Mat3 o;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float f0 = F.m[c * 3], f1 = F.m[c * 3 + 1], f2 = F.m[c * 3 + 2];
    o.m[c * 3 + 0] = fmaf(S.xx, f0, fmaf(S.xy, f1, S.xz * f2));
    o.m[c * 3 + 1] = fmaf(S.xy, f0, fmaf(S.yy, f1, S.yz * f2));
    o.m[c * 3 + 2] = fmaf(S.xz, f0, fmaf(S.yz, f1, S.zz * f2));
  }
  return o;
}

__device__ __forceinline__ Mat3 mat_mul(const Mat3 &A, const Mat3 &B) {
  Mat3 o;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int r = 0; r < 3; r++) o.m[c * 3 + r] = fmaf(A(r, 0), B(0, c), fmaf(A(r, 1), B(1, c), A(r, 2) * B(2, c)));
  return o;
}

struct Material {
  int kind;
  float p[8];
};

#ifndef MPMB_EIG_SWEEPS
#define MPMB_EIG_SWEEPS 3
#endif

__device__ __forceinline__ float det3(const Mat3 &A) {
  return A.m[0] * (A.m[4] * A.m[8] - A.m[7] * A.m[5]) - A.m[3] * (A.m[1] * A.m[8] - A.m[7] * A.m[2]) + A.m[6] * (A.m[1] * A.m[5] - A.m[4] * A.m[2]);
}

// Inverted elements (det F < 0).  The eigen-system of F F^T - I gives |sigma| only; the convention of the
// reference's polar_decomp()/svd() with rotations U, V in SO(3) (DESIGN.md §2) puts the sign of det F on the
// smallest singular value: F = U diag(s^) V^T with s^_k = -s_k on that axis.  Returns k, or -1 for det F >= 0.
__device__ __forceinline__ int argmin3(const float e[3]) { return e[0] <= e[1] ? (e[0] <= e[2] ? 0 : 2) : (e[1] <= e[2] ? 1 : 2); }
__device__ __forceinline__ int reflected_axis(const Mat3 &F, const float e[3]) { return det3(F) < 0.f ? argmin3(e) : -1; }

// Fixed-corotated Kirchhoff stress in principal space from en_i = s_i^2 - 1 (s_i >= 0) and the reflected axis
// `flip` (-1: none):  tau_i = 2 mu s^_i (s^_i - 1) + lambda (J-1) J,  J = prod s^ (signed).
// Kept axes use s - 1 = e/(s+1) and J - 1 = (J^2-1)/(J+1) (no cancellation near I); on the reflected axis
// s^(s^-1) = s(s+1) and J <= 0, where those forms would divide by zero at s^ = -1, J = -1.
__device__ __forceinline__ void fixed_corotated_tau(float mu, float la, const float en[3], int flip, float tau[3]) {
  const float s[3] = {sqrtf(fmaxf(1.f + en[0], 0.f)), sqrtf(fmaxf(1.f + en[1], 0.f)), sqrtf(fmaxf(1.f + en[2], 0.f))};
  float J = s[0] * s[1] * s[2];
  float Jm1;
  if (flip >= 0) {
    J = -J;
    Jm1 = J - 1.f;
  } else {
    const float J2m1 = (en[0] + en[1] + en[2]) + fmaf(en[0], en[1], fmaf(en[0], en[2], en[1] * en[2])) + en[0] * en[1] * en[2];
    Jm1 = J2m1 / (J + 1.f);
  }
  const float vol_term = la * Jm1 * J;
#pragma unroll
  for (int i = 0; i < 3; i++) tau[i] = fmaf(2.f * mu * s[i], i == flip ? s[i] + 1.f : en[i] / (s[i] + 1.f), vol_term);
}

// F' = U diag(r) U^T Ft with the part along axis k rebuilt as sig_k u_k v_k^T.  With m = U^T Ft (rows s^_i v_i^T)
// and U, V in SO(3), v_k = v_i x v_j = unit(m_i x m_j) for (i,j,k) cyclic, whatever s^_k is: the return maps
// take this for the smallest axis where the ratio sig_k / s_k would divide by a vanishing (or 1e-4-clamped)
// singular value that F F^T - I resolves only to ~1e-7 / s_k.  Needs s_i, s_j > 0 (rank >= 2).
// Arguments by value (see ViscoOut below): out of line, on a path physical states never take.
MPMB_NOINLINE_DEVICE Mat3 rebuild_small_axis(Mat3 U, float r0, float r1, float r2, int k, float sig_k, Mat3 Ft) {
  const float r[3] = {k == 0 ? 0.f : r0, k == 1 ? 0.f : r1, k == 2 ? 0.f : r2};
  Mat3 F = sym_mul(sym_from_eig(U, r), Ft);
  const int i = k == 2 ? 0 : k + 1, j = k == 0 ? 2 : k - 1;
  float mi[3], mj[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {  // m_i[c] = sum_r U(r,i) Ft(r,c)
    mi[c] = fmaf(U.m[i * 3], Ft.m[c * 3], fmaf(U.m[i * 3 + 1], Ft.m[c * 3 + 1], U.m[i * 3 + 2] * Ft.m[c * 3 + 2]));
    mj[c] = fmaf(U.m[j * 3], Ft.m[c * 3], fmaf(U.m[j * 3 + 1], Ft.m[c * 3 + 1], U.m[j * 3 + 2] * Ft.m[c * 3 + 2]));
  }
  const float v[3] = {mi[1] * mj[2] - mi[2] * mj[1], mi[2] * mj[0] - mi[0] * mj[2], mi[0] * mj[1] - mi[1] * mj[0]};
  const float n2 = fmaf(v[0], v[0], fmaf(v[1], v[1], v[2] * v[2]));
  const float sc = n2 > 0.f ? sig_k / sqrtf(n2) : 0.f;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int rr = 0; rr < 3; rr++) F.m[c * 3 + rr] = fmaf(sc * U.m[k * 3 + rr], v[c], F.m[c * 3 + rr]);
  return F;
}

// -vol * P(F) F^T  ==  the value of Particle::calculate_force() (src/particles.cpp:216-218,
// 335-337,409-411,463-467,628-637), returned as a symmetric tensor where it is one (all kinds
// except LINEAR, whose P F^T is not symmetric for finite strain).
// Returns through `out` (column-major full matrix).
__device__ __forceinline__ void calculate_force(const Material &mat, const Mat3 &F, float ps, float vol, Mat3 &out) {
  if (mat.kind == MAT_WATER) {
    // p = k (j^-gamma - 1); sigma = -p I; force = -vol j sigma = vol j p I   (463-467)
    float j = ps;
    float p = mat.p[0] * (powf(j, -mat.p[1]) - 1.0f);
    float d = vol * j * p;
#pragma unroll
    for (int i = 0; i < 9; i++) out.m[i] = 0.f;
    out.m[0] = d; out.m[4] = d; out.m[8] = d;
    return;
  }
  if (mat.kind == MAT_LINEAR) {
    // P = mu (F + F^T - 2I) + lambda (tr F - 3) I ; force = -vol P F^T   (329-337)
    float mu = mat.p[0], la = mat.p[1];
    Mat3 P;
    float tr = (F.m[0] - 1.f) + (F.m[4] - 1.f) + (F.m[8] - 1.f);
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
      for (int r = 0; r < 3; r++) {
        float g = (F(r, c) - (r == c ? 1.f : 0.f)) + (F(c, r) - (r == c ? 1.f : 0.f));
        P(r, c) = mu * g + (r == c ? la * tr : 0.f);
      }
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
      for (int r = 0; r < 3; r++) {
        // (P F^T)_rc = sum_k P_rk F_ck
        float s = fmaf(P(r, 0), F(c, 0), fmaf(P(r, 1), F(c, 1), P(r, 2) * F(c, 2)));
        out(r, c) = -vol * s;
      }
    return;
  }
  Mat3 U;
  float e[3];
  eig_sym3<MPMB_EIG_SWEEPS>(left_strain(F), U, e);
  float tau[3];
  if (is_hencky(mat.kind)) {
    // tau_i = 2 mu ln s_i + lambda sum ln s   (628-637: U (2mu S^-1 lnS + lambda tr(lnS) S^-1) V^T F^T)
    float mu = mat.p[0], la = mat.p[1];
    float l0 = 0.5f * log1p_strain(e[0]), l1 = 0.5f * log1p_strain(e[1]), l2 = 0.5f * log1p_strain(e[2]);
    float tr = la * (l0 + l1 + l2);
    tau[0] = fmaf(2.f * mu, l0, tr);
    tau[1] = fmaf(2.f * mu, l1, tr);
    tau[2] = fmaf(2.f * mu, l2, tr);
  } else {
    // fixed corotated (jelly 391-398, snow 207-214, visco 69-82): P F^T = 2mu (F-R)F^T + lambda (J-1) J I
    //   (F-R)F^T = U diag(s^(s^-1)) U^T with R in SO(3) and J = det F signed (fixed_corotated_tau)
    float mu = mat.p[0], la = mat.p[1];
    if (mat.kind == MAT_SNOW) {
      float h = __expf(mat.p[2] * (1.0f - ps));  // 244-252
      mu *= h;
      la *= h;
    }
    fixed_corotated_tau(mu, la, e, reflected_axis(F, e), tau);
  }
  tau[0] *= -vol; tau[1] *= -vol; tau[2] *= -vol;
  Sym3 T = sym_from_eig(U, tau);
  out.m[0] = T.xx; out.m[1] = T.xy; out.m[2] = T.xz;
  out.m[3] = T.xy; out.m[4] = T.yy; out.m[5] = T.yz;
  out.m[6] = T.xz; out.m[7] = T.yz; out.m[8] = T.zz;
}

// VonMisesParticle::plasticity (src/particles.cpp:714-734) in principal log strains: eps = ln s, hat = dev(eps),
// n2 = |hat|^2 — `frobenius_norm2()` at 724 is the SQUARED norm, and that is what enters both the yield test
// dgamma = n2 - yield/(2 mu) and the scaling dgamma/n2 — returns sigma'/sigma per axis and (optionally) ln sigma'.
__device__ __forceinline__ bool von_mises_return(const Material &mat, const float e[3], float ratio[3], float *lsn) {
  float ls[3];
#pragma unroll
  for (int i = 0; i < 3; i++) ls[i] = 0.5f * log1p_strain(e[i]);
  const float tr3 = (ls[0] + ls[1] + ls[2]) * (1.f / 3.f);
  const float hat[3] = {ls[0] - tr3, ls[1] - tr3, ls[2] - tr3};
  const float n2 = fmaf(hat[0], hat[0], fmaf(hat[1], hat[1], hat[2] * hat[2]));
  const float dg = n2 - mat.p[2] / (2.f * mat.p[0]);
  const bool yield = dg > 0.f;
  const float k = yield ? dg / n2 : 0.f;
#pragma unroll
  for (int i = 0; i < 3; i++) {
    ratio[i] = yield ? __expf(-k * hat[i]) : 1.f;
    if (lsn) lsn[i] = fmaf(-k, hat[i], ls[i]);
  }
  return yield;
}

// ViscoParticle::plasticity (src/particles.cpp:104-137) + the fixed-corotated stress of the new state (69-82).
// ps = visco_tau.  Kept out of line: a rarely used material must not shape the register allocation of k_g2p.
//   F^ = approximate_exponent(dt_p, (cdg - I)/dt_p) F   (89-102: (s/2 + I) s + I, halving while det <= 0)
//   pnorm = |P(F_old)|_F = sqrt(sum_i (2 mu (s_i - 1) + lambda (J-1) J / s_i)^2)   (111: dg_e is not yet updated)
//   gamma = clamp(dt_p nu (pnorm - tau)/pnorm, 0, 1);  sigma' = clamp(sigma / (sigma / det^(1/3))^gamma, 0.1, 10)
// Both SVDs of the reference share the factors of F^, so one symmetric eigen-decomposition serves.
// Everything crosses the call BY VALUE: a reference parameter of an out-of-line function would force the caller's
// matrices (and the kernel's material table) into local memory on every path, not only on this one.
struct ViscoOut {
  Mat3 F, force;
  float ps;
};
MPMB_NOINLINE_DEVICE ViscoOut visco_step_impl(float mu, float la, float nu, float kappa, float dtp, Mat3 cdg, Mat3 F, float ps, float vol) {
  Mat3 force;
  // pnorm of the old state (eigenvalues only)
  float pnorm;
  {
    Mat3 U0;
    float e0[3];
    eig_sym3<MPMB_EIG_SWEEPS>(left_strain(F), U0, e0);
    const int fk = reflected_axis(F, e0);  // P of an inverted F with R in SO(3): signed s^, J
    const float s0 = (fk == 0 ? -1.f : 1.f) * sqrtf(fmaxf(1.f + e0[0], 0.f)), s1 = (fk == 1 ? -1.f : 1.f) * sqrtf(fmaxf(1.f + e0[1], 0.f)),
                s2 = (fk == 2 ? -1.f : 1.f) * sqrtf(fmaxf(1.f + e0[2], 0.f));
    const float J = s0 * s1 * s2;
    const float vt = la * (J - 1.f) * J;
    const float p0 = fmaf(2.f * mu, s0 - 1.f, vt / s0), p1 = fmaf(2.f * mu, s1 - 1.f, vt / s1), p2 = fmaf(2.f * mu, s2 - 1.f, vt / s2);
    pnorm = sqrtf(fmaf(p0, p0, fmaf(p1, p1, p2 * p2)));
  }
  // approximate exponent of (cdg - I)
  Mat3 m;
#pragma unroll
  for (int i = 0; i < 9; i++) m.m[i] = (cdg.m[i] - ((i & 3) == 0 ? 1.f : 0.f)) * (1.0f / dtp);
  Mat3 ex;
  int halvings = 0;
  float dth = dtp;
  for (;;) {
    Mat3 sm, h;
#pragma unroll
    for (int i = 0; i < 9; i++) { sm.m[i] = m.m[i] * dth; h.m[i] = sm.m[i] * 0.5f + ((i & 3) == 0 ? 1.f : 0.f); }
    ex = mat_mul(h, sm);
    ex.m[0] += 1.f; ex.m[4] += 1.f; ex.m[8] += 1.f;
    if (det3(ex) > 0.f || halvings >= 16) break;
    dth *= 0.5f;
    halvings++;
  }
  for (int k = 0; k < halvings; k++) ex = mat_mul(ex, ex);
  const Mat3 Fh = mat_mul(ex, F);
  Mat3 U;
  float e[3];
  eig_sym3<MPMB_EIG_SWEEPS>(left_strain(Fh), U, e);
  float gamma = 0.f;
  if (pnorm > 1e-5f) gamma = fminf(fmaxf(dtp * nu * (pnorm - ps) / pnorm, 0.f), 1.f);
  float sg[3] = {sqrtf(fmaxf(1.f + e[0], 0.f)), sqrtf(fmaxf(1.f + e[1], 0.f)), sqrtf(fmaxf(1.f + e[2], 0.f))};
  const float det = sg[0] * sg[1] * sg[2];
  const float scale = fabsf(det) > 1e-5f ? 1.0f / cbrtf(det) : 1.0f;
  float ratio[3], en[3], sn[3];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const float mid = powf(sg[i] * scale, gamma);
    const float mid_inv = fabsf(mid) > 1e-5f ? 1.0f / mid : 1.0f;
    sn[i] = fminf(fmaxf(sg[i] * mid_inv, 0.1f), 10.0f);
    ratio[i] = sn[i] / sg[i];
    en[i] = fmaf(sn[i], sn[i], -1.f);
  }
  ps = fmaf(kappa * gamma, pnorm, ps);
  // the return map reads |sigma| (the reference's pow(det, 1/3) and log of a negative sigma are NaN, DESIGN.md §2):
  // an inverted F^ stays inverted, on the same (smallest) axis
  const int k = argmin3(e), flip = det3(Fh) < 0.f ? k : -1;
  if (1.f + e[k] < 1e-2f) F = rebuild_small_axis(U, ratio[0], ratio[1], ratio[2], k, flip >= 0 ? -sn[k] : sn[k], Fh);
  else F = sym_mul(sym_from_eig(U, ratio), Fh);
  float tau[3];
  fixed_corotated_tau(mu, la, en, flip, tau);
  tau[0] *= -vol; tau[1] *= -vol; tau[2] *= -vol;
  const Sym3 T = sym_from_eig(U, tau);
  force.m[0] = T.xx; force.m[1] = T.xy; force.m[2] = T.xz;
  force.m[3] = T.xy; force.m[4] = T.yy; force.m[5] = T.yz;
  force.m[6] = T.xz; force.m[7] = T.yz; force.m[8] = T.zz;
  ViscoOut o;
  o.F = F;
  o.force = force;
  o.ps = ps;
  return o;
}
__device__ __forceinline__ void visco_step(const Material &mat, const Mat3 &cdg, Mat3 &F, float &ps, float vol, Mat3 &force) {
  const ViscoOut o = visco_step_impl(mat.p[0], mat.p[1], mat.p[2], mat.p[3], mat.p[4], cdg, F, ps, vol);
  F = o.F;
  force = o.force;
  ps = o.ps;
}

// Particle::plasticity(cdg) (src/particles.cpp:222-242,340-344,413-416,469-478,639-647):
// F <- cdg F, then the return map of the material; ps is Jp / j / logJp.
__device__ __forceinline__ void plasticity(const Material &mat, const Mat3 &cdg, Mat3 &F, float &ps) {
  if (mat.kind == MAT_WATER) {
    ps *= (cdg.m[0] + cdg.m[4] + cdg.m[8]) - 2.0f;  // j *= tr(cdg) - (dim-1)
    if (ps < 0.1f) ps = 0.1f;
    return;
  }
  if (mat.kind == MAT_VISCO) {
    Mat3 force;
    visco_step(mat, cdg, F, ps, 0.f, force);
    return;
  }
  Mat3 Ft = mat_mul(cdg, F);
  if (mat.kind == MAT_LINEAR || mat.kind == MAT_JELLY || mat.kind == MAT_ELASTIC) {
    F = Ft;
    return;
  }
  Mat3 U;
  float e[3];
  eig_sym3<MPMB_EIG_SWEEPS>(left_strain(Ft), U, e);
  float ratio[3], sig_k = 0.f;
  bool changed;
  const int k = argmin3(e), flip = det3(Ft) < 0.f ? k : -1;
  if (mat.kind == MAT_VON_MISES) {
    changed = von_mises_return(mat, e, ratio, nullptr);
    sig_k = (flip >= 0 ? -1.f : 1.f) * sqrtf(fmaxf(1.f + e[k], 0.f)) * ratio[k];
  } else if (mat.kind == MAT_SNOW) {
    // signed sigma^ clamped to [1-theta_c, 1+theta_s]; Jp <- clamp(Jp * prod(s^)/prod(s'))   (222-242)
    float lo = 1.f - mat.p[3], hi = 1.f + mat.p[4];
    float prod = 1.f;
    changed = false;
#pragma unroll
    for (int i = 0; i < 3; i++) {
      float s = (i == flip ? -1.f : 1.f) * sqrtf(fmaxf(1.f + e[i], 0.f));
      float sc = fminf(fmaxf(s, lo), hi);
      ratio[i] = sc / s;
      prod *= s / sc;
      changed |= (sc != s);
      if (i == k) sig_k = sc;
    }
    float Jp = ps * prod;
    if (!(Jp <= mat.p[6])) Jp = mat.p[6];
    if (!(Jp >= mat.p[5])) Jp = mat.p[5];
    ps = Jp;
  } else {
    // SandParticle::project (599-626) in log-strain space
    float mu = mat.p[0], la = mat.p[1], alpha = mat.p[2], coh = mat.p[3], beta = mat.p[4];
    float ls[3], eps[3];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 3; i++) {
      // ln max(|s|,1e-4) with s = sqrt(1+e) >= 0 (clamped after the log: 1e-8f - 1.f rounds to -1.f)
      ls[i] = fmaxf(0.5f * log1pf(e[i]), -9.21034037f);
      eps[i] = ls[i] - coh;
      sum += eps[i];
    }
    float tr = sum + ps;
    float hat[3] = {eps[0] - tr * (1.f / 3.f), eps[1] - tr * (1.f / 3.f), eps[2] - tr * (1.f / 3.f)};
    float hn = sqrtf(fmaf(hat[0], hat[0], fmaf(hat[1], hat[1], hat[2] * hat[2])));
    if (tr >= 0.f) {
      // sigma' = e^c I ; logJp += beta * sum(eps)
#pragma unroll
      for (int i = 0; i < 3; i++) ratio[i] = __expf(coh - ls[i]);
      ps = fmaf(beta, sum, ps);
      changed = true;
      sig_k = __expf(coh);
    } else {
      ps = 0.f;
      float dg = hn + (3.f * la + 2.f * mu) / (2.f * mu) * tr * alpha;
      if (dg <= 0.f) {
#pragma unroll
        for (int i = 0; i < 3; i++) ratio[i] = 1.f;
        // NB the reference still rebuilds F = U exp(eps+c) V^T here, which equals cdg F up to rounding
        // unless a singular value was clamped at 1e-4 (the smallest axis, rebuilt below) or F is inverted
        changed = ls[k] <= -9.21034037f;
        sig_k = __expf(ls[k]);
      } else {
        float kp = dg / hn;
#pragma unroll
        for (int i = 0; i < 3; i++) ratio[i] = expf(-kp * hat[i]);
        changed = true;
        sig_k = __expf(ls[k] - kp * hat[k]);
      }
    }
    // project() reads |sigma| and returns sigma' > 0: an inverted F comes out un-inverted
    if (flip >= 0) {
      ratio[k] = -ratio[k];
      changed = true;
    }
  }
  if (changed && 1.f + e[k] < 1e-2f) {
    F = rebuild_small_axis(U, ratio[0], ratio[1], ratio[2], k, sig_k, Ft);
  } else if (changed) {
    Sym3 M = sym_from_eig(U, ratio);
    F = sym_mul(M, Ft);
  } else {
    F = Ft;
  }
}

// Stress tensor (column-major full matrix) from its eigen-form: out = U diag(tau) U^T
__device__ __forceinline__ void store_sym(const Sym3 &T, Mat3 &out) {
  out.m[0] = T.xx; out.m[1] = T.xy; out.m[2] = T.xz;
  out.m[3] = T.xy; out.m[4] = T.yy; out.m[5] = T.yz;
  out.m[6] = T.xz; out.m[7] = T.yz; out.m[8] = T.zz;
}

// ---- symmetric 3x3 helpers for the decomposition-free sand path
__device__ __forceinline__ Sym3 sym_mul_sym(const Sym3 &A, const Sym3 &B) {  // valid when A and B commute
  Sym3 C;
  C.xx = fmaf(A.xx, B.xx, fmaf(A.xy, B.xy, A.xz * B.xz));
  C.yy = fmaf(A.xy, B.xy, fmaf(A.yy, B.yy, A.yz * B.yz));
  C.zz = fmaf(A.xz, B.xz, fmaf(A.yz, B.yz, A.zz * B.zz));
  C.xy = fmaf(A.xx, B.xy, fmaf(A.xy, B.yy, A.xz * B.yz));
  C.xz = fmaf(A.xx, B.xz, fmaf(A.xy, B.yz, A.xz * B.zz));
  C.yz = fmaf(A.xy, B.xz, fmaf(A.yy, B.yz, A.yz * B.zz));
  return C;
}
__device__ __forceinline__ float sym_norm2(const Sym3 &A) {
  return fmaf(A.xx, A.xx, fmaf(A.yy, A.yy, A.zz * A.zz)) + 2.0f * fmaf(A.xy, A.xy, fmaf(A.xz, A.xz, A.yz * A.yz));
}

// Largest value of `v` over the lanes currently executing together (loop trip counts are made
// warp-uniform with it so that the series loops never diverge).
__device__ __forceinline__ int warp_max_active(int v) { return __reduce_max_sync(__activemask(), v); }

// L = log(I + E) for a small symmetric E by the Mercator series in Horner form,
//   L = E (I - E (I/2 - E (I/3 - ...))),  N terms, fully unrolled with immediate coefficients.
// The innermost product E (I/N) is written as the scaling it is.
template <int N>
__device__ __forceinline__ Sym3 sym_log1p_horner(const Sym3 &E) {
  float c = 1.0f / (float)N;
  Sym3 T = {c * E.xx, c * E.yy, c * E.zz, c * E.xy, c * E.xz, c * E.yz};
  Sym3 S;
#pragma unroll
  for (int k = N - 1; k >= 1; k--) {
    c = 1.0f / (float)k;
    S.xx = c - T.xx; S.yy = c - T.yy; S.zz = c - T.zz;
    S.xy = -T.xy; S.xz = -T.xz; S.yz = -T.yz;
    T = sym_mul_sym(E, S);
  }
  return T;
}

// n is chosen from |E| so that the truncation, relative to |L| ~ |E|, |E|^(n-1)/(n+1) <= 1e-7, and
// is the same for the whole warp (one uniform branch, no divergence).  Caller guarantees
// |E|_F <= 0.15.
__device__ __forceinline__ Sym3 sym_log1p_series(const Sym3 &E, float nrm2) {
  int n = 3;
  if (nrm2 > 4.0e-7f) n = 4;    // |E| > 6.3e-4
  if (nrm2 > 6.2e-5f) n = 5;    // |E| > 7.9e-3
  if (nrm2 > 7.8e-4f) n = 6;    // |E| > 2.8e-2
  if (nrm2 > 3.5e-3f) n = 7;    // |E| > 5.9e-2
  if (nrm2 > 9.2e-3f) n = 9;    // |E| > 9.6e-2 (up to 0.15)
  n = warp_max_active(n);
  switch (n) {
    case 3: return sym_log1p_horner<3>(E);
    case 4: return sym_log1p_horner<4>(E);
    case 5: return sym_log1p_horner<5>(E);
    case 6: return sym_log1p_horner<6>(E);
    case 7: return sym_log1p_horner<7>(E);
    default: return sym_log1p_horner<9>(E);
  }
}

// exp(X) for a small symmetric X: I + X (I + X/2 (I + X/3 (...))), N terms unrolled; the innermost
// factor (I + X/N) is formed directly.
template <int N>
__device__ __forceinline__ Sym3 sym_exp_horner(const Sym3 &X) {
  float c = 1.0f / (float)N;
  Sym3 S = {fmaf(c, X.xx, 1.f), fmaf(c, X.yy, 1.f), fmaf(c, X.zz, 1.f), c * X.xy, c * X.xz, c * X.yz};
#pragma unroll
  for (int k = N - 1; k >= 1; k--) {
    const Sym3 T = sym_mul_sym(X, S);
    c = 1.0f / (float)k;
    S.xx = fmaf(c, T.xx, 1.f); S.yy = fmaf(c, T.yy, 1.f); S.zz = fmaf(c, T.zz, 1.f);
    S.xy = c * T.xy; S.xz = c * T.xz; S.yz = c * T.yz;
  }
  return S;
}

// truncation relative to |X|, |X|^n/(n+1)! <= 1e-7; warp-uniform term count.  Caller guarantees
// |X|_F <= 0.28.
__device__ __forceinline__ Sym3 sym_exp_series(const Sym3 &X, float nrm2) {
  int n = 3;
  if (nrm2 > 1.7e-4f) n = 4;    // |X| > 1.3e-2
  if (nrm2 > 3.5e-3f) n = 6;    // |X| > 5.9e-2 (up to 0.28)
  n = warp_max_active(n);
  switch (n) {
    case 3: return sym_exp_horner<3>(X);
    case 4: return sym_exp_horner<4>(X);
    default: return sym_exp_horner<6>(X);
  }
}

// Drucker-Prager sand WITHOUT any matrix decomposition (valid while |F F^T - I| <= 0.15; returns
// false for the lanes that must fall back to the eigen path).  SandParticle::project
// (src/particles.cpp:599-626) acts on the principal log strains only through the invariants tr and
// |hat|, with  hat_i = eps_i - tr/3,  tr = sum(eps) + logJp,  eps_i = ln s_i - c,  i.e. through the
// TENSOR  Hat = dev(L) - (logJp/3) I,  L = 1/2 log(F F^T); the three cases read
//   tr >= 0      : L' = c I                        F' = e^c exp(-L) Ft
//   dgamma <= 0  : L' = L                          F' = Ft
//   else         : L' = L - k Hat, k=dgamma/|Hat|   F' = exp(-k Hat) Ft
// and calculate_force of the new state is -vol (2 mu L' + lambda tr(L') I)  (628-637).
// All three cases run ONE instruction stream (selects, one exp series), so a warp whose lanes sit
// in different cases does not diverge.
__device__ __forceinline__ bool sand_step_series(const Material &mat, const Mat3 &Ft, Mat3 &F, float &ps, float vol, Mat3 &force) {
  const Sym3 E = left_strain(Ft);
  const float nE2 = sym_norm2(E);
  // log(I + E) is the log strain only for det Ft > 0: a reflection (E = 0 for F = diag(1,1,-1)) must take the
  // eigen path, which un-inverts it as project() does
  const bool small = nE2 <= 0.0225f && det3(Ft) > 0.f;
  const float mu = mat.p[0], la = mat.p[1], alpha = mat.p[2], coh = mat.p[3], beta = mat.p[4];
  Sym3 L = sym_log1p_series(E, small ? nE2 : 0.f);
  L.xx *= 0.5f; L.yy *= 0.5f; L.zz *= 0.5f; L.xy *= 0.5f; L.xz *= 0.5f; L.yz *= 0.5f;
  const float trL = L.xx + L.yy + L.zz;
  const float sum = trL - 3.0f * coh;   // sum of eps_i
  const float tr = sum + ps;
  const float sh = (trL + ps) * (1.f / 3.f);
  const Sym3 H = {L.xx - sh, L.yy - sh, L.zz - sh, L.xy, L.xz, L.yz};  // Hat = dev(L) - (ps/3) I
  const float hn2 = sym_norm2(H);
  // |Hat| and 1/|Hat| from one MUFU.RSQ (2 ulp; the clamp keeps rsqrt finite, and |Hat| = 0 then
  // gives dg <= 0 whenever tr < 0, i.e. no projection, so 1/|Hat| is never used at the clamp)
  const float rhn = rsqrt_fast(fmaxf(hn2, 1e-36f));
  const float hn = hn2 * rhn;
  const float dg = fmaf(fmaf(1.5f, __fdividef(la, mu), 1.f) * alpha, tr, hn);  // hn + (3la+2mu)/(2mu) tr alpha
  const bool expand = tr >= 0.f;
  const bool project = !expand && dg > 0.f;
  // X = -L (expansion), -k Hat (projection), 0 (elastic)
  const float kf = expand ? 1.f : (project ? dg * rhn : 0.f);
  const Sym3 B = expand ? L : H;
  const Sym3 X = {-kf * B.xx, -kf * B.yy, -kf * B.zz, -kf * B.xy, -kf * B.xz, -kf * B.yz};
  const float nX2 = sym_norm2(X);
  const bool ok = small && nX2 <= 0.078f;
  if (__any_sync(__activemask(), kf != 0.f)) {
    Sym3 M = sym_exp_series(X, ok ? nX2 : 0.f);
    const float ec = expand ? __expf(coh) : 1.f;
    M.xx *= ec; M.yy *= ec; M.zz *= ec; M.xy *= ec; M.xz *= ec; M.yz *= ec;
    F = (kf != 0.f) ? sym_mul(M, Ft) : Ft;
  } else {
    F = Ft;
  }
  if (!ok) return false;
  ps = expand ? fmaf(beta, sum, ps) : 0.f;
  // log strain of the new state
  Sym3 Ln;
  Ln.xx = expand ? coh : L.xx + X.xx;
  Ln.yy = expand ? coh : L.yy + X.yy;
  Ln.zz = expand ? coh : L.zz + X.zz;
  Ln.xy = expand ? 0.f : L.xy + X.xy;
  Ln.xz = expand ? 0.f : L.xz + X.xz;
  Ln.yz = expand ? 0.f : L.yz + X.yz;
  const float t3 = la * (Ln.xx + Ln.yy + Ln.zz);
  const float m2 = 2.f * mu;
  const Sym3 T = {-vol * fmaf(m2, Ln.xx, t3), -vol * fmaf(m2, Ln.yy, t3), -vol * fmaf(m2, Ln.zz, t3), -vol * m2 * Ln.xy, -vol * m2 * Ln.xz,
                  -vol * m2 * Ln.yz};
  store_sym(T, force);
  return true;
}

// G2P-side constitutive step: Particle::plasticity(cdg) (src/particles.cpp:222-242,340-344,413-416,
// 469-478,639-647) followed by the value Particle::calculate_force() will return at the NEXT
// rasterize for the updated state (src/particles.cpp:216-218,335-337,409-411,463-467,628-637).
// Both come out of ONE eigen-decomposition: F_new = U S' V^T shares U with the trial state, so
// -vol P F^T = U diag(-vol tau(S')) U^T needs no second factorisation.
// EXT = false compiles the elastic / von Mises / visco branches out: k_g2p is instantiated both ways and the host
// launches the lean one while no material group uses those kinds (the three extra branches slow the common kinds through
// code layout alone).
template <bool EXT = true>
__device__ __forceinline__ void material_step(const Material &mat, const Mat3 &cdg, Mat3 &F, float &ps, float vol, Mat3 &force) {
  if (mat.kind == MAT_WATER) {
    ps *= (cdg.m[0] + cdg.m[4] + cdg.m[8]) - 2.0f;  // j *= tr(cdg) - (dim-1)
    if (ps < 0.1f) ps = 0.1f;
    calculate_force(mat, F, ps, vol, force);
    return;
  }
  if (EXT && mat.kind == MAT_VISCO) {
    visco_step(mat, cdg, F, ps, vol, force);
    return;
  }
  const Mat3 Ft = mat_mul(cdg, F);
  if (mat.kind == MAT_LINEAR) {
    F = Ft;
    calculate_force(mat, F, ps, vol, force);
    return;
  }
  if (mat.kind == MAT_SAND) {
    if (sand_step_series(mat, Ft, F, ps, vol, force)) return;
    // large strain: principal-space evaluation below (F is recomputed from Ft, ps is untouched)
  }
  Mat3 U;
  float e[3];
  eig_sym3<MPMB_EIG_SWEEPS>(left_strain(Ft), U, e);
  float ratio[3], tau[3];
  bool changed = false;
  // the smallest axis carries the sign of det Ft (-1: not inverted) and, for the return maps, is rebuilt from the
  // other two where its singular value is too small to divide by (rebuild_small_axis); sig_k is its new s^
  const int k = argmin3(e), flip = reflected_axis(Ft, e);
  float sig_k = 0.f;
  if (EXT && (mat.kind == MAT_ELASTIC || mat.kind == MAT_VON_MISES)) {
    // Hencky elasticity (src/particles.cpp:800-814) with the von Mises return map (714-734) where asked for.
    // Both read |sigma| (the reference's log of a negative sigma is NaN): an inverted element stays inverted.
    const float mu = mat.p[0], la = mat.p[1];
    float lsn[3];
    if (mat.kind == MAT_VON_MISES) {
      changed = von_mises_return(mat, e, ratio, lsn);
      sig_k = (flip >= 0 ? -1.f : 1.f) * sqrtf(fmaxf(1.f + e[k], 0.f)) * ratio[k];
    } else {
#pragma unroll
      for (int i = 0; i < 3; i++) lsn[i] = 0.5f * log1p_strain(e[i]);
    }
    const float trl = la * (lsn[0] + lsn[1] + lsn[2]);
#pragma unroll
    for (int i = 0; i < 3; i++) tau[i] = -vol * fmaf(2.f * mu, lsn[i], trl);
  } else if (mat.kind == MAT_SAND) {
    const float mu = mat.p[0], la = mat.p[1], alpha = mat.p[2], coh = mat.p[3], beta = mat.p[4];
    float ls[3], eps[3];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 3; i++) {
      // ln max(|s|,1e-4), s = sqrt(1+e); clamped after the log (1e-8f - 1.f rounds to -1.f, log1p(-1) = -inf; fmaxf drops a NaN)
      ls[i] = fmaxf(0.5f * log1p_strain(e[i]), -9.21034037f);
      eps[i] = ls[i] - coh;
      sum += eps[i];
    }
    const float tr = sum + ps;
    const float hat[3] = {eps[0] - tr * (1.f / 3.f), eps[1] - tr * (1.f / 3.f), eps[2] - tr * (1.f / 3.f)};
    const float hn = sqrtf(fmaf(hat[0], hat[0], fmaf(hat[1], hat[1], hat[2] * hat[2])));
    float lsn[3];  // ln of the new singular values
    if (tr >= 0.f) {
#pragma unroll
      for (int i = 0; i < 3; i++) { ratio[i] = __expf(coh - ls[i]); lsn[i] = coh; }
      ps = fmaf(beta, sum, ps);
      changed = true;
    } else {
      ps = 0.f;
      const float dg = hn + (3.f * la + 2.f * mu) / (2.f * mu) * tr * alpha;
      if (dg <= 0.f) {
#pragma unroll
        for (int i = 0; i < 3; i++) { ratio[i] = 1.f; lsn[i] = ls[i]; }
        // the reference rebuilds F = U exp(eps+c) V^T, which equals Ft up to rounding unless the smallest singular
        // value was clamped at 1e-4 (rebuilt below) or Ft is inverted
        changed = ls[k] <= -9.21034037f;
      } else {
        const float kp = dg / hn;
#pragma unroll
        for (int i = 0; i < 3; i++) { ratio[i] = __expf(-kp * hat[i]); lsn[i] = fmaf(-kp, hat[i], ls[i]); }
        changed = true;
      }
    }
    // project() reads |sigma| and returns sigma' > 0: an inverted element comes out un-inverted
    if (flip >= 0) {
      ratio[k] = -ratio[k];
      changed = true;
    }
    sig_k = __expf(lsn[k]);
    const float trl = la * (lsn[0] + lsn[1] + lsn[2]);
#pragma unroll
    for (int i = 0; i < 3; i++) tau[i] = -vol * fmaf(2.f * mu, lsn[i], trl);
  } else {
    // fixed corotated family.  JELLY: no return map; SNOW: clamp of the signed s^ + hardening with the NEW Jp.
    float mu = mat.p[0], la = mat.p[1];
    float en[3] = {e[0], e[1], e[2]};  // s'^2 - 1 of the new state
    int flip_new = flip;
    if (mat.kind == MAT_SNOW) {
      const float lo = 1.f - mat.p[3], hi = 1.f + mat.p[4];
      float prod = 1.f;
#pragma unroll
      for (int i = 0; i < 3; i++) {
        const float s = (i == flip ? -1.f : 1.f) * sqrtf(fmaxf(1.f + e[i], 0.f));
        const float sc = fminf(fmaxf(s, lo), hi);
        if (sc != s) {
          changed = true;
          ratio[i] = sc / s;
          prod *= s / sc;  // < 0 on a reflected axis: Jp lands on min_Jp, as src/particles.cpp:225-238 does
          en[i] = fmaf(sc, sc, -1.f);
        } else {
          ratio[i] = 1.f;
        }
        if (i == k) {
          sig_k = sc;
          if (sc > 0.f) flip_new = -1;
        }
      }
      float Jp = ps * prod;
      if (!(Jp <= mat.p[6])) Jp = mat.p[6];
      if (!(Jp >= mat.p[5])) Jp = mat.p[5];
      ps = Jp;
      const float hgain = __expf(mat.p[2] * (1.0f - ps));
      mu *= hgain;
      la *= hgain;
    }
    fixed_corotated_tau(mu, la, en, flip_new, tau);
    tau[0] *= -vol; tau[1] *= -vol; tau[2] *= -vol;
  }
  if (changed && 1.f + e[k] < 1e-2f) F = rebuild_small_axis(U, ratio[0], ratio[1], ratio[2], k, sig_k, Ft);
  else if (changed) F = sym_mul(sym_from_eig(U, ratio), Ft);
  else F = Ft;
  store_sym(sym_from_eig(U, tau), force);
}

// friction_project (src/mpm_fwd.h:25-57) with base velocity 0 (static level set).
__device__ __forceinline__ float3 friction_project0(float3 v, float3 n, float friction) {
  if (friction == -1.0f) return make_float3(0.f, 0.f, 0.f);
  bool slip = friction <= -2.0f;
  if (slip) friction = -friction - 2.0f;
  float nn = n.x * v.x + n.y * v.y + n.z * v.z;
  float3 t = make_float3(v.x - nn * n.x, v.y - nn * n.y, v.z - nn * n.z);
  float tn = sqrtf(t.x * t.x + t.y * t.y + t.z * t.z);
  float scale = fmaxf(tn + fminf(nn, 0.f) * friction, 0.f) / fmaxf(1e-30f, tn);
  float keep = fmaxf(0.f, slip ? 0.f : nn);
  return make_float3(scale * t.x + keep * n.x, scale * t.y + keep * n.y, scale * t.z + keep * n.z);
}

// Quadratic B-spline weights of MLSMPMFastKernel32 (src/transfer.cpp:168-186) for
// rel = x/dx - base in [0.5,1.5): w0 = .5(1.5-r)^2, w1 = .75-(r-1)^2, w2 = .5(r-.5)^2,
// evaluated in the reference's polynomial form.
__device__ __forceinline__ void bspline_weights(float rel, float w[3]) {
  float pf = rel - 0.5f;
  float t0 = pf + 0.5f, t1 = pf - 0.5f, t2 = pf - 1.5f;
  w[0] = fmaf(0.5f, t0 * t0, fmaf(-1.5f, t0, 1.125f));
  w[1] = fmaf(-1.0f, t1 * t1, 0.75f);
  w[2] = fmaf(0.5f, t2 * t2, fmaf(1.5f, t2, 1.125f));
}

}  // namespace mpmb
