// Device math of the 2-D substep (MPM<2>, sm_90a): the eight constitutive models of src/particles.cpp with dim = 2.
//
// Every isotropic update is evaluated from the closed-form eigen-system of the 2x2 symmetric E = F F^T - I, built from
// G = F - I as E = G + G^T + G G^T (no cancellation at small strain).  With F = U S V^T, E = U (S^2 - I) U^T, so
//   * the Hencky stress  -vol P F^T = -vol U diag(tau_i) U^T      tau_i = 2 mu ln s_i + lambda sum ln s
//   * every return map   U S' V^T  = U diag(s'_i / s_i) U^T F
// need e_i = s_i^2 - 1 and the unit vector (cos 2phi, sin 2phi) of U only: no angle, no iteration, and
// ln s_i = 0.5 log1p(e_i) keeps full relative precision.  det F < 0 gives the smaller singular value a negative sign
// (the rotation-variant convention of the oracle's svd); the Hencky logarithm of it is then NaN, as the reference's is.
// Matrices are column-major 2x2: m[c*2+r].
#pragma once
#include "mpmb_math.cuh"

namespace mpmb {

struct Mat2 {  // column-major: m = (a00, a10, a01, a11)
  float m[4];
};

__device__ __forceinline__ Mat2 mat2_mul(const Mat2 &A, const Mat2 &B) {
  Mat2 C;
  C.m[0] = A.m[0] * B.m[0] + A.m[2] * B.m[1];
  C.m[1] = A.m[1] * B.m[0] + A.m[3] * B.m[1];
  C.m[2] = A.m[0] * B.m[2] + A.m[2] * B.m[3];
  C.m[3] = A.m[1] * B.m[2] + A.m[3] * B.m[3];
  return C;
}
__device__ __forceinline__ Mat2 mat2_mul_t(const Mat2 &A, const Mat2 &B) {  // A B^T
  Mat2 C;
  C.m[0] = A.m[0] * B.m[0] + A.m[2] * B.m[2];
  C.m[1] = A.m[1] * B.m[0] + A.m[3] * B.m[2];
  C.m[2] = A.m[0] * B.m[1] + A.m[2] * B.m[3];
  C.m[3] = A.m[1] * B.m[1] + A.m[3] * B.m[3];
  return C;
}
// det F - 1 from G = F - I
__device__ __forceinline__ float det2_m1(const Mat2 &F) {
  const float g0 = F.m[0] - 1.f, g3 = F.m[3] - 1.f;
  return g0 + g3 + (g0 * g3 - F.m[1] * F.m[2]);
}

// e_1 >= e_2: eigenvalues of E = F F^T - I; (c, s) = (cos 2phi, sin 2phi) of its first eigenvector; sgn2 = -1 when det F < 0
struct Eig2 {
  float e1, e2, c, s, sgn2;
};
__device__ __forceinline__ Eig2 eig_strain2(const Mat2 &F) {
  const float g00 = F.m[0] - 1.f, g10 = F.m[1], g01 = F.m[2], g11 = F.m[3] - 1.f;
  const float a = 2.f * g00 + (g00 * g00 + g01 * g01);
  const float d = 2.f * g11 + (g10 * g10 + g11 * g11);
  const float b = (g01 + g10) + (g00 * g10 + g01 * g11);
  const float m = 0.5f * (a + d), h = 0.5f * (a - d);
  const float r = sqrtf(h * h + b * b);
  Eig2 E;
  const float det = a * d - b * b;  // e1 e2
  if (m >= 0.f) {
    E.e1 = m + r;
    E.e2 = E.e1 != 0.f ? det / E.e1 : 0.f;
  } else {
    E.e2 = m - r;
    E.e1 = det / E.e2;
  }
  if (r > 0.f) {
    E.c = h / r;
    E.s = b / r;
  } else {
    E.c = 1.f;
    E.s = 0.f;
  }
  E.sgn2 = det2_m1(F) < -1.f ? -1.f : 1.f;
  return E;
}
// U diag(f1, f2) U^T
__device__ __forceinline__ Mat2 eig_sym2(const Eig2 &E, float f1, float f2) {
  const float p = 0.5f * (f1 + f2), q = 0.5f * (f1 - f2);
  Mat2 M;
  M.m[0] = p + q * E.c;
  M.m[1] = q * E.s;
  M.m[2] = q * E.s;
  M.m[3] = p - q * E.c;
  return M;
}
__device__ __forceinline__ void singular2(const Eig2 &E, float s[2]) {
  s[0] = sqrtf(1.f + E.e1);
  s[1] = E.sgn2 * sqrtf(1.f + E.e2);
}
__device__ __forceinline__ void log_singular2(const Eig2 &E, float l[2]) {
  l[0] = 0.5f * log1pf(E.e1);
  l[1] = E.sgn2 > 0.f ? 0.5f * log1pf(E.e2) : __int_as_float(0x7fc00000);
}

// (F - R) F^T with R the rotation of the polar decomposition, formed from G = F - I: R - I = [[c-1, -s], [s, c-1]] and
// c - 1 = -s_raw^2 / (n (c_raw + n))
__device__ __forceinline__ Mat2 f_minus_r_ft(const Mat2 &F) {
  const float craw = 2.f + (F.m[0] - 1.f) + (F.m[3] - 1.f), sraw = F.m[1] - F.m[2];
  const float n = sqrtf(craw * craw + sraw * sraw), inv = 1.f / n;
  const float cm1 = -(sraw * sraw) / (n * (craw + n)), s = sraw * inv;
  Mat2 D;
  D.m[0] = (F.m[0] - 1.f) - cm1;
  D.m[1] = F.m[1] - s;
  D.m[2] = F.m[2] + s;
  D.m[3] = (F.m[3] - 1.f) - cm1;
  return mat2_mul_t(D, F);
}
// first Piola-Kirchhoff of fixed corotated: 2 mu (F - R) + lambda (J - 1) J F^-T
__device__ __forceinline__ Mat2 piola_fixed_corotated2(const Mat2 &F, float mu, float la) {
  const float craw = F.m[0] + F.m[3], sraw = F.m[1] - F.m[2];
  const float inv = 1.f / sqrtf(craw * craw + sraw * sraw), c = craw * inv, s = sraw * inv;
  const float k = la * det2_m1(F);  // (J - 1) J F^-T = (J - 1) cof(F)
  Mat2 P;
  P.m[0] = 2.f * mu * (F.m[0] - c) + k * F.m[3];
  P.m[1] = 2.f * mu * (F.m[1] - s) - k * F.m[2];
  P.m[2] = 2.f * mu * (F.m[2] + s) - k * F.m[1];
  P.m[3] = 2.f * mu * (F.m[3] - c) + k * F.m[0];
  return P;
}

// calculate_force(): -vol P(F) F^T (src/particles.cpp:69-82,207-218,329-337,391-411,463-467,628-637,703-712,800-809)
__device__ __forceinline__ Mat2 calculate_force2(const Material &mat, const Mat2 &F, float ps, float vol) {
  const float *p = mat.p;
  Mat2 out;
  switch (mat.kind) {
    case MAT_LINEAR: {  // mu (F + F^T - 2 I) + lambda (tr F - dim) I
      const float mu = p[0], la = p[1];
      const float tr = (F.m[0] - 1.f) + (F.m[3] - 1.f);
      Mat2 P;
      P.m[0] = mu * 2.f * (F.m[0] - 1.f) + la * tr;
      P.m[1] = mu * (F.m[1] + F.m[2]);
      P.m[2] = P.m[1];
      P.m[3] = mu * 2.f * (F.m[3] - 1.f) + la * tr;
      out = mat2_mul_t(P, F);
      for (int k = 0; k < 4; k++) out.m[k] *= -vol;
      return out;
    }
    case MAT_WATER: {  // -vol j (-p I), p = k (j^-gamma - 1)
      const float pr = p[0] * (powf(ps, -p[1]) - 1.f);
      const float d = vol * ps * pr;
      out.m[0] = d; out.m[1] = 0.f; out.m[2] = 0.f; out.m[3] = d;
      return out;
    }
    case MAT_SAND:
    case MAT_ELASTIC:
    case MAT_VON_MISES: {
      const Eig2 E = eig_strain2(F);
      float l[2];
      log_singular2(E, l);
      const float tr = l[0] + l[1];
      const float t1 = 2.f * p[0] * l[0] + p[1] * tr, t2 = 2.f * p[0] * l[1] + p[1] * tr;
      return eig_sym2(E, -vol * t1, -vol * t2);
    }
    default: {  // JELLY, SNOW (Lame parameters scaled by exp(h (1 - Jp))), VISCO (mu_0, lambda_0): fixed corotated
      float mu = p[0], la = p[1];
      if (mat.kind == MAT_SNOW) {
        const float e = expf(p[2] * (1.f - ps));
        mu *= e;
        la *= e;
      }
      const Mat2 D = f_minus_r_ft(F);
      const float jm1 = det2_m1(F), jj = la * jm1 * (1.f + jm1);
      out.m[0] = -vol * (2.f * mu * D.m[0] + jj);
      out.m[1] = -vol * (2.f * mu * D.m[1]);
      out.m[2] = -vol * (2.f * mu * D.m[2]);
      out.m[3] = -vol * (2.f * mu * D.m[3] + jj);
      return out;
    }
  }
}

// SandParticle::project (src/particles.cpp:599-626) with d = dim = 2: the new singular values
__device__ __forceinline__ void sand_project2(const float *p, const float s[2], float &logJp, float out[2]) {
  const float mu0 = p[0], la0 = p[1], alpha = p[2], cohesion = p[3], beta = p[4];
  float eps[2];
  for (int i = 0; i < 2; i++) eps[i] = logf(fmaxf(fabsf(s[i]), 1e-4f)) - cohesion;
  const float eps_sum = eps[0] + eps[1];
  const float tr = eps_sum + logJp;
  const float h0 = eps[0] - tr / 2.f, h1 = eps[1] - tr / 2.f;
  const float hn = sqrtf(h0 * h0 + h1 * h1);
  if (tr >= 0.f) {
    out[0] = out[1] = expf(cohesion);
    logJp = beta * eps_sum + logJp;
  } else {
    logJp = 0.f;
    const float dg = hn + (2.f * la0 + 2.f * mu0) / (2.f * mu0) * tr * alpha;
    if (dg <= 0.f) {
      out[0] = expf(eps[0] + cohesion);
      out[1] = expf(eps[1] + cohesion);
    } else {
      out[0] = expf(eps[0] - dg / hn * h0 + cohesion);
      out[1] = expf(eps[1] - dg / hn * h1 + cohesion);
    }
  }
}

// ViscoParticle::plasticity (src/particles.cpp:89-137) with dim = 2
__device__ __forceinline__ void visco_plasticity2(const Material &mat, const Mat2 &cdg, Mat2 &F, float &ps) {
  const float mu0 = mat.p[0], la0 = mat.p[1], nu = mat.p[2], kappa = mat.p[3], dt = mat.p[4];
  Mat2 m;
  m.m[0] = (cdg.m[0] - 1.f) * (1.f / dt);
  m.m[1] = cdg.m[1] * (1.f / dt);
  m.m[2] = cdg.m[2] * (1.f / dt);
  m.m[3] = (cdg.m[3] - 1.f) * (1.f / dt);
  // approximate_exponent: r = (s/2 + I) s + I, s = m dt; while det r <= 0 the step is halved and the result squared
  Mat2 r;
  int depth = 0;
  float h = dt;
  for (;; depth++, h *= 0.5f) {
    Mat2 s, hs;
    for (int k = 0; k < 4; k++) { s.m[k] = m.m[k] * h; hs.m[k] = s.m[k] * 0.5f; }
    hs.m[0] += 1.f;
    hs.m[3] += 1.f;
    r = mat2_mul(hs, s);
    r.m[0] += 1.f;
    r.m[3] += 1.f;
    if (r.m[0] * r.m[3] - r.m[1] * r.m[2] > 0.f || depth >= 16) break;
  }
  for (int k = 0; k < depth; k++) r = mat2_mul(r, r);
  const Mat2 Fh = mat2_mul(r, F);
  const Eig2 E = eig_strain2(Fh);
  float sg[2];
  singular2(E, sg);
  const Mat2 P = piola_fixed_corotated2(F, mu0, la0);  // of the old dg_e
  const float pnorm = sqrtf(P.m[0] * P.m[0] + P.m[1] * P.m[1] + P.m[2] * P.m[2] + P.m[3] * P.m[3]);
  float gamma = 0.f;
  if (pnorm > 1e-5f) gamma = fminf(fmaxf(dt * nu * (pnorm - ps) / pnorm, 0.f), 1.f);
  const float det = sg[0] * sg[1];
  float scale = 1.f;
  if (fabsf(det) > 1e-5f) scale = 1.f / powf(det, 1.f / 2.f);
  float ratio[2];
  for (int d = 0; d < 2; d++) {
    const float mid = powf(sg[d] * scale, gamma);
    const float mid_inv = fabsf(mid) > 1e-5f ? 1.f / mid : 1.f;
    const float sn = fminf(fmaxf(sg[d] * mid_inv, 0.1f), 10.f);
    ratio[d] = sn / sg[d];
  }
  F = mat2_mul(eig_sym2(E, ratio[0], ratio[1]), Fh);
  ps += kappa * gamma * pnorm;
}

// plasticity(cdg): F <- cdg F and the return map of the type (src/particles.cpp:104-137,222-242,340-343,412-415,469-478,
// 639-647,714-734,811-814)
__device__ __forceinline__ void plasticity2(const Material &mat, const Mat2 &cdg, Mat2 &F, float &ps) {
  if (mat.kind == MAT_WATER) {
    ps *= (cdg.m[0] + cdg.m[3]) - 1.f;
    if (ps < 0.1f) ps = 0.1f;
    return;
  }
  if (mat.kind == MAT_VISCO) {
    visco_plasticity2(mat, cdg, F, ps);
    return;
  }
  const Mat2 Fn = mat2_mul(cdg, F);
  if (mat.kind == MAT_LINEAR || mat.kind == MAT_JELLY || mat.kind == MAT_ELASTIC) {
    F = Fn;
    return;
  }
  const Eig2 E = eig_strain2(Fn);
  float s[2], sn[2];
  singular2(E, s);
  if (mat.kind == MAT_VON_MISES) {
    float l[2];
    log_singular2(E, l);
    const float tr = l[0] + l[1];
    const float h0 = l[0] - tr / 2.f, h1 = l[1] - tr / 2.f;
    const float n2 = h0 * h0 + h1 * h1;  // frobenius_norm2 (src/particles.cpp:724)
    const float dg = n2 - mat.p[2] / (2.f * mat.p[0]);
    if (dg <= 0.f) {
      F = Fn;
      return;
    }
    sn[0] = expf(l[0] - (dg / n2) * h0);
    sn[1] = expf(l[1] - (dg / n2) * h1);
  } else if (mat.kind == MAT_SNOW) {
    float det_orig = 1.f, det_new = 1.f;
    for (int i = 0; i < 2; i++) {
      det_orig *= s[i];
      sn[i] = fminf(fmaxf(s[i], 1.f - mat.p[3]), 1.f + mat.p[4]);
      det_new *= sn[i];
    }
    float jp = ps * det_orig / det_new;
    if (!(jp <= mat.p[6])) jp = mat.p[6];
    if (!(jp >= mat.p[5])) jp = mat.p[5];
    ps = jp;
  } else {  // MAT_SAND
    sand_project2(mat.p, s, ps, sn);
  }
  F = mat2_mul(eig_sym2(E, sn[0] / s[0], sn[1] / s[1]), Fn);
}

// friction_project (src/mpm_fwd.h:25-57), base velocity 0 (static level set)
__device__ __forceinline__ float2 friction_project2(float2 v, float2 n, float friction) {
  if (friction == -1.0f) return make_float2(0.f, 0.f);
  const bool slip = friction <= -2.0f;
  if (slip) friction = -friction - 2.0f;
  const float nn = n.x * v.x + n.y * v.y;
  const float tx = v.x - nn * n.x, ty = v.y - nn * n.y;
  const float tn = sqrtf(tx * tx + ty * ty);
  const float scale = fmaxf(tn + fminf(nn, 0.f) * friction, 0.f) / fmaxf(1e-30f, tn);
  const float keep = fmaxf(0.f, slip ? 0.f : nn);
  return make_float2(scale * tx + keep * n.x, scale * ty + keep * n.y);
}

// MPMKernel<2,2>::calculate_kernel (src/kernel.h:122-134) on one axis: X in grid units, stencil start int(X - 0.5)
// (src/transfer.cpp:188-190); f = fract(X - 0.5), t = f - (-0.5, 0.5, 1.5)
__device__ __forceinline__ void quadratic_weights2(float X, int &base, float w[3]) {
  const float s = __fsub_rn(X, 0.5f);
  base = (int)s;
  const float f = __fsub_rn(s, floorf(s));
  const float t0 = f + 0.5f, t1 = f - 0.5f, t2 = f - 1.5f;
  w[0] = 0.5f * (t0 * t0) + -1.5f * t0 + 1.125f;
  w[1] = -1.0f * (t1 * t1) + 0.75f;
  w[2] = 0.5f * (t2 * t2) + 1.5f * t2 + 1.125f;
}

}  // namespace mpmb
