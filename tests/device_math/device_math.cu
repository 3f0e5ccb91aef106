// C entry points over the device math header compiled for sm_90a with the product's nvcc flags
// (taichi_mpm_b200.build.NVCC_FLAGS): the same functions as tests/host_math/host_math.cpp, one kernel each, one
// thread per state, so that rsqrt.approx.ftz, __expf, __fdividef and nvcc's FMA contraction are what is checked.
// Host buffers are copied in and out inside each call; each returns a cudaError_t.
#include <cuda_runtime.h>
#include <cstdint>
#include "mpmb_math.cuh"

using namespace mpmb;

namespace {

__device__ Mat3 load9(const float *p) {
  Mat3 m;
#pragma unroll
  for (int i = 0; i < 9; i++) m.m[i] = p[i];
  return m;
}
__device__ void store9(float *p, const Mat3 &m) {
#pragma unroll
  for (int i = 0; i < 9; i++) p[i] = m.m[i];
}

__global__ void k_material_step(int64_t n, Material mat, const float *cdg, float *F, float *ps, const float *vol, float *force) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Mat3 f = load9(F + 9 * i), out;
  float s = ps[i];
  material_step<true>(mat, load9(cdg + 9 * i), f, s, vol[i], out);
  store9(F + 9 * i, f);
  ps[i] = s;
  store9(force + 9 * i, out);
}

__global__ void k_plasticity(int64_t n, Material mat, const float *cdg, float *F, float *ps) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Mat3 f = load9(F + 9 * i);
  float s = ps[i];
  plasticity(mat, load9(cdg + 9 * i), f, s);
  store9(F + 9 * i, f);
  ps[i] = s;
}

__global__ void k_calculate_force(int64_t n, Material mat, const float *F, const float *ps, const float *vol, float *force) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Mat3 out;
  calculate_force(mat, load9(F + 9 * i), ps[i], vol[i], out);
  store9(force + 9 * i, out);
}

// the series path alone (sand): `ok` = 0 where the lane must fall back to the eigen path
__global__ void k_sand_step_series(int64_t n, Material mat, const float *cdg, float *F, float *ps, const float *vol, float *force, int *ok) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Mat3 Ft = mat_mul(load9(cdg + 9 * i), load9(F + 9 * i));
  Mat3 f, out;
  float s = ps[i];
#pragma unroll
  for (int k = 0; k < 9; k++) out.m[k] = 0.f;
  ok[i] = sand_step_series(mat, Ft, f, s, vol[i], out) ? 1 : 0;
  store9(F + 9 * i, f);
  ps[i] = s;
  store9(force + 9 * i, out);
}

__global__ void k_eig_sym3(int64_t n, const float *A6, float *U9, float *e3) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float *a = A6 + 6 * i;
  Mat3 U;
  float e[3];
  eig_sym3<MPMB_EIG_SWEEPS>(Sym3{a[0], a[1], a[2], a[3], a[4], a[5]}, U, e);
  store9(U9 + 9 * i, U);
  e3[3 * i] = e[0]; e3[3 * i + 1] = e[1]; e3[3 * i + 2] = e[2];
}

// device copies of host arrays; copies back the ones marked `out` at the end
struct Buffers {
  static const int kMax = 8;
  void *dev[kMax] = {};
  void *host[kMax] = {};
  size_t bytes[kMax] = {};
  bool out[kMax] = {};
  int count = 0;
  cudaError_t err = cudaSuccess;
  template <class T> T *add(const T *h, int64_t elems, bool is_out) {
    const int k = count++;
    host[k] = (void *)h;
    bytes[k] = (size_t)elems * sizeof(T);
    out[k] = is_out;
    if (err == cudaSuccess) err = cudaMalloc(&dev[k], bytes[k] ? bytes[k] : 1);
    if (err == cudaSuccess && bytes[k]) err = cudaMemcpy(dev[k], h, bytes[k], cudaMemcpyHostToDevice);
    return (T *)dev[k];
  }
  cudaError_t finish() {
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err == cudaSuccess) err = cudaDeviceSynchronize();
    for (int k = 0; k < count; k++)
      if (err == cudaSuccess && out[k] && bytes[k]) err = cudaMemcpy(host[k], dev[k], bytes[k], cudaMemcpyDeviceToHost);
    for (int k = 0; k < count; k++) cudaFree(dev[k]);
    return err;
  }
};

Material make_mat(int kind, const float *params8) {
  Material m;
  m.kind = kind;
  for (int i = 0; i < 8; i++) m.p[i] = params8[i];
  return m;
}

unsigned blocks(int64_t n) { return (unsigned)((n + 127) / 128); }

}  // namespace

extern "C" {

int dm_material_step(int64_t n, int kind, const float *params8, const float *cdg, float *F, float *ps, const float *vol, float *force) {
  Buffers b;
  const float *dc = b.add(cdg, 9 * n, false);
  float *dF = b.add(F, 9 * n, true), *dps = b.add(ps, n, true);
  const float *dv = b.add(vol, n, false);
  float *df = b.add(force, 9 * n, true);
  if (b.err == cudaSuccess && n) k_material_step<<<blocks(n), 128>>>(n, make_mat(kind, params8), dc, dF, dps, dv, df);
  return (int)b.finish();
}

int dm_plasticity(int64_t n, int kind, const float *params8, const float *cdg, float *F, float *ps) {
  Buffers b;
  const float *dc = b.add(cdg, 9 * n, false);
  float *dF = b.add(F, 9 * n, true), *dps = b.add(ps, n, true);
  if (b.err == cudaSuccess && n) k_plasticity<<<blocks(n), 128>>>(n, make_mat(kind, params8), dc, dF, dps);
  return (int)b.finish();
}

int dm_calculate_force(int64_t n, int kind, const float *params8, const float *F, const float *ps, const float *vol, float *force) {
  Buffers b;
  const float *dF = b.add(F, 9 * n, false), *dps = b.add(ps, n, false), *dv = b.add(vol, n, false);
  float *df = b.add(force, 9 * n, true);
  if (b.err == cudaSuccess && n) k_calculate_force<<<blocks(n), 128>>>(n, make_mat(kind, params8), dF, dps, dv, df);
  return (int)b.finish();
}

int dm_sand_step_series(int64_t n, const float *params8, const float *cdg, float *F, float *ps, const float *vol, float *force, int *ok) {
  Buffers b;
  const float *dc = b.add(cdg, 9 * n, false);
  float *dF = b.add(F, 9 * n, true), *dps = b.add(ps, n, true);
  const float *dv = b.add(vol, n, false);
  float *df = b.add(force, 9 * n, true);
  int *dok = b.add(ok, n, true);
  if (b.err == cudaSuccess && n) k_sand_step_series<<<blocks(n), 128>>>(n, make_mat(MAT_SAND, params8), dc, dF, dps, dv, df, dok);
  return (int)b.finish();
}

int dm_eig_sym3(int64_t n, const float *A6, float *U9, float *e3) {
  Buffers b;
  const float *dA = b.add(A6, 6 * n, false);
  float *dU = b.add(U9, 9 * n, true), *de = b.add(e3, 3 * n, true);
  if (b.err == cudaSuccess && n) k_eig_sym3<<<blocks(n), 128>>>(n, dA, dU, de);
  return (int)b.finish();
}

}  // extern "C"
