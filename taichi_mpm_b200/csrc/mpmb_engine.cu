// libmpmb.so — H100-native MLS-MPM substep engine (sm_90a).  C-ABI in include/mpmb.h.
//
// Data layout in HBM (DESIGN.md §3):
//   * particles: SoA of ten float4 streams (160 B/particle), double buffered.
//       P2G set  q0=(x,y,z,mass) q1=(vx,vy,vz,A0) q2=(A1..A4) q3=(A5..A8)
//       G2P set  q4=(F0..F3) q5=(F4..F7) q6=(F8,scalar,vol,tag)     tag = group<<28 | id
//       state    q7=(b0..b3) q8=(b4..b7) q9=(b8,-,-,-)             b = apic_b
//     A = calculate_force()*(-4 dt/dx) + apic_b*(4 m) is the affine matrix rasterize needs
//     (src/transfer.cpp:503,521-522).  G2P produces it for the NEXT substep from the same
//     constitutive evaluation as the return map, so P2G reads 64 B/particle and does no
//     constitutive math, and each particle is factorised at most once per substep.
//   * order: every active tile (4x4x4 nodes) owns a contiguous RUN of storage rows plus a short
//     ARRIVAL list.  G2P writes each tile's particles (cell-sorted) into one contiguous run of the
//     other buffer, so storage is re-compacted every substep for free; a particle whose base node
//     left its tile (~0.5 % per substep) is appended to a mover list and re-binned by four tiny
//     kernels (count, scan, place, rank).  There is NO per-substep radix sort and no permutation
//     array: run rows are read with unit stride.  The radix sort runs once, at upload.
//     This replaces sort_particles_and_populate_grid (src/mpm.cpp:770-918).
//   * grid: no dense grid.  P2G leaves one 6x6x6 float4 "arena" (tile + the +2 stencil halo,
//     the reference's GridCache footprint src/transfer.cpp:59-63) per active tile; G2P rebuilds
//     each node as the fixed-order sum of the <=8 arenas covering it, normalises and applies the
//     level-set boundary.  No global float atomics, no float atomics at all: single-GPU results
//     are bit-reproducible run to run.
#include <cuda_runtime.h>
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mpmb.h"
#include "mpmb_math.cuh"
#include "mpmb_math2d.cuh"

namespace mpmb {

constexpr int ARENA = 216;  // 6*6*6 nodes
constexpr int N_Q = 10;
// tag = group << TAG_ID_BITS | id: MPMB_MAX_GROUPS = 16 groups, ids below 2^28 = 268 M (BASELINE config 5 holds 64 M)
constexpr int TAG_ID_BITS = 28;
constexpr uint32_t TAG_ID_MASK = (1u << TAG_ID_BITS) - 1u;
static_assert(MPMB_MAX_GROUPS <= (1 << (32 - TAG_ID_BITS)), "group bits");
// keys: [0, ntiles_total) = tile index; ntiles_total + {0,1,2} = left through -z / +z face, dead
enum { SPECIAL_MIG_DOWN = 0, SPECIAL_MIG_UP = 1, SPECIAL_DEAD = 2 };

struct Params {
  int res[3];
  int nnode[3];
  // DENSE tile grid of this engine.  world == 1: the whole domain.  z-slab rank: its own tile layers plus one ghost
  // layer on each side, i.e. local layer l holds global layer l + tz_off — the ordering scans, the slot map and the
  // keys are slab-local, so their cost does not grow with the number of ranks.
  int nt[3];
  int tz_off;
  int ntiles_total;
  float dx, inv_dx, dt;
  float gdt[3];
  int particle_gravity, clean_boundary;
  float friction;
  int has_sdf;
  int world, tile_z0, tile_z1;
  Material mats[MPMB_MAX_GROUPS];
};

struct Counters {  // device-resident
  int n_store;        // rows of the current storage that hold a particle record
  int n_tiles;        // active tiles of this substep
  int n_ghost;        // ghost tiles appended after the owned ones (world>1)
  int error;          // sticky device-side error flags
  int n_movers;       // mover list consumed by the next ordering
  int n_movers_next;  // mover list being filled by G2P / migrate_unpack
  int n_alive;        // particles binned by the last ordering
  int n_live;         // scratch of k_count_live (mpmb_num_particles)
  unsigned long long updates;  // sum over substeps of the particles binned: the reference's update_counter (src/mpm.cpp:436)
  int g2p_done;       // CTAs of the running k_g2p that have finished (the last one commits the substep)
  // tiles handed out beyond the first gridDim.x by the substep's k_p2g [0] / k_g2p [1] launch of each part (tile_in_part):
  // each launch has its own counter, zeroed by the ordering that precedes the launches
  int claim[2][3];
  int xstep;          // substeps completed since the peers were connected: the sequence number of the peer exchange
                      // (kept on the device so that a captured CUDA graph of a substep stays valid from replay to replay)
  int chk[8];         // MPMB_CHECKED builds: first violated index check {site, a, b, c, ...}
};
// Bounds-checked debug build (-DMPMB_CHECKED): an index that would leave its array is recorded (first one wins) and the
// access skipped, so a corrupted ordering shows up as a report (mpmb_debug_check) instead of an illegal-address fault.
#ifdef MPMB_CHECKED
#define MPMB_CHK(cnt, cond, site, a, b, c)                                                                        \
  ((cond) ? true : (atomicCAS(&(cnt)->chk[0], 0, (site)) == 0 ? ((cnt)->chk[1] = (int)(a), (cnt)->chk[2] = (int)(b), (cnt)->chk[3] = (int)(c), false) : false))
#else
#define MPMB_CHK(cnt, cond, site, a, b, c) true
#endif
enum { DEVERR_TILE_CAPACITY = 1, DEVERR_MIGRATE_CAPACITY = 2, DEVERR_PARTICLE_CAPACITY = 4, DEVERR_PEER_TIMEOUT = 8, DEVERR_BAD_INPUT = 16,
       DEVERR_BAD_SLOT = 32 };   // BAD_SLOT: a 2-D AoS call met an id or slot index outside its vectors (Counters2::aos_error)

// Tile-scheduling trace (-DMPMB_TILE_TRACE, read by bench_tail.py through mpmb_debug_tile_trace): every CTA of k_p2g
// and k_g2p records when it started and ended (%globaltimer, ns), its SM and the tiles and particle rows it
// processed.  Each kernel keeps the records of its last launch.
#ifdef MPMB_TILE_TRACE
struct CtaTrace { unsigned long long t0, t1; int sm, tiles, rows, pad; };
enum { TRACE_P2G = 0, TRACE_G2P = 1, TRACE_CTAS = 4096 };
__device__ CtaTrace g_trace[2][TRACE_CTAS];
#ifndef MPMB_SIMT_HOST
__device__ __forceinline__ unsigned long long trace_clock() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ int trace_smid() {
  int s;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}
#else
__device__ __forceinline__ unsigned long long trace_clock() { return 0; }
__device__ __forceinline__ int trace_smid() { return 0; }
#endif
#define MPMB_TRACE_BEGIN const unsigned long long trace_t0 = trace_clock(); int trace_tiles = 0, trace_rows = 0
#define MPMB_TRACE_TILE(rows) (trace_tiles++, trace_rows += (rows))
#define MPMB_TRACE_END(k) \
  if (threadIdx.x == 0 && blockIdx.x < TRACE_CTAS) g_trace[k][blockIdx.x] = CtaTrace{trace_t0, trace_clock(), trace_smid(), trace_tiles, trace_rows, 0}
#else
#define MPMB_TRACE_BEGIN
#define MPMB_TRACE_TILE(rows)
#define MPMB_TRACE_END(k)
#endif

struct TileMeta {  // one 32-byte record per active tile (slot)
  int tile, run_begin, run_len, arr_off, arr_len, out_begin, xy, z;  // xy = tile x | y << 16, z = GLOBAL tile layer
};
// TileMeta::pad0/pad1 carry the tile's (x | y<<16, z) coordinates, decoded once per tile by k_order_c, so the tile
// kernels skip two runtime integer divisions per CTA per tile/chunk.
// Alternatives tried and dropped: a 192-thread x-plane P2G (more instructions and three times the row reads) and per-tile
// level-set flags for the grid update (the band test is not its limiter).

struct View {  // raw pointers handed to kernels
  float4 *q[N_Q];        // current (read) buffer
  float4 *qn[N_Q];       // next (written by G2P)
  uint32_t *keys;        // tile of every current row (specials: dead / migrating)
  uint32_t *keys_next;
  uint32_t *outpos;      // per live current row: its row in the next storage (written by P2G)
  // dense per-tile ordering state
  int *run_begin, *run_len;      // run of the tile in the current storage
  int *out_begin, *total;        // run of the tile in the next storage (= next substep's run)
  int *stay_cnt, *stay_next;     // rows of the run still owned by the tile (now / after this G2P)
  int *arr_cnt, *arr_off, *arr_len, *arr_cur;
  int *slot_map;
  TileMeta *meta;                // [slot]
  uint32_t *mover_dst, *mover_idx;      // consumed by the ordering
  uint32_t *mover_dst_n, *mover_idx_n;  // produced by G2P
  uint32_t *arrivals, *arrivals_sorted;
  int *blocksum;
  float4 *arena;
  const float4 *sdf4;
  Counters *cnt;
  int cap_tiles;
  int cap_particles;
  const unsigned char *rigid_flag;  // [slot] 1 = the tile lies in a rigid page: k_g2p leaves it to k_g2p_rigid (null: no rigid bodies)
};

// ------------------------------------------------------------------------------ helpers
// Asynchronous 16-byte global->shared copies (LDGSTS): the gathered particle rows of a tile are
// put in flight in one batch, no register staging, and waited for once.
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src) {
  unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// TMA bulk copies (cp.async.bulk, SASS UBLKCP) completing on an mbarrier: ONE elected thread moves a whole unit-stride
// run chunk (4 KB per stream) or a tile's 3.4 KB node block global -> shared; nobody computes addresses per row, and the
// consumers wait on the barrier's phase parity instead of on their own copy groups.
#ifndef MPMB_SIMT_HOST
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// the elected thread's arrival + the number of bytes the copies of this phase will deliver
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, unsigned bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
#else
// SIMT emulator (tests/simt): a phase completes at the elected thread's arrival (the word counts completed phases and a
// waiter yields to the other coroutines until the phase of its parity is over), but the bulk copies LAND LATE — they are
// queued and performed by the first thread that waits on their barrier — so a consumer that reads without waiting, or
// another copy that races with a bulk copy's bytes, shows up in the emulated parity runs.
struct SimtBulk { void *dst; const void *src; unsigned bytes; uint64_t *bar; };
static std::vector<SimtBulk> g_simt_bulk;
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned) { *bar = 0; }
__device__ __forceinline__ void mbar_init_fence() {}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, unsigned) { *bar += 1; }
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, unsigned bytes, uint64_t *bar) {
  g_simt_bulk.push_back(SimtBulk{smem_dst, gmem_src, bytes, bar});
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
  while ((unsigned)(*(volatile uint64_t *)bar & 1u) == parity) simt::yield();
  for (size_t i = 0; i < g_simt_bulk.size();) {
    if (g_simt_bulk[i].bar == bar) {
      memcpy(g_simt_bulk[i].dst, g_simt_bulk[i].src, g_simt_bulk[i].bytes);
      g_simt_bulk.erase(g_simt_bulk.begin() + i);
    } else {
      i++;
    }
  }
}
#endif

// A float4 quantity (x, y | z, w) and its weights as pairs.  The operations are the scalar fmaf / mul / sub (sm_90 has
// no packed fp32 arithmetic); the node loops keep the pair structure, which the scalar code generator schedules better
// than float[27][4] accumulators.
struct F4 {
  float2 lo, hi;  // (x, y), (z, w)
};
__device__ __forceinline__ float2 bc2(float w) { return make_float2(w, w); }
__device__ __forceinline__ F4 f4_load(const float4 &v) { return F4{make_float2(v.x, v.y), make_float2(v.z, v.w)}; }
__device__ __forceinline__ F4 f4_zero() { return F4{make_float2(0.f, 0.f), make_float2(0.f, 0.f)}; }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ F4 f4_fma(float2 w, const F4 &a, const F4 &c) {
  return F4{make_float2(fmaf(w.x, a.lo.x, c.lo.x), fmaf(w.y, a.lo.y, c.lo.y)), make_float2(fmaf(w.x, a.hi.x, c.hi.x), fmaf(w.y, a.hi.y, c.hi.y))};
}
__device__ __forceinline__ F4 f4_mul(float2 w, const F4 &a) { return F4{make_float2(w.x * a.lo.x, w.y * a.lo.y), make_float2(w.x * a.hi.x, w.y * a.hi.y)}; }
__device__ __forceinline__ F4 f4_sub(const F4 &a, const F4 &b) {
  return F4{make_float2(a.lo.x - b.lo.x, a.lo.y - b.lo.y), make_float2(a.hi.x - b.hi.x, a.hi.y - b.hi.y)};
}

__device__ __forceinline__ void base_rel(float x, float inv_dx, int &base, float &rel) {
  // pos_ = p.pos * inv_delta_x (src/transfer.cpp:490); base = int(x - 0.5f) (src/kernel.h:119-121).
  // Explicit round-to-nearest ops so that no FMA contraction changes the cell assignment.
  float X = __fmul_rn(x, inv_dx);
  base = (int)__fsub_rn(X, 0.5f);
  rel = __fsub_rn(X, (float)base);
}

__device__ __forceinline__ uint32_t make_key(const Params &P, float x, float y, float z) {
  int bx, by, bz;
  float r;
  base_rel(x, P.inv_dx, bx, r);
  base_rel(y, P.inv_dx, by, r);
  base_rel(z, P.inv_dx, bz, r);
  // the 27-node stencil [base, base+2] must stay on the node grid
  bool in_domain = (bx >= 0) && (by >= 0) && (bz >= 0) && (bx + 2 < P.nnode[0]) && (by + 2 < P.nnode[1]) && (bz + 2 < P.nnode[2]);
  if (!in_domain) return (uint32_t)(P.ntiles_total + SPECIAL_DEAD);
  int tx = bx >> 2, ty = by >> 2, tz = bz >> 2;
  if (P.world > 1) {
    if (tz < P.tile_z0) return (uint32_t)(P.ntiles_total + SPECIAL_MIG_DOWN);
    if (tz >= P.tile_z1) return (uint32_t)(P.ntiles_total + SPECIAL_MIG_UP);
  }
  return (uint32_t)((tx * P.nt[1] + ty) * P.nt[2] + (tz - P.tz_off));
}

// near_boundary + abnormal (src/mpm.h:269-276, src/mpm.cpp:595-598)
__device__ __forceinline__ bool reference_deletes(const Params &P, float3 x, float3 v) {
  float X = x.x * P.inv_dx, Y = x.y * P.inv_dx, Z = x.z * P.inv_dx;
  float mn = fminf(X, fminf(Y, Z));
  float mx = fmaxf(X - (float)P.res[0], fmaxf(Y - (float)P.res[1], Z - (float)P.res[2]));
  bool bad = (mn < 7.0f) || (mx > -7.0f);
  bad |= !isfinite((x.x + x.y + x.z) + (v.x + v.y + v.z));  // any inf/NaN poisons the sum (pos.abnormal() || v.abnormal())
  return bad;
}

// z-slab runs split every tile kernel in two launches so that the halo exchange overlaps compute:
// part 1 = tiles of the slab's boundary layers (they produce / consume halo data), part 2 = the rest,
// part 0 = all tiles.
__device__ __forceinline__ bool tile_in_part(const Params &P, int tile, int part) {
  if (part == 0) return true;
  const int tz = tile % P.nt[2] + P.tz_off;
  const bool boundary = (P.world > 1) && (tz == P.tile_z0 || tz == P.tile_z1 - 1);
  return part == 1 ? boundary : !boundary;
}

// affine = stress * (-4 inv_dx dt) + apic_b * (inv_D * mass)  (src/transfer.cpp:465,503,521-522)
__device__ __forceinline__ void make_affine(const Mat3 &force, const Mat3 &b, float mass, float S, Mat3 &A) {
  const float bm = 4.0f * mass;
#pragma unroll
  for (int k = 0; k < 9; k++) A.m[k] = fmaf(force.m[k], S, b.m[k] * bm);
}

template <bool STORE_B = true>
__device__ __forceinline__ void store_particle(float4 *const *q, size_t i, float3 x, float mass, float3 v, const Mat3 &A, const Mat3 &F,
                                               float ps, float vol, uint32_t tag, const Mat3 &b) {
  q[0][i] = make_float4(x.x, x.y, x.z, mass);
  q[1][i] = make_float4(v.x, v.y, v.z, A.m[0]);
  q[2][i] = make_float4(A.m[1], A.m[2], A.m[3], A.m[4]);
  q[3][i] = make_float4(A.m[5], A.m[6], A.m[7], A.m[8]);
  q[4][i] = make_float4(F.m[0], F.m[1], F.m[2], F.m[3]);
  q[5][i] = make_float4(F.m[4], F.m[5], F.m[6], F.m[7]);
  q[6][i] = make_float4(F.m[8], ps, vol, __uint_as_float(tag));
  if (STORE_B) {
    q[7][i] = make_float4(b.m[0], b.m[1], b.m[2], b.m[3]);
    q[8][i] = make_float4(b.m[4], b.m[5], b.m[6], b.m[7]);
    q[9][i] = make_float4(b.m[8], 0.f, 0.f, 0.f);
  }
}

// ------------------------------------------------------------------------------ upload kernels
__global__ void k_iota(uint32_t *a, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = (uint32_t)i;
}

// one particle into storage row `row` with id `id` (an upload: row = upload index, id = id_base + upload index; an append:
// the rows after the resident ones and the ids after the ones handed out so far)
__device__ __forceinline__ void pack_one(View &V, const Params &P, int row, uint32_t id, float3 x, float3 v, Mat3 F, Mat3 b, float mass, float vol, float ps,
                                         int g, uint32_t *keys) {
  // a hole is encoded by the sign of the mass and the group by 4 tag bits: reject what cannot be represented
  if (g < 0 || g >= MPMB_MAX_GROUPS || !(mass > 0.f)) {
    atomicOr(&V.cnt->error, DEVERR_BAD_INPUT);
    g = min(max(g, 0), MPMB_MAX_GROUPS - 1);
    mass = 1e-30f;
  }
  Mat3 force, A;
  calculate_force(P.mats[g], F, ps, vol, force);
  make_affine(force, b, mass, -4.0f * P.inv_dx * P.dt, A);
  store_particle(V.q, (size_t)row, x, mass, v, A, F, ps, vol, ((uint32_t)g << TAG_ID_BITS) | id, b);
  keys[row] = make_key(P, x.x, x.y, x.z);
}

// Field-wise host arrays (staged on the device) -> q streams: particle i into row row0 + i with id id0 + i.  With
// `prefix` (the exclusive scan of k_owned_flags over n + 1 entries) only the flagged particles are packed, compacted:
// particle i into row row0 + prefix[i], still with id id0 + i.
__global__ void k_pack_particles(View V, Params P, int n, const float *x, const float *v, const float *F, const float *b,
                                 const float *mass, const float *vol, const float *scalar, const int *group, uint32_t *keys, int row0, uint32_t id0,
                                 const int *prefix) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int row = row0 + i;
  if (prefix) {
    if (prefix[i + 1] == prefix[i]) return;
    row = row0 + prefix[i];
  }
  Mat3 f, bb;
#pragma unroll
  for (int k = 0; k < 9; k++) {
    f.m[k] = F ? F[9 * (size_t)i + k] : ((k % 4 == 0) ? 1.f : 0.f);
    bb.m[k] = b ? b[9 * (size_t)i + k] : 0.f;
  }
  int g = group ? group[i] : 0;
  float ps;
  if (scalar) ps = scalar[i];
  else {
    int kind = P.mats[g].kind;
    ps = (kind == MAT_SNOW || kind == MAT_WATER) ? 1.0f : 0.0f;  // Jp=1 (205), j=1 (461), logJp=0 (595)
  }
  float3 xx = make_float3(x[3 * (size_t)i], x[3 * (size_t)i + 1], x[3 * (size_t)i + 2]);
  float3 vv = make_float3(v[3 * (size_t)i], v[3 * (size_t)i + 1], v[3 * (size_t)i + 2]);
  pack_one(V, P, row, id0 + (uint32_t)i, xx, vv, f, bb, mass[i], vol[i], ps, g, keys);
}

// Ownership of a particle of a batch that every z-slab rank receives: the rank whose own tiles hold the particle's key
// (make_key: the tile layer of its base node lies in [tile_z0, tile_z1)).  An in-domain, finite particle is owned by
// exactly one rank; on world == 1 every in-domain particle is owned.  The rest are not packed at all (an upload packs
// them with the dead key and the ordering drops them: the same live rows in the same order).
__global__ void k_owned_flags(Params P, int n, const float *x, int *flags) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = make_key(P, x[3 * (size_t)i], x[3 * (size_t)i + 1], x[3 * (size_t)i + 2]) < (uint32_t)P.ntiles_total ? 1 : 0;
}

// Per-kind plastic scalars of a mixed AoS pool (MpmbAosLayout.off_scalar_by_kind), resolved per group on the host from the
// group -> kind snapshot of mpmb_upload_aos: the slot offset of the group's scalar (-1: none in the slot) and the value a row
// without one starts with.  on == 0: the single off_scalar of the layout applies.
struct AosScalars {
  int on;
  int32_t off[MPMB_MAX_GROUPS];
  float dflt[MPMB_MAX_GROUPS];
};

// Reference AoS slots (staged on the device) -> q streams.
__global__ void k_pack_aos(View V, Params P, int n, const unsigned char *pool, const uint32_t *indices, MpmbAosLayout L, AosScalars S,
                           const int *group, uint32_t *keys, uint32_t id_base) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned char *s = pool + (size_t)indices[i] * L.stride;
  const float *pos = (const float *)(s + L.off_pos);
  const float *vm = (const float *)(s + L.off_v_and_m);
  Mat3 f, bb;
  for (int c = 0; c < 3; c++) {
    const float *fc = (const float *)(s + L.off_dg_e + c * L.col_pitch);
    const float *bc = (const float *)(s + L.off_apic_b + c * L.col_pitch);
    for (int r = 0; r < 3; r++) {
      f.m[c * 3 + r] = fc[r];
      bb.m[c * 3 + r] = bc[r];
    }
  }
  int g = group ? group[i] : 0;
  float vol = *(const float *)(s + L.off_vol);
  float ps;
  if (S.on) {
    const int gs = min(max(g, 0), MPMB_MAX_GROUPS - 1);   // a group out of range is flagged by pack_one
    ps = S.off[gs] >= 0 ? *(const float *)(s + S.off[gs]) : S.dflt[gs];
  } else {
    ps = L.off_scalar >= 0 ? *(const float *)(s + L.off_scalar) : 0.f;
  }
  pack_one(V, P, i, id_base + (uint32_t)i, make_float3(pos[0], pos[1], pos[2]), make_float3(vm[0], vm[1], vm[2]), f, bb, vm[3], vol, ps, g, keys);
}

// q streams -> field-wise arrays, compacting live particles (storage order).
__global__ void k_unpack_particles(View V, const uint32_t *keys, int n, uint32_t special_min, uint32_t *id, float *x, float *v, float *F,
                                   float *b, float *mass, float *vol, float *scalar, int *group, const int *prefix) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (keys[i] >= special_min) return;
  int o = prefix[i];
  float4 q0 = V.q[0][i], q1 = V.q[1][i], q4 = V.q[4][i], q5 = V.q[5][i], q6 = V.q[6][i], q7 = V.q[7][i], q8 = V.q[8][i], q9 = V.q[9][i];
  uint32_t tag = __float_as_uint(q6.w);
  if (id) id[o] = tag & TAG_ID_MASK;
  if (group) group[o] = (int)(tag >> TAG_ID_BITS);
  if (x) { x[3 * (size_t)o] = q0.x; x[3 * (size_t)o + 1] = q0.y; x[3 * (size_t)o + 2] = q0.z; }
  if (mass) mass[o] = fabsf(q0.w);
  if (v) { v[3 * (size_t)o] = q1.x; v[3 * (size_t)o + 1] = q1.y; v[3 * (size_t)o + 2] = q1.z; }
  if (F) {
    float *f = F + 9 * (size_t)o;
    f[0] = q4.x; f[1] = q4.y; f[2] = q4.z; f[3] = q4.w; f[4] = q5.x; f[5] = q5.y; f[6] = q5.z; f[7] = q5.w; f[8] = q6.x;
  }
  if (scalar) scalar[o] = q6.y;
  if (vol) vol[o] = q6.z;
  if (b) {
    float *p = b + 9 * (size_t)o;
    p[0] = q7.x; p[1] = q7.y; p[2] = q7.z; p[3] = q7.w; p[4] = q8.x; p[5] = q8.y; p[6] = q8.z; p[7] = q8.w; p[8] = q9.x;
  }
}

// live rows of the current storage (keys below the specials), reduced on the device: mpmb_num_particles reads 4 bytes
__global__ void __launch_bounds__(256) k_count_live(const uint32_t *keys, uint32_t special_min, Counters *cnt) {
  typedef cub::BlockReduce<int, 256> Red;
  __shared__ typename Red::TempStorage tmp;
  const int n = cnt->n_store;
  int c = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) c += keys[i] < special_min;
  c = Red(tmp).Sum(c);
  if (threadIdx.x == 0 && c) atomicAdd(&cnt->n_live, c);
}

__global__ void k_alive_flags(const uint32_t *keys, int n, uint32_t special_min, int *flags) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = keys[i] < special_min ? 1 : 0;
}

__global__ void k_fill_u32(uint32_t *a, int n, uint32_t v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}

// LevelSet.sample (mpm.py): phi at X (grid units), trilinear in the node phi (X clamped to [0, nnode - 1 - 1e-9], node
// values capped at 1e20), in double
__device__ __forceinline__ double sdf_phi_trilinear(const float4 *sdf4, const Params &P, const double Xg[3]) {
  int i0[3];
  double f[3];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double X = fmin(fmax(Xg[a], 0.0), (double)(P.nnode[a] - 1) - 1e-9);
    i0[a] = (int)floor(X);
    f[a] = X - (double)i0[a];
  }
  double phi = 0.0;
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int b = 0; b < 2; b++)
#pragma unroll
      for (int c = 0; c < 2; c++) {
        const double w = (a ? f[0] : 1.0 - f[0]) * (b ? f[1] : 1.0 - f[1]) * (c ? f[2] : 1.0 - f[2]);
        const float s = sdf4[((size_t)(i0[0] + a) * P.nnode[1] + (i0[1] + b)) * P.nnode[2] + (i0[2] + c)].w;
        phi += w * (double)fminf(s, 1e20f);
      }
  return phi;
}

// delete_particles_inside_level_set (src/mpm.cpp:959-973): phi at X = x / dx (sdf_phi_trilinear).  A live row with phi < 0
// gets the dead key (the next ordering drops it); the killed rows are counted into cnt->n_live.
__global__ void __launch_bounds__(256) k_delete_inside(View V, Params P, int n, uint32_t special_min, uint32_t key_dead) {
  typedef cub::BlockReduce<int, 256> Red;
  __shared__ typename Red::TempStorage tmp;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int killed = 0;
  if (i < n && V.keys[i] < special_min) {
    const float4 q0 = V.q[0][i];
    const double X[3] = {(double)q0.x / (double)P.dx, (double)q0.y / (double)P.dx, (double)q0.z / (double)P.dx};
    const double phi = sdf_phi_trilinear(V.sdf4, P, X);
    if (phi < 0.0) {
      V.keys[i] = key_dead;
      killed = 1;
    }
  }
  killed = Red(tmp).Sum(killed);
  if (threadIdx.x == 0 && killed) atomicAdd(&V.cnt->n_live, killed);
}

// ------------------------------------------------------------------------------ device-side seeding
// Replaces the `benchmark` lattice of MPM<3>::add_particles (src/mpm.cpp:149-186: 8 particles per cell at the cell
// centre +- 0.25 dx) without a host array: optional jitter from a counter-based hash of the particle's LATTICE index, so
// the same particle gets the same position whatever the z-slab partition (and from the numpy twin
// scenes.lattice_block_hashed, the parity reference).  id = lattice index; a z-slab rank keeps the particles whose base
// node lies in its tile layers; particles in the 7-cell boundary band are not created (src/mpm.cpp:129-132).
struct SeedBox {
  int lo[3], n[3];      // first cell and number of cells of the whole block
  int z_first, z_count; // candidate cell layers of this rank (relative to lo[2])
  float jitter, vol, mass, v0[3];
  float ps;             // plastic scalar of the material's fresh state
  uint32_t seed, id_base;
  int group;
};
__host__ __device__ __forceinline__ uint32_t seed_hash(uint32_t idx, uint32_t axis, uint32_t seed) {
  uint32_t h = (idx * 3u + axis) ^ seed;
  h *= 0x9E3779B1u; h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}
// candidate c -> lattice index, position; returns whether this rank creates the particle
__device__ __forceinline__ bool seed_candidate(const Params &P, const SeedBox &B, size_t c, uint32_t &lattice, float3 &x, uint32_t &key) {
  const int corner = (int)(c & 7u);
  size_t cell = c >> 3;
  const int kz = (int)(cell % (size_t)B.z_count) + B.z_first;
  cell /= (size_t)B.z_count;
  const int ky = (int)(cell % (size_t)B.n[1]), kx = (int)(cell / (size_t)B.n[1]);
  lattice = (uint32_t)((((size_t)kx * B.n[1] + ky) * B.n[2] + kz) * 8u + corner);
  const int ic[3] = {B.lo[0] + kx, B.lo[1] + ky, B.lo[2] + kz};
  float X[3];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const float off = ((corner >> a) & 1) ? 0.75f : 0.25f;
    const float u = __fsub_rn((float)(seed_hash(lattice, (uint32_t)a, B.seed) >> 8) * (1.0f / 8388608.0f), 1.0f);  // [-1, 1)
    X[a] = __fadd_rn(__fadd_rn((float)ic[a], off), __fmul_rn(B.jitter, u));                                        // grid units
  }
  x = make_float3(__fmul_rn(X[0], P.dx), __fmul_rn(X[1], P.dx), __fmul_rn(X[2], P.dx));
  const float mn = fminf(X[0], fminf(X[1], X[2]));
  const float mx = fmaxf(X[0] - (float)P.res[0], fmaxf(X[1] - (float)P.res[1], X[2] - (float)P.res[2]));
  if (mn < 7.0f || mx > -7.0f) return false;  // near_boundary (src/mpm.h:269-276)
  key = make_key(P, x.x, x.y, x.z);
  return key < (uint32_t)P.ntiles_total;      // owned by this rank (not a migration / dead key)
}
__global__ void k_seed_flags(Params P, SeedBox B, size_t n_cand, int *flags) {
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n_cand; c += (size_t)gridDim.x * blockDim.x) {
    uint32_t lattice, key;
    float3 x;
    flags[c] = seed_candidate(P, B, c, lattice, x, key) ? 1 : 0;
  }
}
__global__ void k_seed_write(View V, Params P, SeedBox B, size_t n_cand, const int *flags, const int *prefix, uint32_t *keys) {
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n_cand; c += (size_t)gridDim.x * blockDim.x) {
    if (!flags[c]) continue;
    uint32_t lattice, key;
    float3 x;
    seed_candidate(P, B, c, lattice, x, key);
    Mat3 F, b, force, A;
#pragma unroll
    for (int k = 0; k < 9; k++) { F.m[k] = (k % 4 == 0) ? 1.f : 0.f; b.m[k] = 0.f; }
    calculate_force(P.mats[B.group], F, B.ps, B.vol, force);
    make_affine(force, b, B.mass, -4.0f * P.inv_dx * P.dt, A);
    const size_t o = (size_t)prefix[c];
    store_particle(V.q, o, x, B.mass, make_float3(B.v0[0], B.v0[1], B.v0[2]), A, F, B.ps, B.vol, ((uint32_t)B.group << TAG_ID_BITS) | (B.id_base + lattice), b);
    keys[o] = key;
  }
}

// mpmb_set_material on RESIDENT particles: the cached affine matrix A (q1.w..q3) was computed with the old parameters
// (pack_one at upload, or the last G2P); rebuild it from (F, scalar, vol, apic_b) for the rows of that group so that
// the next rasterize uses the new material's stress (src/transfer.cpp:503,509,521-522).
__global__ void k_refresh_affine(View V, Params P, const uint32_t *keys, int n, uint32_t special_min, int group) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || keys[i] >= special_min) return;
  const float4 q6 = V.q[6][i];
  if ((int)(__float_as_uint(q6.w) >> TAG_ID_BITS) != group) return;
  const float4 q0 = V.q[0][i], q1 = V.q[1][i], q4 = V.q[4][i], q5 = V.q[5][i], q7 = V.q[7][i], q8 = V.q[8][i], q9 = V.q[9][i];
  Mat3 F, b, force, A;
  F.m[0] = q4.x; F.m[1] = q4.y; F.m[2] = q4.z; F.m[3] = q4.w; F.m[4] = q5.x; F.m[5] = q5.y; F.m[6] = q5.z; F.m[7] = q5.w; F.m[8] = q6.x;
  b.m[0] = q7.x; b.m[1] = q7.y; b.m[2] = q7.z; b.m[3] = q7.w; b.m[4] = q8.x; b.m[5] = q8.y; b.m[6] = q8.z; b.m[7] = q8.w; b.m[8] = q9.x;
  calculate_force(P.mats[group], F, q6.y, q6.z, force);
  make_affine(force, b, fabsf(q0.w), -4.0f * P.inv_dx * P.dt, A);
  V.q[1][i] = make_float4(q1.x, q1.y, q1.z, A.m[0]);
  V.q[2][i] = make_float4(A.m[1], A.m[2], A.m[3], A.m[4]);
  V.q[3][i] = make_float4(A.m[5], A.m[6], A.m[7], A.m[8]);
}

// ------------------------------------------------------------------------------ frame dump
// The per-point records of MPM<3>::write_partio -> Partio's BGEO writer (src/visualize.cpp:16-100,
// external/partio/src/io/BGEO.cpp:131-150) packed on the device: big-endian 4-byte words
//   position xyz, w = 1.0f, type = 0 (is_rigid), index = id, limit = (1,1,1), v xyz        (12 words, non-verbose dump)
// in id order, which is the order the reference sorts its particles into before writing (visualize.cpp:39-43).
__device__ __forceinline__ uint32_t be32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }
__global__ void k_id_flags(View V, const uint32_t *keys, int n, uint32_t special_min, uint32_t id_base, int64_t id_range, int *flags, Counters *cnt) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || keys[i] >= special_min) return;
  const uint32_t id = (__float_as_uint(V.q[6][i].w) & TAG_ID_MASK) - id_base;
  if ((int64_t)id >= id_range) { atomicOr(&cnt->error, DEVERR_BAD_INPUT); return; }
  flags[id] = 1;
}
__global__ void k_bgeo_points(View V, const uint32_t *keys, int n, uint32_t special_min, uint32_t id_base, int64_t id_range, const int *prefix, uint32_t *out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || keys[i] >= special_min) return;
  const float4 q0 = V.q[0][i], q1 = V.q[1][i];
  const uint32_t gid = __float_as_uint(V.q[6][i].w) & TAG_ID_MASK, id = gid - id_base;
  if ((int64_t)id >= id_range) return;
  uint4 *rec = reinterpret_cast<uint4 *>(out + (size_t)prefix[id] * 12);
  rec[0] = make_uint4(be32(__float_as_uint(q0.x)), be32(__float_as_uint(q0.y)), be32(__float_as_uint(q0.z)), be32(__float_as_uint(1.0f)));
  rec[1] = make_uint4(0u, be32(gid), be32(1u), be32(1u));
  rec[2] = make_uint4(be32(1u), be32(__float_as_uint(q1.x)), be32(__float_as_uint(q1.y)), be32(__float_as_uint(q1.z)));
}

// ------------------------------------------------------------------------------ AoS write-back
// mpmb_download_aos on the device: every live row goes back into its slot of the (device image of the) reference's
// pool and raises the alive flag of its id; the survivors' slots, in id order, are then one stream compaction away.
__global__ void k_aos_scatter(View V, const uint32_t *keys, int n, uint32_t special_min, unsigned char *pool, const uint32_t *indices,
                              int64_t n_indices, int64_t pool_slots, MpmbAosLayout L, AosScalars S, uint32_t id_base, int *alive_flag,
                              Counters *cnt) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (keys[i] >= special_min) return;
  const float4 q0 = V.q[0][i], q1 = V.q[1][i], q4 = V.q[4][i], q5 = V.q[5][i], q6 = V.q[6][i], q7 = V.q[7][i], q8 = V.q[8][i], q9 = V.q[9][i];
  const uint32_t id = (__float_as_uint(q6.w) & TAG_ID_MASK) - id_base;
  if ((int64_t)id >= n_indices) { atomicOr(&cnt->error, DEVERR_BAD_INPUT); return; }
  const uint32_t slot = indices[id];
  if ((int64_t)slot >= pool_slots) { atomicOr(&cnt->error, DEVERR_BAD_INPUT); return; }
  alive_flag[id] = 1;
  unsigned char *sl = pool + (size_t)slot * L.stride;
  float *pos = (float *)(sl + L.off_pos), *vm = (float *)(sl + L.off_v_and_m);
  pos[0] = q0.x; pos[1] = q0.y; pos[2] = q0.z;
  vm[0] = q1.x; vm[1] = q1.y; vm[2] = q1.z; vm[3] = fabsf(q0.w);
  const float Fm[9] = {q4.x, q4.y, q4.z, q4.w, q5.x, q5.y, q5.z, q5.w, q6.x}, bm[9] = {q7.x, q7.y, q7.z, q7.w, q8.x, q8.y, q8.z, q8.w, q9.x};
#pragma unroll
  for (int c = 0; c < 3; c++) {
    float *fc = (float *)(sl + L.off_dg_e + c * L.col_pitch), *bc = (float *)(sl + L.off_apic_b + c * L.col_pitch);
#pragma unroll
    for (int r = 0; r < 3; r++) { fc[r] = Fm[c * 3 + r]; bc[r] = bm[c * 3 + r]; }
  }
  if (S.on) {
    const int32_t off = S.off[__float_as_uint(q6.w) >> TAG_ID_BITS];
    if (off >= 0) *(float *)(sl + off) = q6.y;
  } else if (L.off_scalar >= 0) {
    *(float *)(sl + L.off_scalar) = q6.y;
  }
}
__global__ void k_compact_survivors(const uint32_t *indices, const int *alive_flag, const int *prefix, int64_t n, uint32_t *out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n && alive_flag[i]) out[prefix[i]] = indices[i];
}

// ------------------------------------------------------------------------------ ordering
// Replaces sort_particles_and_populate_grid (src/mpm.cpp:770-918) incrementally.
//   (arr_cnt[dst]++ for every mover is done where the mover is appended: k_g2p, the migration unpack kernels)
//   k_order_a/b/c : exclusive scans over the dense tile arrays of (stay+arrivals, arrivals, active)
//                   -> next-run offsets, arrival-segment offsets, compact active-tile list + slot_map
//   k_mover_place : movers into their tile's arrival segment (order arbitrary)
//   k_mover_rank  : segment sorted by storage row => deterministic visiting order
constexpr int ORD_B = 256, ORD_IPT = 4, ORD_TILE = ORD_B * ORD_IPT;

// arrival counted where the mover is appended (k_g2p, the migration unpack kernels): no counting pass in the ordering
#define MPMB_COUNT_ARRIVAL(V, P, key) if ((key) < (uint32_t)(P).ntiles_total) atomicAdd(&(V).arr_cnt[key], 1)
// arrivals per tile straight from radix-sorted keys (upload path: every particle is an arrival)
__global__ void k_count_sorted(View V, const uint32_t *keys_sorted, int n, int ntot) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t t = keys_sorted[i];
  if (t >= (uint32_t)ntot) return;
  if (i > 0 && keys_sorted[i - 1] == t) return;
  int lo = i + 1, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (keys_sorted[mid] == t) lo = mid + 1;
    else hi = mid;
  }
  V.arr_cnt[t] = lo - i;
}

__global__ void __launch_bounds__(ORD_B) k_order_a(View V, int ntot) {
  typedef cub::BlockReduce<int, ORD_B> Red;
  __shared__ typename Red::TempStorage tmp;
  int s_tot = 0, s_arr = 0, s_act = 0;
#pragma unroll
  for (int k = 0; k < ORD_IPT; k++) {
    const int t = blockIdx.x * ORD_TILE + threadIdx.x * ORD_IPT + k;
    if (t < ntot) {
      const int a = V.arr_cnt[t], tot = V.stay_cnt[t] + a;
      s_tot += tot; s_arr += a; s_act += tot > 0;
    }
  }
  s_tot = Red(tmp).Sum(s_tot); __syncthreads();
  s_arr = Red(tmp).Sum(s_arr); __syncthreads();
  s_act = Red(tmp).Sum(s_act);
  if (threadIdx.x == 0) { V.blocksum[3 * blockIdx.x] = s_tot; V.blocksum[3 * blockIdx.x + 1] = s_arr; V.blocksum[3 * blockIdx.x + 2] = s_act; }
}

__global__ void __launch_bounds__(1024) k_order_b(View V, int nblocks) {
  // single CTA: exclusive scan of the three block sums (nblocks is a few thousand at most)
  typedef cub::BlockScan<int, 1024> Scan;
  __shared__ typename Scan::TempStorage tmp;
  int carry[3] = {0, 0, 0};
  for (int base = 0; base < nblocks; base += 1024) {
    const int i = base + threadIdx.x;
#pragma unroll
    for (int c = 0; c < 3; c++) {
      int v = i < nblocks ? V.blocksum[3 * i + c] : 0, ex, agg;
      Scan(tmp).ExclusiveSum(v, ex, agg);
      __syncthreads();
      if (i < nblocks) V.blocksum[3 * i + c] = ex + carry[c];
      carry[c] += agg;
    }
  }
  if (threadIdx.x == 0) {
    V.cnt->n_alive = carry[0];
    V.cnt->updates += (unsigned long long)carry[0];
    V.cnt->n_tiles = carry[2];
    V.cnt->n_ghost = 0;
    for (int k = 0; k < 6; k++) (&V.cnt->claim[0][0])[k] = 0;
    if (carry[2] > V.cap_tiles) atomicOr(&V.cnt->error, DEVERR_TILE_CAPACITY);
    if (carry[0] > V.cap_particles) atomicOr(&V.cnt->error, DEVERR_PARTICLE_CAPACITY);
  }
}

#define MPMB_TILE_XYZ(P, tm, tx, ty, tz) const int tx = (tm).xy & 0xffff, ty = (tm).xy >> 16, tz = (tm).z
__global__ void __launch_bounds__(ORD_B) k_order_c(View V, int ntot, int nt1, int nt2, int tz_off) {
  typedef cub::BlockScan<int, ORD_B> Scan;
  __shared__ typename Scan::TempStorage tmp;
  int tot[ORD_IPT], arr[ORD_IPT], act[ORD_IPT];
  int s_tot = 0, s_arr = 0, s_act = 0;
#pragma unroll
  for (int k = 0; k < ORD_IPT; k++) {
    const int t = blockIdx.x * ORD_TILE + threadIdx.x * ORD_IPT + k;
    tot[k] = arr[k] = act[k] = 0;
    if (t < ntot) {
      arr[k] = V.arr_cnt[t];
      tot[k] = V.stay_cnt[t] + arr[k];
      act[k] = tot[k] > 0;
    }
    s_tot += tot[k]; s_arr += arr[k]; s_act += act[k];
  }
  int e_tot, e_arr, e_act;
  Scan(tmp).ExclusiveSum(s_tot, e_tot); __syncthreads();
  Scan(tmp).ExclusiveSum(s_arr, e_arr); __syncthreads();
  Scan(tmp).ExclusiveSum(s_act, e_act);
  e_tot += V.blocksum[3 * blockIdx.x];
  e_arr += V.blocksum[3 * blockIdx.x + 1];
  e_act += V.blocksum[3 * blockIdx.x + 2];
#pragma unroll
  for (int k = 0; k < ORD_IPT; k++) {
    const int t = blockIdx.x * ORD_TILE + threadIdx.x * ORD_IPT + k;
    if (t < ntot) {
      V.out_begin[t] = e_tot;
      V.total[t] = tot[k];
      V.arr_off[t] = e_arr;
      V.arr_len[t] = arr[k];
      V.arr_cnt[t] = 0;   // ready for the next substep's count
      V.arr_cur[t] = 0;   // cursor of k_mover_place
      V.stay_next[t] = 0; // G2P writes it for the tiles it visits
      int slot = -1;
      if (act[k] && e_act < V.cap_tiles) {
        slot = e_act;
        TileMeta m;
        m.tile = t; m.run_begin = V.run_begin[t]; m.run_len = V.run_len[t]; m.arr_off = e_arr; m.arr_len = arr[k]; m.out_begin = e_tot;
        m.xy = (t / (nt2 * nt1)) | (((t / nt2) % nt1) << 16); m.z = t % nt2 + tz_off;
        V.meta[slot] = m;
      }
      V.slot_map[t] = slot;
    }
    e_tot += tot[k]; e_arr += arr[k]; e_act += act[k];
  }
}

__global__ void k_mover_place(View V, int ntot) {
  const int n = V.cnt->n_movers;
  for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < n; m += gridDim.x * blockDim.x) {
    const uint32_t d = V.mover_dst[m];
    if (d < (uint32_t)ntot) {
      const int pos = atomicAdd(&V.arr_cur[d], 1);
      if (!MPMB_CHK(V.cnt, pos < V.arr_len[d] && V.arr_off[d] + pos < V.cap_particles && V.mover_idx[m] < (uint32_t)V.cap_particles, 1, d, pos, V.arr_len[d])) continue;
      V.arrivals[V.arr_off[d] + pos] = V.mover_idx[m];
    }
  }
}

__global__ void k_mover_rank(View V, int ntot) {
  const int n = V.cnt->n_movers;
  for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < n; m += gridDim.x * blockDim.x) {
    const uint32_t d = V.mover_dst[m];
    if (d < (uint32_t)ntot) {
      const uint32_t idx = V.mover_idx[m];
      const int off = V.arr_off[d], len = V.arr_len[d];
      int rank = 0;
      for (int e = 0; e < len; e++) rank += V.arrivals[off + e] < idx;
      if (!MPMB_CHK(V.cnt, off + rank < V.cap_particles && rank < len, 2, d, rank, len)) continue;
      V.arrivals_sorted[off + rank] = idx;
    }
  }
}

#ifdef MPMB_VALIDATE
// debug: after the ordering every tile must have received exactly the arrivals that were counted for it, its arrival
// rows must be live storage rows, and the runs must tile the next storage without overlap
__global__ void k_validate_order(View V, int ntot) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < ntot; t += gridDim.x * blockDim.x) {
    if (V.arr_cur[t] != V.arr_len[t]) {
      if (atomicCAS(&V.cnt->chk[0], 0, 20) == 0) { V.cnt->chk[1] = t; V.cnt->chk[2] = V.arr_cur[t]; V.cnt->chk[3] = V.arr_len[t]; }
    }
    if (V.run_begin[t] + V.run_len[t] > V.cnt->n_store || V.run_len[t] < V.stay_cnt[t]) {
      if (atomicCAS(&V.cnt->chk[0], 0, 21) == 0) { V.cnt->chk[1] = t; V.cnt->chk[2] = V.run_len[t]; V.cnt->chk[3] = V.stay_cnt[t]; }
    }
    for (int e = 0; e < V.arr_len[t]; e++) {
      const uint32_t row = V.arrivals_sorted[V.arr_off[t] + e];
      if (row >= (uint32_t)V.cnt->n_store || V.keys[row] != (uint32_t)t || (e > 0 && V.arrivals_sorted[V.arr_off[t] + e - 1] >= row)) {
        if (atomicCAS(&V.cnt->chk[0], 0, 22) == 0) { V.cnt->chk[1] = t; V.cnt->chk[2] = (int)row; V.cnt->chk[3] = row < (uint32_t)V.cnt->n_store ? (int)V.keys[row] : -7; }
      }
    }
  }
}
extern "C" int mpmb_debug_check(MpmbHandle h, int *out8);
#endif

// ------------------------------------------------------------------------------ P2G
// Replaces MPM<3>::rasterize_optimized / block_op_normal (src/transfer.cpp:467-569).
// One 128-thread CTA per active tile (persistent round-robin).  A tile's rows are its run (unit
// stride, holes where a particle left) followed by its arrivals.  Per chunk of <=CH rows:
//   1. stage: 16-byte async copies (LDGSTS) of the P2G set (64 B/particle) into padded shared rows,
//      all in flight at once;
//   2. sort:  stable counting sort of the rows by cell (warp match + per-32-row-group histograms),
//             bit-reproducible; publishes each particle's row in the next storage (outpos);
//   3. accumulate: two threads own cell c (tid = c and c + 64) and both stream that cell's particles;
//      each accumulates HALF of the 27-node stencil x (p_x,p_y,p_z,m) in registers — every particle of
//      a cell shares one stencil.  Flush steps n = i*9 + j*3 + k in [0, 14) belong to warps 0-1,
//      [14, 27) to warps 2-3; both halves compute every particle's weights and Q;
//   4. flush: each warp adds its registers into a shared 6x6x6 arena, conflict-free by layout
//      (node strides 68/8/1 put the 32 cells of a warp on 32 banks), step after step;
// then one coalesced store of the arena.  No atomics on floats anywhere.
constexpr int P2G_T = 128;         // threads = 2 per cell of the tile
constexpr int P2G_SPLIT = 14;      // flush steps of the first stencil half
// particles staged per chunk: a full interior tile is 512 rows at 8 particles per cell, and in a developed flow a quarter
// of the tiles sit a little above that — 576 keeps most of them in ONE chunk; the per-row passes below skip the empty
// tail of a short chunk
#ifndef MPMB_P2G_CH
#define MPMB_P2G_CH 576
#endif
constexpr int P2G_CH = MPMB_P2G_CH;
static_assert(P2G_CH % 32 == 0 && P2G_CH <= 65536, "P2G chunk: whole warps of rows, row ids in 16 bits");
constexpr int P2G_K = (P2G_CH + P2G_T - 1) / P2G_T;  // staging passes (r = k*T + tid); the last one may be partial
constexpr int P2G_G = P2G_CH / 32;                   // 32-row groups = (pass, warp) histogram buckets, row order
constexpr int P2G_ROWS = P2G_CH + P2G_CH / 8;  // padded row index r + (r>>3): cell-run reads hit distinct banks
constexpr int P2G_DYN_BYTES = 4 * P2G_ROWS * (int)sizeof(float4);
constexpr int AR_SX = 68, AR_SY = 8;           // arena strides in shared memory
constexpr int AR_SIZE = 6 * AR_SX;

// Step 3 for one stencil half H: the cell's particles s_order[i0, i1) into acc[n - lo] for the flush steps n in [lo, hi).
// The half is a template parameter, so the unrolled node chain keeps only its own nodes, straight-line.  Each node gets
// the same operations as in a whole-stencil loop, so the sums do not depend on the split.
template <int H>
__device__ __forceinline__ void p2g_accumulate(F4 (&acc)[P2G_SPLIT], const float4 (*s_rows)[P2G_ROWS], const unsigned short *s_order,
                                               int i0, int i1, const Params &P, float fbx, float fby, float fbz) {
  constexpr int lo = H ? P2G_SPLIT : 0, hi = H ? 27 : P2G_SPLIT;
  for (int it = i0; it < i1; it++) {
    const int r = s_order[it];
    const int ri = r + (r >> 3);
    const float4 a0 = s_rows[0][ri], a1 = s_rows[1][ri], a2 = s_rows[2][ri], a3 = s_rows[3][ri];
    const float mass = fabsf(a0.w);
    float vx = a1.x, vy = a1.y, vz = a1.z;
    if (P.particle_gravity) {  // src/transfer.cpp:485-487
      vx += P.gdt[0]; vy += P.gdt[1]; vz += P.gdt[2];
    }
    // rel = pos/dx - base node of this cell (src/transfer.cpp:490,518)
    const float rx = __fsub_rn(__fmul_rn(a0.x, P.inv_dx), fbx), ry = __fsub_rn(__fmul_rn(a0.y, P.inv_dx), fby),
                rz = __fsub_rn(__fmul_rn(a0.z, P.inv_dx), fbz);
    float wx[3], wy[3], wz[3];
    bspline_weights(rx, wx);
    bspline_weights(ry, wy);
    bspline_weights(rz, wz);
    // A columns: c0 = (a1.w,a2.x,a2.y) c1 = (a2.z,a2.w,a3.x) c2 = (a3.y,a3.z,a3.w)
    // q = m v + A rel ;  node (i,j,k): q - i c0 - j c1 - k c2   (dpos = rel - node, 528-536)
    const float q0 = fmaf(a3.y, rz, fmaf(a2.z, ry, fmaf(a1.w, rx, mass * vx)));
    const float q1 = fmaf(a3.z, rz, fmaf(a2.w, ry, fmaf(a2.x, rx, mass * vy)));
    const float q2 = fmaf(a3.w, rz, fmaf(a3.x, ry, fmaf(a2.y, rx, mass * vz)));
    // (momentum | mass) as register pairs; the mass lane rides along with zero column entries
    const F4 Q = {make_float2(q0, q1), make_float2(q2, mass)};
    const F4 c0 = {make_float2(a1.w, a2.x), make_float2(a2.y, 0.f)}, c1 = {make_float2(a2.z, a2.w), make_float2(a3.x, 0.f)},
             c2 = {make_float2(a3.y, a3.z), make_float2(a3.w, 0.f)};
    const float2 m2 = bc2(-2.0f);
    const float2 wx2[3] = {bc2(wx[0]), bc2(wx[1]), bc2(wx[2])}, wy2[3] = {bc2(wy[0]), bc2(wy[1]), bc2(wy[2])},
                 wz2[3] = {bc2(wz[0]), bc2(wz[1]), bc2(wz[2])};
#pragma unroll
    for (int i = 0; i < 3; i++) {
      if (i * 9 + 8 < lo || i * 9 >= hi) continue;
      const F4 U = i == 0 ? Q : (i == 1 ? f4_sub(Q, c0) : f4_fma(m2, c0, Q));    // q - i c0
#pragma unroll
      for (int j = 0; j < 3; j++) {
        if (i * 9 + j * 3 + 2 < lo || i * 9 + j * 3 >= hi) continue;
        const F4 T = j == 0 ? U : (j == 1 ? f4_sub(U, c1) : f4_fma(m2, c1, U));  // ... - j c1
        const float2 wij = mul2(wx2[i], wy2[j]);
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const int n = i * 9 + j * 3 + k;
          if (n < lo || n >= hi) continue;
          const float2 w = mul2(wij, wz2[k]);
          const F4 N = k == 0 ? T : (k == 1 ? f4_sub(T, c2) : f4_fma(m2, c2, T));  // ... - k c2
          acc[n - lo] = f4_fma(w, N, acc[n - lo]);
        }
      }
    }
  }
}

// Step 4 for one stencil half H: add acc into the arena `ar` at the cell's base node nb, flush step after flush step.
template <int H>
__device__ __forceinline__ void p2g_flush(const F4 (&acc)[P2G_SPLIT], float (*ar)[AR_SIZE], int nb) {
  constexpr int lo = H ? P2G_SPLIT : 0, hi = H ? 27 : P2G_SPLIT;
#pragma unroll
  for (int n = lo; n < hi; n++) {
    const int node = nb + (n / 9) * AR_SX + ((n / 3) % 3) * AR_SY + n % 3;
    const F4 &a = acc[n - lo];
    ar[0][node] += a.lo.x;
    ar[1][node] += a.lo.y;
    ar[2][node] += a.hi.x;
    ar[3][node] += a.hi.y;
    __syncwarp();
  }
}

// The time of this kernel is in-warp latency of the per-particle dependency chain.  Two threads per cell halve the
// accumulators (56 registers instead of 108), so 4 CTAs per SM — the limit of its 51.7 KB of shared memory — are 16 warps
// instead of 8.  The persistent grid is sized from the occupancy query in mpmb_create.
__global__ void __launch_bounds__(P2G_T, 4) k_p2g(View V, Params P, int part) {
  // the row staging area is dynamic shared memory (static + dynamic = 51.7 KB, above the 48 KB static limit)
#ifndef MPMB_SIMT_HOST
  extern __shared__ __align__(16) unsigned char p2g_dyn[];
#else
  __shared__ __align__(16) unsigned char p2g_dyn[P2G_DYN_BYTES];
#endif
  float4 (*s_rows)[P2G_ROWS] = reinterpret_cast<float4 (*)[P2G_ROWS]>(p2g_dyn);
  __shared__ unsigned short s_order[P2G_CH];
  __shared__ unsigned short s_hist[P2G_G][64];
  __shared__ int s_start[65];
  __shared__ float s_arena[4][AR_SIZE];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int own = tid & 63, half = tid >> 6;  // my cell, and which half of its stencil I accumulate (warp-uniform)
  const int cx = own >> 4, cy = (own >> 2) & 3, cz = own & 3;
  const int n_tiles = V.cnt->n_tiles;
  MPMB_TRACE_BEGIN;
  // Tiles are handed out in slot order from the launch's counter (the first gridDim.x by block index): a CTA that drew
  // small tiles takes more, so the launch ends at most one tile after its average CTA instead of with its most loaded
  // one.  Thread 0 claims the next tile at the top of the current one and publishes it with the tile's last barrier,
  // in s_claim[cp ^ 1] while everyone reads this tile's s_claim[cp].
  __shared__ int s_claim[2];
  int *const counter = &V.cnt->claim[0][part];
  auto claim = [&](int slot) {  // the first tile of the part at or after `slot`, drawing replacements from the counter
    while (slot < n_tiles && part != 0 && !tile_in_part(P, V.meta[slot].tile, part)) slot = (int)gridDim.x + atomicAdd(counter, 1);
    return slot;
  };
  if (tid == 0) s_claim[0] = claim(blockIdx.x);
  __syncthreads();
  for (int slot = s_claim[0], cp = 0; slot < n_tiles; cp ^= 1, slot = s_claim[cp]) {
    int ahead = 0;
    if (tid == 0) ahead = (int)gridDim.x + atomicAdd(counter, 1);  // consumed after the tile's work: the latency is hidden
    const TileMeta tm = V.meta[slot];
    const int nrow_tile = tm.run_len + tm.arr_len;
    // (the tile's output rows are not indexed here; out_begin + run_len + arr_len may pass the capacity when the run has holes)
    if (!MPMB_CHK(V.cnt, tm.run_begin >= 0 && tm.run_len >= 0 && tm.arr_len >= 0 && tm.run_begin + tm.run_len <= V.cap_particles && tm.arr_off + tm.arr_len <= V.cap_particles,
                  3, slot, tm.run_begin, tm.run_len)) {
      if (tid == 0) s_claim[cp ^ 1] = claim(ahead);
      __syncthreads();
      continue;
    }
    MPMB_TRACE_TILE(nrow_tile);
    MPMB_TILE_XYZ(P, tm, tx, ty, tz);
    const float fbx = (float)(tx * 4 + cx), fby = (float)(ty * 4 + cy), fbz = (float)(tz * 4 + cz);
    F4 acc[P2G_SPLIT];  // (p_x, p_y | p_z, m) of my half of my cell's stencil
#pragma unroll
    for (int n = 0; n < P2G_SPLIT; n++) acc[n] = f4_zero();
    for (int n = tid; n < AR_SIZE; n += P2G_T) { s_arena[0][n] = 0.f; s_arena[1][n] = 0.f; s_arena[2][n] = 0.f; s_arena[3][n] = 0.f; }
    int vbase = 0;  // valid rows in the chunks already processed
    // storage row of tile-row g: run rows first, then arrivals
    auto row_of = [&](int g) -> uint32_t {
      return g < tm.run_len ? (uint32_t)(tm.run_begin + g) : V.arrivals_sorted[tm.arr_off + (g - tm.run_len)];
    };

    for (int cb = 0; cb < nrow_tile; cb += P2G_CH) {
      const int nrows = min(P2G_CH, nrow_tile - cb);
      for (int n = tid; n < P2G_G * 64; n += P2G_T) (&s_hist[0][0])[n] = 0;
      // ---- 1: stage rows: all copies of the chunk in flight at once
      uint32_t pidx[P2G_K];
      if (cb + nrows <= tm.run_len) {  // whole chunk inside the run (the common case): pure arithmetic, no loads
#pragma unroll
        for (int k = 0; k < P2G_K; k++) pidx[k] = (uint32_t)(tm.run_begin + cb + k * P2G_T + tid);
      } else {
#pragma unroll
        for (int k = 0; k < P2G_K; k++) {
          const int r = k * P2G_T + tid;
          pidx[k] = r < nrows ? row_of(cb + r) : 0u;
          if (!MPMB_CHK(V.cnt, pidx[k] < (uint32_t)V.cap_particles, 4, slot, pidx[k], cb + r)) pidx[k] = 0u;
        }
      }
#pragma unroll
      for (int k = 0; k < P2G_K; k++) {
        const int r = k * P2G_T + tid;
        if (r < nrows) {
          const int ri = r + (r >> 3);
          cp_async16(&s_rows[0][ri], &V.q[0][pidx[k]]);
          cp_async16(&s_rows[1][ri], &V.q[1][pidx[k]]);
          cp_async16(&s_rows[2][ri], &V.q[2][pidx[k]]);
          cp_async16(&s_rows[3][ri], &V.q[3][pidx[k]]);
        }
      }
      cp_async_commit();
      cp_async_wait_all();
      __syncthreads();
      // ---- 2a: per-32-row-group cell histograms (each thread reads back its own rows; group r>>5 = (pass, warp))
      uint32_t cr[P2G_K];
#pragma unroll
      for (int k = 0; k < P2G_K; k++) {
        const int r = k * P2G_T + tid;
        int cell = 64 + warp;  // holes and rows past the end: a private bucket
        if (k * P2G_T >= nrows) {  // uniform: nothing staged for this pass
          cr[k] = (uint32_t)cell << 16;
          continue;
        }
        float4 a0 = make_float4(0.f, 0.f, 0.f, -1.f);
        if (r < nrows) a0 = s_rows[0][r + (r >> 3)];
        // G2P stores the mass NEGATED when the particle's base node left the tile of the run it was
        // written to: run rows with mass < 0 are holes (the particle is in another tile's arrivals)
        if (r < nrows && (a0.w > 0.f || cb + r >= tm.run_len)) {
          int bx, by, bz;
          float rr;
          base_rel(a0.x, P.inv_dx, bx, rr);
          base_rel(a0.y, P.inv_dx, by, rr);
          base_rel(a0.z, P.inv_dx, bz, rr);
          cell = (((bx - tx * 4) & 3) << 4) | (((by - ty * 4) & 3) << 2) | ((bz - tz * 4) & 3);
        }
        const unsigned m = __match_any_sync(0xffffffffu, cell);
        const int rank = __popc(m & ((1u << lane) - 1u));
        if (cell < 64) {  // implies r < nrows <= CH: the group exists
          if (rank == 0) s_hist[r >> 5][cell] = (unsigned short)__popc(m);
        }
        cr[k] = ((uint32_t)cell << 16) | (uint32_t)rank;
      }
      __syncthreads();
      // ---- 2b: exclusive scan over the row groups per cell (threads 0..63, one per cell), then over cells
      {
        int run = 0, incl = 0;
        if (tid < 64) {
#pragma unroll
          for (int e = 0; e < P2G_G; e++) {
            const int h = s_hist[e][tid];
            s_hist[e][tid] = (unsigned short)run;
            run += h;
          }
          incl = run;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
          }
          if (tid == 31) s_start[64] = incl;  // total of warp 0, fixed up below
        }
        __syncthreads();
        const int base0 = warp ? s_start[64] : 0;
        if (tid < 64) s_start[tid] = base0 + incl - run;
        __syncthreads();
        if (tid == 63) s_start[64] = base0 + incl;
      }
      // ---- 2c: scatter row ids to their sorted position; publish the output row for G2P
#pragma unroll
      for (int k = 0; k < P2G_K; k++) {
        const int r = k * P2G_T + tid;
        const int cell = (int)(cr[k] >> 16);
        if (cell < 64) {
          const int pos = s_start[cell] + s_hist[r >> 5][cell] + (int)(cr[k] & 0xffffu);
          s_order[pos] = (unsigned short)r;
          V.outpos[pidx[k]] = (uint32_t)(tm.out_begin + vbase + pos);
        }
        // holes are NOT marked here: the same storage row is a hole of its old tile and an arrival of
        // its new one, and two CTAs must not write different values to one outpos entry
      }
      __syncthreads();
      // ---- 3: accumulate my half of my cell's stencil in registers.  A warp iterates as long as its fullest cell has
      // particles; in a developed flow (cells hold 0..30 particles) that is the kernel's cost.  Tried and dropped:
      // capping the loop and adding the excess particles with one lane per stencil node (the serialised excess pass
      // costs more than the idle tail), re-assigning cells to threads per tile so that warp 0 owns the fuller cells, and
      // software-pipelining the row fetch: the kernel is latency-bound, an early warp's issue slots are not what it lacks.
      const int i0 = s_start[own], i1 = s_start[own + 1];
      if (half == 0)
        p2g_accumulate<0>(acc, s_rows, s_order, i0, i1, P, fbx, fby, fbz);
      else
        p2g_accumulate<1>(acc, s_rows, s_order, i0, i1, P, fbx, fby, fbz);
      vbase += s_start[64];
      __syncthreads();  // rows / order / hist are reused by the next chunk
    }
    // ---- 4: cells 0-31 flush into s_arena, cells 32-63 into a second arena laid over the row staging area (free after
    // the last chunk's barrier; zeroed by warp 1 itself, so a __syncwarp is all it needs).  Warps 0-1 flush steps
    // [0, 14), then warps 2-3 flush [14, 27): every node receives its adds in ascending step order, as from one thread
    // holding the whole stencil.  The store below sums the two arenas in a fixed order: still bit-reproducible.
    float (*ar1)[AR_SIZE] = reinterpret_cast<float (*)[AR_SIZE]>(&s_rows[0][0]);
    {
      float (*ar)[AR_SIZE] = (warp & 1) ? ar1 : s_arena;
      const int nb = cx * AR_SX + cy * AR_SY + cz;
      if (half == 0) {
        if (warp == 1) {
          for (int n = lane; n < 4 * AR_SIZE; n += 32) (&ar1[0][0])[n] = 0.f;
          __syncwarp();
        }
        p2g_flush<0>(acc, ar, nb);
      }
      __syncthreads();
      if (half == 1) p2g_flush<1>(acc, ar, nb);
    }
    __syncthreads();
    float4 *out = V.arena + (size_t)slot * ARENA;
    for (int n = tid; n < ARENA; n += P2G_T) {
      const int a = n / 36, b = (n / 6) % 6, c = n % 6;
      const int node = a * AR_SX + b * AR_SY + c;
      out[n] = make_float4(s_arena[0][node] + ar1[0][node], s_arena[1][node] + ar1[1][node], s_arena[2][node] + ar1[2][node],
                           s_arena[3][node] + ar1[3][node]);
    }
    if (tid == 0) s_claim[cp ^ 1] = claim(ahead);
    __syncthreads();
  }
  MPMB_TRACE_END(TRACE_P2G);
}


// ------------------------------------------------------------------------------ grid node
// Momentum/mass of global node g = fixed-order sum of the arenas that cover it:
// owner tile T=(g>>2) holds it at local l=g&3; tile T-o (o in {0,1}^3) holds it at l+4o (needs l<=1).
// The <=8 loads are predicated, not branched around, so they stay independent and issue back to back.
template <class SlotOf>
__device__ __forceinline__ float4 gather_node(const float4 *arena, int zero_slot, int lx, int ly, int lz, SlotOf slot_of) {
  (void)zero_slot;
  float4 a[8];
#pragma unroll
  for (int o = 0; o < 8; o++) {
    const int ox = o >> 2, oy = (o >> 1) & 1, oz = o & 1;
    const int slot = slot_of(ox, oy, oz);
    const bool covered = !(ox && lx > 1) && !(oy && ly > 1) && !(oz && lz > 1) && slot >= 0;
    const int idx = ((lx + 4 * ox) * 6 + (ly + 4 * oy)) * 6 + (lz + 4 * oz);
    a[o] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (covered) a[o] = arena[(size_t)slot * ARENA + idx];
  }
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int o = 0; o < 8; o++) { acc.x += a[o].x; acc.y += a[o].y; acc.z += a[o].z; acc.w += a[o].w; }
  return acc;
}

// the level set at node (gx, gy, gz), or nothing to project on (no level set, or a node past the grid)
__device__ __forceinline__ bool node_sdf(const Params &P, const float4 *sdf4, int gx, int gy, int gz, float4 &s) {
  s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!(P.has_sdf && gx < P.nnode[0] && gy < P.nnode[1] && gz < P.nnode[2])) return false;
  s = sdf4[((size_t)gx * P.nnode[1] + gy) * P.nnode[2] + gz];
  return true;
}

// normalize_grid_and_apply_external_force (src/mpm.cpp:277-294) + apply_grid_boundary_conditions
// (src/mpm.cpp:296-372, static level set) for one node; has_s / s: node_sdf of the node.
__device__ __forceinline__ float4 node_update(const Params &P, float4 g, bool has_s, float4 s) {
  float m = g.w;
  if (m > 0.f) {
    float inv = 1.0f / m;
    float ix = P.particle_gravity ? 0.f : P.gdt[0], iy = P.particle_gravity ? 0.f : P.gdt[1], iz = P.particle_gravity ? 0.f : P.gdt[2];
    g.x = fmaf(g.x, inv, ix);
    g.y = fmaf(g.y, inv, iy);
    g.z = fmaf(g.z, inv, iz);
  }
  if (has_s && m != 0.f) {
    if (!(s.w < -3.0f || 0.0f < s.w)) {
      float3 v = friction_project0(make_float3(g.x, g.y, g.z), make_float3(s.x, s.y, s.z), P.friction);
      g.x = v.x; g.y = v.y; g.z = v.z;
    }
  }
  return g;
}

// ------------------------------------------------------------------------------ grid update
// Replaces normalize_grid_and_apply_external_force (src/mpm.cpp:277-294) + apply_grid_boundary_conditions
// (src/mpm.cpp:296-372) for the nodes one tile's particles gather from.  Every arena is final once k_p2g (and, on a
// z-slab rank, the halo exchange) has run, so the G2P kernels build each tile's block themselves, in shared memory,
// instead of reading it back from a node array that a separate grid pass wrote.

// slot of the neighbour tile k (= (ox+1)*9 + (oy+1)*3 + (oz+1), o in {-1,0,1}^3) of tile (tx, ty, tz); -1: none
__device__ __forceinline__ int neighbour_slot(const View &V, const Params &P, int slot, int tx, int ty, int tz, int k) {
  const int x = tx + k / 9 - 1, y = ty + (k / 3) % 3 - 1, z = tz + k % 3 - 1 - P.tz_off;  // z: local layer
  int nb = -1;
  if (x >= 0 && y >= 0 && z >= 0 && x < P.nt[0] && y < P.nt[1] && z < P.nt[2]) nb = V.slot_map[(x * P.nt[1] + y) * P.nt[2] + z];
  if (!MPMB_CHK(V.cnt, nb >= -1 && nb < V.cap_tiles, 5, slot, nb, k)) nb = -1;
  return nb;
}

// The 6x6x6 nodes of tile (tx, ty, tz), each the fixed-order sum of the arenas that cover it (nb: the tile's 27
// neighbour slots), normalised and projected on the level set, into s_vel; the CTA's BLOCK threads share the nodes.
// The caller puts a block barrier between this and the first read of s_vel.  Every global load of a thread's nodes
// (arenas and level set) is issued before its first store to s_vel, which the compiler cannot move loads across: the
// build costs one round trip to L2 / HBM, not two per node with the nodes one after the other.
template <int BLOCK>
__device__ __forceinline__ void build_node_block(const View &V, const Params &P, int tx, int ty, int tz, const int *nb, float4 *s_vel) {
  constexpr int NPT = (ARENA + BLOCK - 1) / BLOCK;  // nodes per thread
  float4 g[NPT], s[NPT];
  bool has_s[NPT];
#pragma unroll
  for (int k = 0; k < NPT; k++) {
    const int n = min(k * BLOCK + (int)threadIdx.x, ARENA - 1);  // the last pass is partial: clamp, store guarded
    const int a = n / 36, b = (n / 6) % 6, c = n % 6;
    const int wx_ = a >> 2, wy_ = b >> 2, wz_ = c >> 2;  // owner tile offset (0/1)
    g[k] = gather_node(V.arena, V.cap_tiles, a & 3, b & 3, c & 3,
                       [&](int ox, int oy, int oz) { return nb[(wx_ - ox + 1) * 9 + (wy_ - oy + 1) * 3 + (wz_ - oz + 1)]; });
    has_s[k] = node_sdf(P, V.sdf4, tx * 4 + a, ty * 4 + b, tz * 4 + c, s[k]);
  }
#pragma unroll
  for (int k = 0; k < NPT; k++) {
    const int n = k * BLOCK + (int)threadIdx.x;
    if (n < ARENA) s_vel[n] = node_update(P, g[k], has_s[k], s[k]);
  }
}

// ------------------------------------------------------------------------------ G2P
// Replaces MPM<3>::resample_optimized / block_op_normal (src/transfer.cpp:837-954) + Particle::plasticity +
// clear_boundary_particles (src/mpm.cpp:583-633); produces the affine matrix of the NEXT rasterize
// (calculate_force of the updated state), writes the tile's particles cell-sorted into one contiguous
// run of the other buffer, and appends the particles whose base node left the tile to the mover list.
// Persistent CTAs walk their tiles chunk by chunk through a two-stage cp.async pipeline: while the
// warps compute chunk i out of one shared buffer, the rows (64 B/particle) of chunk i+1 are already
// in flight into the other.  At the first chunk of a tile the CTA builds the tile's 216 node
// velocities from the arenas (build_node_block) while that chunk's successor is in flight.
constexpr int G2P_CH = 256;  // rows per pipeline stage
// STORE_B = false skips the apic_b streams (48 B/particle): no kernel reads apic_b — rasterize uses the
// affine matrix A — so inside mpmb_substep(h, n) only the LAST substep has to leave it behind for the
// host (downloads, visualize, save).
// EXT_MATS = false leaves the elastic / von Mises / visco branches of material_step out (see mpmb_math.cuh).
template <int BLOCK, bool STORE_B, bool EXT_MATS>
__global__ void __launch_bounds__(BLOCK, 5) k_g2p(View V, Params P, int part, int commit) {
  // node block of the current tile: written at its first chunk, after the previous tile's last end-of-chunk barrier
  __shared__ __align__(16) float4 s_vel[ARENA];
  // the 27 neighbour slots of the current tile [sp] and of the tile claimed ahead [sp ^ 1], loaded one tile ahead so
  // that the build's first loads are the arenas'
  __shared__ int s_nb[2][27];
  __shared__ __align__(16) float4 s_in[2][4][G2P_CH];
  // output row of every staged row: run rows at [sh + r] (sh = 16-byte alignment shift of the run's outpos words),
  // arrival rows at [r + 8] — clear of the up to 3 words by which the bulk copy of the run part is rounded up
  __shared__ __align__(16) uint32_t s_out[2][G2P_CH + 8];
  __shared__ __align__(8) uint64_t s_bar[2];               // one mbarrier per pipeline stage
  // particles of the current tile that stay in it.  TWO slots, alternating per tile: thread 0 reads and clears a tile's
  // slot after the tile's last barrier while the other warps are already adding to the next tile's slot — with one slot
  // (round 1, when a barrier at the top of the loop covered it) a late warp 0 folded the next tile's first additions
  // into this tile's count: stay counts drifted, runs overlapped (found with -DMPMB_VALIDATE)
  __shared__ int s_stay[2];
  constexpr int KPT = G2P_CH / BLOCK;
  const int tid = threadIdx.x;
  const int n_tiles = V.cnt->n_tiles;
  MPMB_TRACE_BEGIN;
  const float scale = -4.0f * P.inv_dx * P.dt;  // src/transfer.cpp:938
  // Tiles are handed out in slot order from the launch's counter (the first gridDim.x by block index), as in k_p2g.  The
  // pipeline puts a tile's first chunk in flight while the previous tile's last chunk is computed, so thread 0 claims
  // ONE TILE AHEAD: s_ahead[sp ^ 1] is the CTA's next tile, read by everyone at the tile change; thread 0 then claims the
  // one after it into s_ahead[sp], which the end-of-chunk barrier publishes (sp alternates per tile, as for s_stay).  A
  // tile's chunks stay with its CTA.  (No pointer or index of its own is kept live: the loop is at the register limit.)
  __shared__ int s_ahead[2];
  auto next_claim = [&]() { return (int)gridDim.x + atomicAdd(&V.cnt->claim[1][part], 1); };
  auto claim = [&](int slot) {  // the first tile at or after `slot` this kernel processes, drawing replacements from the counter
    // z-slab parts: tiles of the other part; CPIC scenes: tiles of rigid pages belong to k_g2p_rigid
    while (slot < n_tiles && ((part != 0 && !tile_in_part(P, V.meta[slot].tile, part)) || (V.rigid_flag && V.rigid_flag[slot]))) slot = next_claim();
    return slot;
  };
  int sp = 0;
  struct Item { int slot, rb, first; TileMeta tm; };
  auto first_item = [&](int slot) {
    Item it;
    it.rb = 0; it.first = 1;
    it.slot = slot;
    if (slot < n_tiles) it.tm = V.meta[slot];
    else {
      it.tm.run_len = 0; it.tm.arr_len = 0; it.tm.tile = 0; it.tm.run_begin = 0; it.tm.arr_off = 0; it.tm.out_begin = 0;
      it.tm.xy = 0; it.tm.z = 0;
    }
    return it;
  };
  auto next_item = [&](const Item &it) {
    if (it.rb + G2P_CH < it.tm.run_len + it.tm.arr_len) { Item n = it; n.rb += G2P_CH; n.first = 0; return n; }
    return first_item(s_ahead[sp ^ 1]);
  };
  // rows of the chunk that lie inside the tile's run (unit stride in storage) / alignment shift of their outpos words
  auto run_rows = [&](const Item &it) { return max(0, min(G2P_CH, it.tm.run_len - it.rb)); };
  auto out_shift = [&](const Item &it) { return run_rows(it) > 0 ? (int)((uint32_t)(it.tm.run_begin + it.rb) & 3u) : 0; };
  // puts one item in flight: rows of the G2P set (x|mass, F, scalar|vol|tag) and their output rows.  The run part of
  // the chunk is TMA bulk copies issued by thread 0 and tracked by the stage's mbarrier; the (few) arrival rows are
  // gathered with 16-byte LDGSTS copies by the thread that will consume them, tracked by its own copy groups.
  auto prefetch = [&](const Item &it, int buf) {
    if (it.slot < n_tiles) {
      const int nrow_tile = it.tm.run_len + it.tm.arr_len;
      const int nrows = min(G2P_CH, nrow_tile - it.rb);
      const int nrun = run_rows(it);
      const int sh = out_shift(it);
      if (tid == 0) {
        const uint32_t r0 = (uint32_t)(it.tm.run_begin + it.rb);
        const unsigned row_bytes = (unsigned)nrun * 16u, out_bytes = nrun > 0 ? (((unsigned)(sh + nrun) * 4u + 15u) & ~15u) : 0u;
        mbar_arrive_expect_tx(&s_bar[buf], 4u * row_bytes + out_bytes);
        if (nrun > 0) {
          bulk_g2s(&s_in[buf][0][0], &V.q[0][r0], row_bytes, &s_bar[buf]);
          bulk_g2s(&s_in[buf][1][0], &V.q[4][r0], row_bytes, &s_bar[buf]);
          bulk_g2s(&s_in[buf][2][0], &V.q[5][r0], row_bytes, &s_bar[buf]);
          bulk_g2s(&s_in[buf][3][0], &V.q[6][r0], row_bytes, &s_bar[buf]);
          bulk_g2s(&s_out[buf][0], &V.outpos[r0 - (uint32_t)sh], out_bytes, &s_bar[buf]);
        }
      }
      if (nrun < nrows) {
#pragma unroll
        for (int k = 0; k < KPT; k++) {
          const int r = k * BLOCK + tid;
          if (r >= nrun && r < nrows) {
            uint32_t pidx = V.arrivals_sorted[it.tm.arr_off + (it.rb + r - it.tm.run_len)];
            if (!MPMB_CHK(V.cnt, pidx < (uint32_t)V.cap_particles, 6, it.slot, pidx, r)) pidx = 0u;
            cp_async16(&s_in[buf][0][r], &V.q[0][pidx]);
            cp_async16(&s_in[buf][1][r], &V.q[4][pidx]);
            cp_async16(&s_in[buf][2][r], &V.q[5][pidx]);
            cp_async16(&s_in[buf][3][r], &V.q[6][pidx]);
            unsigned d = (unsigned)__cvta_generic_to_shared(&s_out[buf][r + 8]);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(&V.outpos[pidx]));
          }
        }
      }
    }
    cp_async_commit();
  };
  if (tid == 0) {
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    mbar_init_fence();
    s_stay[0] = 0;
    s_stay[1] = 0;
    s_ahead[0] = claim(blockIdx.x);
    s_ahead[1] = s_ahead[0] < n_tiles ? claim(next_claim()) : n_tiles;
  }
  __syncthreads();
  Item cur = first_item(s_ahead[0]);
  if (tid < 27 && cur.slot < n_tiles) s_nb[0][tid] = neighbour_slot(V, P, cur.slot, cur.tm.xy & 0xffff, cur.tm.xy >> 16, cur.tm.z, tid);
  __syncthreads();  // s_ahead[0] is claimed into again at the first tile change
  int buf = 0;
  unsigned phase = 0;  // bit b = parity of the phase stage b's barrier is in
  prefetch(cur, 0);
  while (cur.slot < n_tiles) {
    const Item nxt = next_item(cur);
    prefetch(nxt, buf ^ 1);
    if (nxt.first && nxt.slot < n_tiles) {  // nxt took the tile claimed ahead
      if (tid == 0) s_ahead[sp] = claim(next_claim());
      if (tid < 27) s_nb[sp ^ 1][tid] = neighbour_slot(V, P, nxt.slot, nxt.tm.xy & 0xffff, nxt.tm.xy >> 16, nxt.tm.z, tid);
    }
    if (cur.first) {  // the previous tile's last end-of-chunk barrier has retired every read of s_vel
      build_node_block<BLOCK>(V, P, cur.tm.xy & 0xffff, cur.tm.xy >> 16, cur.tm.z, s_nb[sp], s_vel);
      __syncthreads();
    }
    asm volatile("cp.async.wait_group 1;\n" ::: "memory");  // my arrival rows of the current item have landed; the next item stays in flight
    mbar_wait(&s_bar[buf], (phase >> buf) & 1u);              // ... and so have its bulk copies (every thread reads only rows it waited for)
    phase ^= 1u << buf;
    {
      const int tile = cur.tm.tile;
      const int sh = out_shift(cur), nrun = run_rows(cur);
      MPMB_TILE_XYZ(P, cur.tm, tx, ty, tz);
      const int nrows = min(G2P_CH, cur.tm.run_len + cur.tm.arr_len - cur.rb);
      const float4 *sv = s_vel;
      int my_stay = 0;
      for (int r = tid; r < nrows; r += BLOCK) {
        const float4 q0 = s_in[buf][0][r];
        // run rows with negative mass are holes (the particle now belongs to another tile's arrivals);
        // same rule as k_p2g, so both kernels visit exactly the same particles
        if (cur.rb + r < cur.tm.run_len && !(q0.w > 0.f)) continue;
        const float mass = fabsf(q0.w);
        int bx, by, bz;
        float rx, ry, rz;
        base_rel(q0.x, P.inv_dx, bx, rx);
        base_rel(q0.y, P.inv_dx, by, ry);
        base_rel(q0.z, P.inv_dx, bz, rz);
        bx -= tx * 4; by -= ty * 4; bz -= tz * 4;
        if (!MPMB_CHK(V.cnt, (unsigned)bx < 4u && (unsigned)by < 4u && (unsigned)bz < 4u, 8, cur.slot, (bx & 255) | ((by & 255) << 8) | ((bz & 255) << 16), cur.rb + r)) continue;
        float wx[3], wy[3], wz[3];
        bspline_weights(rx, wx);
        bspline_weights(ry, wy);
        bspline_weights(rz, wz);
        // v = sum w g ; b = sum w g (x) (rel - node) = v (x) rel - [sum_i i S_i | sum_j j T_j | sum_k k R_k]
        // (src/transfer.cpp:888-904), evaluated slab by slab: ~250 FMA instead of 27*16.
        // every node value (v_x,v_y | v_z,m) as two pairs; the mass lane of the sums is never read
        const float2 wz0 = bc2(wz[0]), wz1 = bc2(wz[1]), wz2 = bc2(wz[2]), wz2x = bc2(2.0f * wz[2]);
        const float2 wy2[3] = {bc2(wy[0]), bc2(wy[1]), bc2(wy[2])}, wx2[3] = {bc2(wx[0]), bc2(wx[1]), bc2(wx[2])};
        const float2 wyj[3] = {wy2[0], wy2[1], bc2(2.0f * wy[2])}, wxi[3] = {wx2[0], wx2[1], bc2(2.0f * wx[2])};
        F4 V4 = f4_zero(), CX = f4_zero(), CY = f4_zero(), CZ = f4_zero();
#pragma unroll
        for (int i = 0; i < 3; i++) {
          F4 pi = f4_zero(), jy = f4_zero(), kz = f4_zero();
#pragma unroll
          for (int jn = 0; jn < 3; jn++) {
            const int row = ((bx + i) * 6 + (by + jn)) * 6 + bz;
            const F4 g0 = f4_load(sv[row]), g1 = f4_load(sv[row + 1]), g2 = f4_load(sv[row + 2]);
            const F4 a = f4_fma(wz2, g2, f4_fma(wz1, g1, f4_mul(wz0, g0)));
            const F4 c = f4_fma(wz2x, g2, f4_mul(wz1, g1));
            pi = f4_fma(wy2[jn], a, pi);
            kz = f4_fma(wy2[jn], c, kz);
            if (jn > 0) jy = f4_fma(wyj[jn], a, jy);
          }
          V4 = f4_fma(wx2[i], pi, V4);
          CY = f4_fma(wx2[i], jy, CY);
          CZ = f4_fma(wx2[i], kz, CZ);
          if (i > 0) CX = f4_fma(wxi[i], pi, CX);
        }
        const float3 v = make_float3(V4.lo.x, V4.lo.y, V4.hi.x), colx = make_float3(CX.lo.x, CX.lo.y, CX.hi.x),
                     coly = make_float3(CY.lo.x, CY.lo.y, CY.hi.x), colz = make_float3(CZ.lo.x, CZ.lo.y, CZ.hi.x);
        // the rest of the particle's row is read only now: nothing of it is live across the gather (registers)
        asm volatile("" ::: "memory");
        const float4 q4 = s_in[buf][1][r], q5 = s_in[buf][2][r], q6 = s_in[buf][3][r];
        const size_t o = s_out[buf][r < nrun ? sh + r : r + 8];
        if (!MPMB_CHK(V.cnt, o < (size_t)V.cap_particles && (int)o >= cur.tm.out_begin && (int)o < cur.tm.out_begin + cur.tm.run_len + cur.tm.arr_len, 7, cur.slot, o, r)) continue;
        const float vol = q6.z;
        const uint32_t tag = __float_as_uint(q6.w);
        const Material &mat = P.mats[tag >> TAG_ID_BITS];
        Mat3 B;
        B.m[0] = fmaf(v.x, rx, -colx.x); B.m[1] = fmaf(v.y, rx, -colx.y); B.m[2] = fmaf(v.z, rx, -colx.z);
        B.m[3] = fmaf(v.x, ry, -coly.x); B.m[4] = fmaf(v.y, ry, -coly.y); B.m[5] = fmaf(v.z, ry, -coly.z);
        B.m[6] = fmaf(v.x, rz, -colz.x); B.m[7] = fmaf(v.y, rz, -colz.y); B.m[8] = fmaf(v.z, rz, -colz.z);
        Mat3 cdg;  // cdg = I + (-4 inv_dx dt) b   (src/transfer.cpp:938-942)
#pragma unroll
        for (int k = 0; k < 9; k++) cdg.m[k] = fmaf(scale, B.m[k], (k % 4 == 0) ? 1.f : 0.f);
        Mat3 F;
        F.m[0] = q4.x; F.m[1] = q4.y; F.m[2] = q4.z; F.m[3] = q4.w; F.m[4] = q5.x; F.m[5] = q5.y; F.m[6] = q5.z; F.m[7] = q5.w; F.m[8] = q6.x;
        float ps = q6.y;
        Mat3 force, A;
        material_step<EXT_MATS>(mat, cdg, F, ps, vol, force);
        make_affine(force, B, mass, scale, A);
        float3 x = make_float3(fmaf(v.x, P.dt, q0.x), fmaf(v.y, P.dt, q0.y), fmaf(v.z, P.dt, q0.z));  // 951
        uint32_t key = make_key(P, x.x, x.y, x.z);
        if (P.clean_boundary && reference_deletes(P, x, v)) key = (uint32_t)(P.ntiles_total + SPECIAL_DEAD);
        if (!isfinite(x.x + x.y + x.z)) key = (uint32_t)(P.ntiles_total + SPECIAL_DEAD);
        // one contiguous, cell-sorted run per tile in the other buffer
        store_particle<STORE_B>(V.qn, o, x, key == (uint32_t)tile ? mass : -mass, v, A, F, ps, vol, tag, B);
        V.keys_next[o] = key;
        if (key == (uint32_t)tile) {
          my_stay++;
        } else if (key != (uint32_t)(P.ntiles_total + SPECIAL_DEAD)) {
          const int m = atomicAdd(&V.cnt->n_movers_next, 1);  // ~0.5 % of the particles per substep
          if (!MPMB_CHK(V.cnt, m < V.cap_particles, 9, m, key, 0)) continue;
          V.mover_dst_n[m] = key;
          V.mover_idx_n[m] = (uint32_t)o;
          MPMB_COUNT_ARRIVAL(V, P, key);  // the next ordering's arrival count of that tile
        }
      }
      if (my_stay) atomicAdd(&s_stay[sp], my_stay);
    }
    __syncthreads();  // everyone is done with `buf` before the prefetch after next overwrites it
    if (nxt.slot != cur.slot) {
      if (tid == 0) { V.stay_next[cur.tm.tile] = s_stay[sp]; s_stay[sp] = 0; }
      sp ^= 1;
      MPMB_TRACE_TILE(cur.tm.run_len + cur.tm.arr_len);
    }
    cur = nxt;
    buf ^= 1;
  }
  cp_async_wait_all();
  MPMB_TRACE_END(TRACE_G2P);
  // end of the substep: the lists and runs this kernel produced become the current ones — done by the last CTA to
  // finish (no separate 1-thread launch)
  if (commit) {
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      if (atomicAdd(&V.cnt->g2p_done, 1) == (int)gridDim.x - 1) {
        __threadfence();
        Counters *c = V.cnt;
        c->n_movers = atomicAdd(&c->n_movers_next, 0);
        c->n_movers_next = 0;
        c->n_store = c->n_alive;  // G2P wrote one row per binned particle
        c->xstep += 1;
        c->g2p_done = 0;
      }
    }
  }
}

// ------------------------------------------------------------------------------ CPIC rigid coupling (SURVEY §8f row 2)
// Replaces, for scenes with rigid bodies: update_rigid_page_map (src/mpm.cpp:1026-1076), rasterize_rigid_boundary and
// gather_cdf (src/rigid_transfer.cpp:18-113, 120-274) and the block_op_rigid branches of rasterize_optimized /
// resample_optimized (src/transfer.cpp:367-463, 706-835).  The rigid bodies themselves (RigidBody, its integrator, the
// rigid-rigid solver, articulation) belong to the reference's un-vendored core.  By default the host advances them: the engine
// takes poses and velocities (mpmb_set_rigid_state), applies the impulses of both transfers as apply_tmp_impulse /
// apply_tmp_velocity would (assumptions stated in include/mpmb.h) and hands the velocities back (mpmb_get_rigid_state).  With
// mpmb_set_rigid_motion the engine advances scripted and free bodies itself (k_rigid_contacts, k_rigid_advance below); the
// rigid-rigid solver and articulation are not built.
// Layout: RigidBoundaryParticles are NOT MPM particles here but a sample list (anchor offset + untransformed triangle + body);
// node colour data is two dense node arrays (a 64-bit key (distance bits, body) taken with atomicMin, the tags with atomicOr),
// cleared sample by sample; particle colour state is kept by particle id.  Tiles whose 4x4x8 page is a rigid page are
// skipped by k_g2p and processed by k_g2p_rigid; their arenas are rewritten by k_p2g_rigid after k_p2g (which still provides
// the output rows).  This is the reference's slow path too: simple kernels, shared-memory float atomics, no pipelining.
constexpr int RIGID_MAX = 12;                     // GridState::max_num_rigid_bodies (src/mpm_fwd.h:79)
constexpr uint32_t CDF_STATE_MASK = 0xAAAAAAAAu;  // state_mask (src/mpm.h:36)
constexpr uint32_t CDF_TAG_MASK = 0x00FFFFFFu;    // GridState::tag_mask
constexpr unsigned long long CDF_NO_KEY = ~0ull;

struct RigidDev {  // one body on the device
  float pos[3], rot[9], vel[3], ang[3], inv_mass, inv_inertia[9], fric[2];
  float acc[6];    // impulses of the running transfer: sum j, sum (p - pos) x j
};
struct RigidView {
  RigidDev *bodies;
  int n_bodies;
  int n_samples;
  const float *s_offset, *s_tri;
  const int *s_rigid;
  int *s_base;                     // packed base node of each sample's last rasterisation (-1: none), for the clear
  unsigned long long *node_key;    // (distance bits << 32) | (body + 1); CDF_NO_KEY = no rigid boundary near this node
  uint32_t *node_tags;             // GridState tag bits
  unsigned char *page;             // rigid_page_map over 4x4x8 blocks
  int nb[3];
  unsigned char *tile_flag;        // [slot]
  uint32_t *p_states;              // MPMParticle::states by particle id - id_base (persists)
  float4 *p_cdf;                   // (boundary_normal, boundary_distance) of this substep
  uint32_t *p_mark;                // (epoch << 1) | near_boundary_: p_cdf / near of a particle count only if its mark carries THIS substep's
                                   // epoch — gather_cdf then touches only the particles of rigid pages (no 8 M scattered zero-writes)
  uint32_t *epoch;                 // device word, advanced by k_cdf_clear once per substep (a graph replays it correctly)
  uint32_t id_base;
  int id_cap;
  float penalty, pushing_force;
};

__device__ __forceinline__ uint32_t cdf_word(const RigidView &R, size_t node) {  // GridState::states: tags | (body + 1) << 24
  const unsigned long long k = R.node_key[node];
  return (R.node_tags[node] & CDF_TAG_MASK) | (k == CDF_NO_KEY ? 0u : ((uint32_t)k & 0xffu) << 24);
}
__device__ __forceinline__ float cdf_dist_world(const RigidView &R, size_t node, float dx) {  // GridState::distance after line 77-78
  const unsigned long long k = R.node_key[node];
  return k == CDF_NO_KEY ? 0.f : __uint_as_float((uint32_t)(k >> 32)) * dx;
}
__device__ __forceinline__ bool cdf_compatible(uint32_t word, uint32_t pst) {  // src/transfer.cpp:416-420
  const uint32_t gs = word & CDF_TAG_MASK;
  const uint32_t mask = (gs & pst & CDF_STATE_MASK) >> 1;
  return (gs & mask) == (pst & mask);
}
__device__ __forceinline__ float3 rigid_to_world(const RigidDev &b, const float *l) {
  return make_float3(b.pos[0] + (b.rot[0] * l[0] + b.rot[3] * l[1] + b.rot[6] * l[2]), b.pos[1] + (b.rot[1] * l[0] + b.rot[4] * l[1] + b.rot[7] * l[2]),
                     b.pos[2] + (b.rot[2] * l[0] + b.rot[5] * l[1] + b.rot[8] * l[2]));
}
__device__ __forceinline__ float3 rigid_velocity_at(const RigidDev &b, float3 p) {  // velocity + angular_velocity x (p - position)
  const float dx = p.x - b.pos[0], dy = p.y - b.pos[1], dz = p.z - b.pos[2];
  return make_float3(b.vel[0] + (b.ang[1] * dz - b.ang[2] * dy), b.vel[1] + (b.ang[2] * dx - b.ang[0] * dz), b.vel[2] + (b.ang[0] * dy - b.ang[1] * dx));
}
// Per-thread impulse accumulator for ONE body at a time: every incompatible (particle, node) pair of a tile otherwise hits the
// same six shared floats (a 128-way contended CAS loop);
// a thread flushes only when the body changes and at the end of its rows.
struct ImpulseAcc {
  float a[6];
  int id;
  __device__ __forceinline__ void init() { id = -1; a[0] = a[1] = a[2] = a[3] = a[4] = a[5] = 0.f; }
  __device__ __forceinline__ void flush(float (*s_acc)[6]) {
    if (id >= 0) {
#pragma unroll
      for (int k = 0; k < 6; k++) if (a[k] != 0.f) atomicAdd(&s_acc[id][k], a[k]);
    }
    a[0] = a[1] = a[2] = a[3] = a[4] = a[5] = 0.f;
  }
  __device__ __forceinline__ void add(float (*s_acc)[6], int rid, const RigidDev &b, float3 j, float3 p) {
    if (rid != id) { flush(s_acc); id = rid; }
    const float dx = p.x - b.pos[0], dy = p.y - b.pos[1], dz = p.z - b.pos[2];
    a[0] += j.x; a[1] += j.y; a[2] += j.z;
    a[3] += dy * j.z - dz * j.y; a[4] += dz * j.x - dx * j.z; a[5] += dx * j.y - dy * j.x;
  }
};
// friction_project (src/mpm_fwd.h:25-57) against a moving base
__device__ __forceinline__ float3 friction_project_rel(float3 v, float3 base, float3 n, float friction) {
  const float3 r = friction_project0(make_float3(v.x - base.x, v.y - base.y, v.z - base.z), n, friction);
  return make_float3(r.x + base.x, r.y + base.y, r.z + base.z);
}
__device__ __forceinline__ int pack_base(int bx, int by, int bz) { return (bx << 20) | (by << 10) | bz; }   // node coordinates < 1024

// nodes of the previous rasterisation back to "no boundary"; thread 0 opens the substep's epoch (0 is never current)
__global__ void k_cdf_clear(RigidView R, Params P) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s == 0) {
    uint32_t e = (*R.epoch + 1u) & 0x7fffffffu;
    *R.epoch = e == 0u ? 1u : e;
  }
  if (s >= R.n_samples) return;
  const int pb = R.s_base[s];
  if (pb < 0) return;
  const int bx = pb >> 20, by = (pb >> 10) & 1023, bz = pb & 1023;
  for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) for (int c = 0; c < 3; c++) {
    const int i = bx + a, j = by + b, k = bz + c;
    if (i >= P.nnode[0] || j >= P.nnode[1] || k >= P.nnode[2]) continue;
    const size_t node = ((size_t)i * P.nnode[1] + j) * P.nnode[2] + k;
    R.node_key[node] = CDF_NO_KEY;
    R.node_tags[node] = 0u;
  }
}

// update_rigid_page_map + rasterize_rigid_boundary, one thread per RigidBoundaryParticle
__global__ void k_cdf_raster(RigidView R, Params P) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= R.n_samples) return;
  const int id = R.s_rigid[s];
  const RigidDev &B = R.bodies[id];
  const float3 pos = rigid_to_world(B, R.s_offset + 3 * s);   // align_with_rigid_body (src/boundary_particle.h:48-53)
  int bx, by, bz;
  float rr;
  base_rel(pos.x, P.inv_dx, bx, rr);
  base_rel(pos.y, P.inv_dx, by, rr);
  base_rel(pos.z, P.inv_dx, bz, rr);
  if (bx < 0 || by < 0 || bz < 0 || bx + 2 >= P.nnode[0] || by + 2 >= P.nnode[1] || bz + 2 >= P.nnode[2]) { R.s_base[s] = -1; return; }
  R.s_base[s] = pack_base(bx, by, bz);
  // page of the block the particle is sorted into, and (src/mpm.cpp:1062: the range test is on the OFFSET) its {0,1}^3 upper neighbours
  for (int i = 0; i < 2; i++) for (int j = 0; j < 2; j++) for (int k = 0; k < 2; k++) {
    const int x = (bx >> 2) + i, y = (by >> 2) + j, z = (bz >> 3) + k;
    if (x < R.nb[0] && y < R.nb[1] && z < R.nb[2]) R.page[((size_t)x * R.nb[1] + y) * R.nb[2] + z] = 1;
  }
  const float3 v0 = rigid_to_world(B, R.s_tri + 9 * s), v1 = rigid_to_world(B, R.s_tri + 9 * s + 3), v2 = rigid_to_world(B, R.s_tri + 9 * s + 6);
  // world_to_element: [v1 - v0, v2 - v0, n]^-1
  Mat3 M, Mi;
  const float e1[3] = {v1.x - v0.x, v1.y - v0.y, v1.z - v0.z}, e2[3] = {v2.x - v0.x, v2.y - v0.y, v2.z - v0.z};
  float n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
  const float nl = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  for (int k = 0; k < 3; k++) { n[k] /= nl; M(k, 0) = e1[k]; M(k, 1) = e2[k]; M(k, 2) = n[k]; }
  {
    const float d = det3(M), idet = 1.0f / d;
    Mi(0, 0) = (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) * idet; Mi(0, 1) = (M(0, 2) * M(2, 1) - M(0, 1) * M(2, 2)) * idet; Mi(0, 2) = (M(0, 1) * M(1, 2) - M(0, 2) * M(1, 1)) * idet;
    Mi(1, 0) = (M(1, 2) * M(2, 0) - M(1, 0) * M(2, 2)) * idet; Mi(1, 1) = (M(0, 0) * M(2, 2) - M(0, 2) * M(2, 0)) * idet; Mi(1, 2) = (M(0, 2) * M(1, 0) - M(0, 0) * M(1, 2)) * idet;
    Mi(2, 0) = (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0)) * idet; Mi(2, 1) = (M(0, 1) * M(2, 0) - M(0, 0) * M(2, 1)) * idet; Mi(2, 2) = (M(0, 0) * M(1, 1) - M(0, 1) * M(1, 0)) * idet;
  }
  for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) for (int c = 0; c < 3; c++) {
    const int i = bx + a, j = by + b, k = bz + c;
    const float d0 = (float)i * P.dx - v0.x, d1 = (float)j * P.dx - v0.y, d2 = (float)k * P.dx - v0.z;
    const float c0 = Mi(0, 0) * d0 + Mi(0, 1) * d1 + Mi(0, 2) * d2, c1 = Mi(1, 0) * d0 + Mi(1, 1) * d1 + Mi(1, 2) * d2, c2 = Mi(2, 0) * d0 + Mi(2, 1) * d1 + Mi(2, 2) * d2;
    if (!(0.f <= c0 && 0.f <= c1 && c0 + c1 <= 1.f)) continue;                          // src/rigid_transfer.cpp:50-53
    const float dist = fabsf(c2) * P.inv_dx;                                              // 43, 60
    const size_t node = ((size_t)i * P.nnode[1] + j) * P.nnode[2] + k;
    // 65-69 under the node's lock: the nearest body wins (a tie goes to the smaller id here, to whoever came first there)
    atomicMin(&R.node_key[node], ((unsigned long long)__float_as_uint(dist) << 32) | (unsigned long long)(id + 1));
    atomicOr(&R.node_tags[node], (uint32_t)(2 + (c2 < 0.f ? 1 : 0)) << (id * 2));     // 73-74
  }
}

__global__ void k_rigid_tile_flags(View V, Params P, RigidView R) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= V.cnt->n_tiles) return;
  const TileMeta tm = V.meta[slot];
  MPMB_TILE_XYZ(P, tm, tx, ty, tz);
  R.tile_flag[slot] = R.page[((size_t)tx * R.nb[1] + ty) * R.nb[2] + (tz >> 1)];   // tile (4x4x4 nodes) -> page (4x4x8 nodes)
}

__device__ __forceinline__ float det4(const float *m) {  // m[c*4+r]
  float det = 0.f;
#pragma unroll
  for (int c = 0; c < 4; c++) {
    int cc[3], k = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) if (j != c) cc[k++] = j;
#define A4(r, c_) m[(c_) * 4 + (r)]
    const float minor = A4(1, cc[0]) * (A4(2, cc[1]) * A4(3, cc[2]) - A4(2, cc[2]) * A4(3, cc[1])) - A4(1, cc[1]) * (A4(2, cc[0]) * A4(3, cc[2]) - A4(2, cc[2]) * A4(3, cc[0])) +
                        A4(1, cc[2]) * (A4(2, cc[0]) * A4(3, cc[1]) - A4(2, cc[1]) * A4(3, cc[0]));
    det += ((c & 1) ? -1.f : 1.f) * A4(0, c) * minor;
#undef A4
  }
  return det;
}

// gather_cdf (src/rigid_transfer.cpp:120-274): one thread per storage row that holds a live particle
__global__ void __launch_bounds__(128) k_gather_cdf(View V, Params P, RigidView R) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= V.cnt->n_store) return;
  if (V.keys[row] >= (uint32_t)P.ntiles_total) return;   // dead or migrating
  const float4 q0 = V.q[0][row];
  const float X = __fmul_rn(q0.x, P.inv_dx), Y = __fmul_rn(q0.y, P.inv_dx), Z = __fmul_rn(q0.z, P.inv_dx);
  {  // 142-146: the page of the particle's CELL.  Outside: boundary_distance = 0, normal = 0, near_boundary_ = false (138-140)
     // and the colours untouched — expressed by NOT renewing the particle's mark
    const int cx = (int)X >> 2, cy = (int)Y >> 2, cz = (int)Z >> 3;
    if (cx < 0 || cy < 0 || cz < 0 || cx >= R.nb[0] || cy >= R.nb[1] || cz >= R.nb[2] || !R.page[((size_t)cx * R.nb[1] + cy) * R.nb[2] + cz]) return;
  }
  const uint32_t id = (__float_as_uint(V.q[6][row].w) & TAG_ID_MASK) - R.id_base;
  if (id >= (uint32_t)R.id_cap) { atomicOr(&V.cnt->error, DEVERR_BAD_INPUT); return; }
  const uint32_t epoch = *R.epoch;
  R.p_cdf[id] = make_float4(0.f, 0.f, 0.f, 0.f);
  R.p_mark[id] = epoch << 1;
  int bx, by, bz;
  float rx, ry, rz;
  base_rel(q0.x, P.inv_dx, bx, rx);
  base_rel(q0.y, P.inv_dx, by, ry);
  base_rel(q0.z, P.inv_dx, bz, rz);
  float wx[3], wy[3], wz[3];
  bspline_weights(rx, wx);
  bspline_weights(ry, wy);
  bspline_weights(rz, wz);
  uint32_t pst = R.p_states[id];
  uint32_t words[27];
  uint32_t all_b = 0;
  for (int n = 0; n < 27; n++) {
    const size_t node = ((size_t)(bx + n / 9) * P.nnode[1] + (by + (n / 3) % 3)) * P.nnode[2] + (bz + n % 3);
    words[n] = cdf_word(R, node);
    all_b |= words[n] & CDF_TAG_MASK & CDF_STATE_MASK;                                   // 155-159
  }
  pst &= (all_b + (all_b >> 1));                                                         // 162
  uint32_t to_add = all_b & ~pst;                                                        // 164
  while (to_add) {
    const uint32_t bit = to_add & (0u - to_add);
    to_add ^= bit;
    float wd0 = 0.f, wd1 = 0.f;
    for (int n = 0; n < 27; n++) {
      if ((words[n] >> 24) == 0u) continue;                                              // 182-184
      const size_t node = ((size_t)(bx + n / 9) * P.nnode[1] + (by + (n / 3) % 3)) * P.nnode[2] + (bz + n % 3);
      const float d = cdf_dist_world(R, node, P.dx) * P.inv_dx;
      const float w = (wx[n / 9] * wy[(n / 3) % 3]) * wz[n % 3];
      if (words[n] & CDF_TAG_MASK & bit) { if (words[n] & (bit >> 1)) wd1 += d * w; else wd0 += d * w; }   // 195-198
    }
    if (wd0 + wd1 > 1e-7f) pst |= bit | ((bit >> 1) * (uint32_t)(wd0 < wd1));           // 200-205
  }
  R.p_states[id] = pst;
  if (pst == 0u) return;
  float XtX[16], XtY[4];
  for (int k = 0; k < 16; k++) XtX[k] = 0.f;
  for (int k = 0; k < 4; k++) XtY[k] = 0.f;
  for (int n = 0; n < 27; n++) {
    if ((words[n] >> 24) == 0u) continue;                                                // 217-219
    const uint32_t gs = words[n] & CDF_TAG_MASK;
    if (gs == 0u) continue;
    const uint32_t mask = (gs & pst & CDF_STATE_MASK) >> 1;
    float sgn;
    if ((gs & mask) == (pst & mask)) sgn = 1.f;                                          // 232-236: same colour
    else {
      const uint32_t diff = (gs & mask) ^ (pst & mask);                                  // 239-243: exactly one colour differs
      if (diff > 0u && (diff & (diff - 1u)) == 0u) sgn = -1.f; else continue;
    }
    const int a = n / 9, b = (n / 3) % 3, c = n % 3;
    const size_t node = ((size_t)(bx + a) * P.nnode[1] + (by + b)) * P.nnode[2] + (bz + c);
    const float d = cdf_dist_world(R, node, P.dx) * P.inv_dx;
    const float w = (wx[a] * wy[b]) * wz[c];
    const float xp[4] = {-(rx - (float)a), -(ry - (float)b), -(rz - (float)c), 1.f};   // (-dpos, 1)
    for (int i = 0; i < 4; i++) {
      for (int j = 0; j < 4; j++) XtX[j * 4 + i] += xp[i] * xp[j] * w;
      XtY[i] += sgn * (d * xp[i]) * w;                                                   // (-d dpos, d) resp. its negative
    }
  }
  if (fabsf(det4(XtX)) > 1e-4f) {                                                        // 251: mpm_reconstruction_guard<3>
    // inversed(XtX) * XtY by Gaussian elimination with partial pivoting
    float A[4][5];
    for (int r = 0; r < 4; r++) { for (int c = 0; c < 4; c++) A[r][c] = XtX[c * 4 + r]; A[r][4] = XtY[r]; }
    for (int c = 0; c < 4; c++) {
      int pv = c;
      for (int r = c + 1; r < 4; r++) if (fabsf(A[r][c]) > fabsf(A[pv][c])) pv = r;
      for (int k = 0; k < 5; k++) { const float t = A[c][k]; A[c][k] = A[pv][k]; A[pv][k] = t; }
      for (int r = c + 1; r < 4; r++) { const float f = A[r][c] / A[c][c]; for (int k = c; k < 5; k++) A[r][k] -= f * A[c][k]; }
    }
    float sol[4];
    for (int r = 3; r >= 0; r--) { float sum = A[r][4]; for (int c = r + 1; c < 4; c++) sum -= A[r][c] * sol[c]; sol[r] = sum / A[r][r]; }
    R.p_mark[id] = (epoch << 1) | 1u;
    const float l2 = sol[0] * sol[0] + sol[1] * sol[1] + sol[2] * sol[2];
    float4 o = make_float4(0.f, 0.f, 0.f, sol[3] * P.dx);
    if (l2 > 1e-4f) { const float il = 1.0f / sqrtf(l2); o.x = sol[0] * il; o.y = sol[1] * il; o.z = sol[2] * il; }
    R.p_cdf[id] = o;
  }
}

// Node colour words of a tile's 6x6x6 stencil block into shared memory
__device__ __forceinline__ void load_tile_words(const RigidView &R, const Params &P, int tx, int ty, int tz, uint32_t *s_word) {
  for (int n = threadIdx.x; n < ARENA; n += blockDim.x) {
    const int i = tx * 4 + n / 36, j = ty * 4 + (n / 6) % 6, k = tz * 4 + n % 6;
    s_word[n] = (i < P.nnode[0] && j < P.nnode[1] && k < P.nnode[2]) ? cdf_word(R, ((size_t)i * P.nnode[1] + j) * P.nnode[2] + k) : 0u;
  }
}

// block_op_rigid of rasterize_optimized (src/transfer.cpp:367-463) for the tiles of rigid pages: rewrites the tile's arena
// (k_p2g ran on it first and provided the output rows).  One CTA per tile, one thread per row, shared float atomics.
// Owned tiles only (slots below n_tiles; a ghost slot holds a neighbour's partial sums), those of `part` (tile_in_part).
__global__ void __launch_bounds__(128) k_p2g_rigid(View V, Params P, RigidView R, int part) {
  __shared__ float s_arena[4][ARENA];
  __shared__ uint32_t s_word[ARENA];
  __shared__ float s_acc[RIGID_MAX][6];
  const int tid = threadIdx.x;
  const int n_tiles = V.cnt->n_tiles;
  const uint32_t epoch = *R.epoch;
    for (int slot = blockIdx.x; slot < n_tiles; slot += gridDim.x) {
    if (!R.tile_flag[slot]) continue;
    const TileMeta tm = V.meta[slot];
    if (!tile_in_part(P, tm.tile, part)) continue;
    MPMB_TILE_XYZ(P, tm, tx, ty, tz);
    for (int n = tid; n < ARENA; n += blockDim.x) { s_arena[0][n] = 0.f; s_arena[1][n] = 0.f; s_arena[2][n] = 0.f; s_arena[3][n] = 0.f; }
    for (int n = tid; n < RIGID_MAX * 6; n += blockDim.x) (&s_acc[0][0])[n] = 0.f;
    load_tile_words(R, P, tx, ty, tz, s_word);
    __syncthreads();
    const int nrow = tm.run_len + tm.arr_len;
    // A tile's run is cell-sorted, so neighbouring rows scatter to the same nodes: lanes take rows a large odd stride apart
    // (a bijection of [0, nrow)), which cuts the retries of the shared float atomics (CAS loops)
    const int stride = (nrow % 61) ? 61 : ((nrow % 67) ? 67 : 1);
    ImpulseAcc imp;
    imp.init();
    for (int idx = tid; idx < nrow; idx += blockDim.x) {
      const int g = (int)(((long long)idx * stride) % nrow);
      const uint32_t row = g < tm.run_len ? (uint32_t)(tm.run_begin + g) : V.arrivals_sorted[tm.arr_off + (g - tm.run_len)];
      const float4 a0 = V.q[0][row];
      if (g < tm.run_len && !(a0.w > 0.f)) continue;   // hole
      const float4 a1 = V.q[1][row], a2 = V.q[2][row], a3 = V.q[3][row];
      const float4 b0 = V.q[7][row], b1 = V.q[8][row], b2 = V.q[9][row];
      const float mass = fabsf(a0.w);
      const uint32_t id = (__float_as_uint(V.q[6][row].w) & TAG_ID_MASK) - R.id_base;
      const uint32_t pst = id < (uint32_t)R.id_cap ? R.p_states[id] : 0u;
      const bool fresh = id < (uint32_t)R.id_cap && (R.p_mark[id] >> 1) == epoch;   // gather_cdf saw this particle in this substep
      const float4 pc = fresh ? R.p_cdf[id] : make_float4(0.f, 0.f, 0.f, 0.f);
      float3 v = make_float3(a1.x, a1.y, a1.z);
      if (P.particle_gravity) { v.x += P.gdt[0]; v.y += P.gdt[1]; v.z += P.gdt[2]; }
      int bx, by, bz;
      float rx, ry, rz;
      base_rel(a0.x, P.inv_dx, bx, rx);
      base_rel(a0.y, P.inv_dx, by, ry);
      base_rel(a0.z, P.inv_dx, bz, rz);
      const int lx = bx - tx * 4, ly = by - ty * 4, lz = bz - tz * 4;
      if ((unsigned)lx >= 4u || (unsigned)ly >= 4u || (unsigned)lz >= 4u) continue;
      float wx[3], wy[3], wz[3], gx[3], gy[3], gz[3];
      bspline_weights(rx, wx); bspline_weights(ry, wy); bspline_weights(rz, wz);
      // dw of MPMKernel<3,2> (src/kernel.h:133-134), in world units (shuffle(): * inv_delta_x)
      { const float f = rx - 0.5f; gx[0] = (f - 1.0f) * P.inv_dx; gx[1] = (-2.0f * f + 1.0f) * P.inv_dx; gx[2] = f * P.inv_dx; }
      { const float f = ry - 0.5f; gy[0] = (f - 1.0f) * P.inv_dx; gy[1] = (-2.0f * f + 1.0f) * P.inv_dx; gy[2] = f * P.inv_dx; }
      { const float f = rz - 0.5f; gz[0] = (f - 1.0f) * P.inv_dx; gz[1] = (-2.0f * f + 1.0f) * P.inv_dx; gz[2] = f * P.inv_dx; }
      const float A[9] = {a1.w, a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
      const float bb[9] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w, b2.x};
      // dt * calculate_force() back out of the cached affine matrix: A = force * S + apic_b * 4 m, S = -4 dt / dx
      float tf[9];
      for (int k = 0; k < 9; k++) tf[k] = (A[k] - bb[k] * (4.0f * mass)) * (-0.25f * P.dx);
      for (int n = 0; n < 27; n++) {
        const int a = n / 9, b = (n / 3) % 3, c = n % 3;
        const int ln = ((lx + a) * 6 + (ly + b)) * 6 + (lz + c);
        const float w = (wx[a] * wy[b]) * wz[c];
        const float dpx = rx - (float)a, dpy = ry - (float)b, dpz = rz - (float)c;
        const uint32_t word = s_word[ln];
        if (!cdf_compatible(word, pst)) {   // different colour: project against the body instead of writing to the grid (420-446)
          const int rid = (int)(word >> 24) - 1;
          if (rid < 0 || rid >= R.n_bodies) continue;
          const RigidDev &B = R.bodies[rid];
          const float3 gp = make_float3(P.dx * (float)(bx + a), P.dx * (float)(by + b), P.dx * (float)(bz + c));
          const float3 rv = rigid_velocity_at(B, gp);
          const float3 pr = friction_project_rel(v, rv, make_float3(pc.x, pc.y, pc.z), B.fric[(pst >> (2 * rid)) & 1u]);
          const float dwx = (gx[a] * wy[b]) * wz[c], dwy = (wx[a] * gy[b]) * wz[c], dwz = (wx[a] * wy[b]) * gz[c];
          const float3 j = make_float3(mass * w * (v.x - pr.x) + (tf[0] * dwx + tf[3] * dwy + tf[6] * dwz), mass * w * (v.y - pr.y) + (tf[1] * dwx + tf[4] * dwy + tf[7] * dwz),
                                       mass * w * (v.z - pr.z) + (tf[2] * dwx + tf[5] * dwy + tf[8] * dwz));
          imp.add(s_acc, rid, B, j, gp);
          continue;
        }
        atomicAdd(&s_arena[0][ln], w * (mass * v.x + (A[0] * dpx + A[3] * dpy + A[6] * dpz)));   // 451-459
        atomicAdd(&s_arena[1][ln], w * (mass * v.y + (A[1] * dpx + A[4] * dpy + A[7] * dpz)));
        atomicAdd(&s_arena[2][ln], w * (mass * v.z + (A[2] * dpx + A[5] * dpy + A[8] * dpz)));
        atomicAdd(&s_arena[3][ln], w * mass);
      }
    }
    imp.flush(s_acc);
    __syncthreads();
    float4 *out = V.arena + (size_t)slot * ARENA;
    for (int n = tid; n < ARENA; n += blockDim.x) out[n] = make_float4(s_arena[0][n], s_arena[1][n], s_arena[2][n], s_arena[3][n]);
    for (int n = tid; n < RIGID_MAX * 6; n += blockDim.x) {
      const float a = (&s_acc[0][0])[n];
      if (a != 0.f) atomicAdd(&R.bodies[n / 6].acc[n % 6], a);
    }
    __syncthreads();
  }
}

// apply_tmp_velocity (src/transfer.cpp:578-580, 967-969): velocity += inv_mass * sum j, angular_velocity += Iw^-1 * sum (p - c) x j
__global__ void k_rigid_apply(RigidView R) {
  const int b = threadIdx.x;
  if (b >= R.n_bodies) return;
  RigidDev &B = R.bodies[b];
  for (int k = 0; k < 3; k++) {
    B.vel[k] += B.inv_mass * B.acc[k];
    B.ang[k] += B.inv_inertia[k] * B.acc[3] + B.inv_inertia[3 + k] * B.acc[4] + B.inv_inertia[6 + k] * B.acc[5];
  }
  for (int k = 0; k < 6; k++) B.acc[k] = 0.f;
}

// z-slab ranks: each rank's transfers sum only its own particles' impulses.  Every rank sums the partials of all `world`
// ranks (RIGID_IMPULSE_FLOATS floats each, rank r's at parts + r * stride floats) in rank order 0..world-1 and applies the
// sum as k_rigid_apply does, so the bodies stay bit-identical on every rank.  One thread per body.
constexpr int RIGID_IMPULSE_FLOATS = RIGID_MAX * 6;
__device__ __forceinline__ void rigid_sum_apply(RigidView R, const float *parts, size_t stride, int world) {
  const int b = threadIdx.x;
  if (b >= R.n_bodies) return;
  float s[6];
  for (int k = 0; k < 6; k++) s[k] = parts[b * 6 + k];
  for (int w = 1; w < world; w++)
    for (int k = 0; k < 6; k++) s[k] += parts[(size_t)w * stride + b * 6 + k];
  RigidDev &B = R.bodies[b];
  for (int k = 0; k < 3; k++) {
    B.vel[k] += B.inv_mass * s[k];
    B.ang[k] += B.inv_inertia[k] * s[3] + B.inv_inertia[3 + k] * s[4] + B.inv_inertia[6 + k] * s[5];
  }
  for (int k = 0; k < 6; k++) B.acc[k] = 0.f;
}
// this rank's partial sums of the running transfer into out[RIGID_IMPULSE_FLOATS]
__global__ void k_rigid_impulse_pack(RigidView R, float *out) {
  for (int n = threadIdx.x; n < RIGID_IMPULSE_FLOATS; n += blockDim.x) out[n] = R.bodies[n / 6].acc[n % 6];
}
__global__ void k_rigid_impulse_apply(RigidView R, const float *parts, int world) { rigid_sum_apply(R, parts, RIGID_IMPULSE_FLOATS, world); }

// Bodies advanced on the device (mpmb_set_rigid_motion): advect_rigid_bodies (src/mpm_rigid_body.cpp:273-287) and
// rigid_body_levelset_collision (:347-384) with the arithmetic of HostRigidBody.advect / levelset_collision
// (taichi_mpm_b200/rigid.py) step for step, in fp64 on a master state per body; RigidDev gets the fp32 copy the transfers read.
struct RigidMaster {
  double pos[3], rot[9], vel[3], ang[3];   // rot column-major
  double mass, inv_mass, inv_inertia_body[9], axis[3], lin_damp, ang_damp, restitution;
  int scripted_pos, scripted_rot;
};
constexpr int SCRIPT_STRIDE = 18;          // script entry of one body: position, rotation, velocity, angular velocity
constexpr int CONTACT_STRIDE = 7;          // contact of one boundary sample: world position, phi, unit gradient of phi
struct MotionView {
  RigidMaster *m;                          // [RIGID_MAX]
  const double *script;                    // [entry][n_bodies][SCRIPT_STRIDE]
  int *cursor;                             // next script entry (device word: replayed graphs advance it)
  const int *s_order;                      // sample indices grouped by body, in sample order within a body
  int s_begin[RIGID_MAX + 1];              // body b owns s_order[s_begin[b] .. s_begin[b + 1])
  double *contact;                         // [sample][CONTACT_STRIDE]: world position, phi, unit gradient of phi
  int collide;                             // the level-set collision runs in this substep (asked for and a level set is set)
};

__device__ __forceinline__ bool motion_collides(const RigidMaster &B) {   // levelset_collision skips fully scripted bodies
  if (B.inv_mass != 0.0) return true;
  for (int k = 0; k < 9; k++) if (B.inv_inertia_body[k] != 0.0) return true;
  return false;
}
// R * A * R^T, all column-major
__device__ __forceinline__ void rot_conj(const double *R, const double *A, double *out) {
  double T[9];
  for (int c = 0; c < 3; c++)
    for (int r = 0; r < 3; r++) T[c * 3 + r] = R[r] * A[c * 3] + R[3 + r] * A[c * 3 + 1] + R[6 + r] * A[c * 3 + 2];
  for (int c = 0; c < 3; c++)
    for (int r = 0; r < 3; r++) out[c * 3 + r] = T[r] * R[c] + T[3 + r] * R[3 + c] + T[6 + r] * R[6 + c];
}
__device__ __forceinline__ void mat3_vec(const double *M, const double *v, double *out) {
  for (int r = 0; r < 3; r++) out[r] = M[r] * v[0] + M[3 + r] * v[1] + M[6 + r] * v[2];
}
__device__ __forceinline__ void cross3(const double *a, const double *b, double *out) {
  out[0] = a[1] * b[2] - a[2] * b[1]; out[1] = a[2] * b[0] - a[0] * b[2]; out[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
__device__ __forceinline__ void enforce_axis(RigidMaster &B) {   // enforce_angular_velocity_parallel_to
  if (fmax(fabs(B.axis[0]), fmax(fabs(B.axis[1]), fabs(B.axis[2]))) > 0.1) {
    const double l = sqrt(dot3(B.axis, B.axis));
    const double a[3] = {B.axis[0] / l, B.axis[1] / l, B.axis[2] / l};
    const double p = dot3(a, B.ang);
    for (int k = 0; k < 3; k++) B.ang[k] = a[k] * p;
  }
}

// phi and its normalised central-difference gradient (eps = 0.25 grid units) at every boundary sample of a colliding body
__global__ void k_rigid_contacts(RigidView R, MotionView M, Params P, const float4 *sdf4) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= R.n_samples) return;
  const RigidMaster &B = M.m[R.s_rigid[s]];
  if (!motion_collides(B)) return;
  const float *o = R.s_offset + 3 * s;
  double *c = M.contact + CONTACT_STRIDE * (size_t)s;
  double X[3];
  for (int r = 0; r < 3; r++) {
    c[r] = B.pos[r] + (B.rot[r] * (double)o[0] + B.rot[3 + r] * (double)o[1] + B.rot[6 + r] * (double)o[2]);
    X[r] = c[r] / (double)P.dx;
  }
  c[3] = sdf_phi_trilinear(sdf4, P, X);
  const double eps = 0.25;
  double g[3];
  for (int a = 0; a < 3; a++) {
    double Xp[3] = {X[0], X[1], X[2]}, Xm[3] = {X[0], X[1], X[2]};
    Xp[a] += eps;
    Xm[a] -= eps;
    g[a] = (sdf_phi_trilinear(sdf4, P, Xp) - sdf_phi_trilinear(sdf4, P, Xm)) / (2 * eps);
  }
  const double n = fmax(sqrt(dot3(g, g)), 1e-12);
  for (int a = 0; a < 3; a++) c[4 + a] = g[a] / n;
}

// one thread per body: the level-set impulses in sample order (the reference's loop is order dependent), then the advance
__global__ void k_rigid_advance(RigidView R, MotionView M, Params P, float3 gravity) {
  const int b = threadIdx.x;
  const int entry = *M.cursor;
  __syncthreads();
  if (b == 0) *M.cursor = entry + 1;
  if (b < 1 || b >= R.n_bodies) return;   // body 0 is the background body
  RigidMaster &B = M.m[b];
  RigidDev &D = R.bodies[b];
  const double dt = (double)P.dt;
  for (int k = 0; k < 3; k++) { B.vel[k] = (double)D.vel[k]; B.ang[k] = (double)D.ang[k]; }   // what the transfers left
  if (M.collide && motion_collides(B)) {
    double Iw[9];
    rot_conj(B.rot, B.inv_inertia_body, Iw);
    const double f0 = (double)D.fric[0];
    auto contribution = [&](const double *r0, const double *n) {   // 1/m + n . ((I^-1 (r0 x n)) x r0)
      double t[3], u[3], w[3];
      cross3(r0, n, t); mat3_vec(Iw, t, u); cross3(u, r0, w);
      return B.inv_mass + dot3(n, w);
    };
    auto velocity_at = [&](const double *r0, double *v) { double t[3]; cross3(B.ang, r0, t); for (int k = 0; k < 3; k++) v[k] = B.vel[k] + t[k]; };
    auto apply_impulse = [&](const double *j, const double *r0) {
      double t[3], u[3];
      cross3(r0, j, t); mat3_vec(Iw, t, u);
      for (int k = 0; k < 3; k++) { B.vel[k] += B.inv_mass * j[k]; B.ang[k] += u[k]; }
    };
    for (int i = M.s_begin[b]; i < M.s_begin[b + 1]; i++) {
      const double *c = M.contact + CONTACT_STRIDE * (size_t)M.s_order[i];
      if (!(c[3] < 0.0)) continue;
      const double r0[3] = {c[0] - B.pos[0], c[1] - B.pos[1], c[2] - B.pos[2]};
      const double *g = c + 4;
      double v[3];
      velocity_at(r0, v);
      const double J = -((1.0 + B.restitution) * dot3(g, v)) / contribution(r0, g);
      if (J < 0.0) continue;
      const double jn[3] = {J * g[0], J * g[1], J * g[2]};
      apply_impulse(jn, r0);
      velocity_at(r0, v);
      const double vn = dot3(g, v);
      double tao[3] = {v[0] - g[0] * vn, v[1] - g[1] * vn, v[2] - g[2] * vn};
      if (fmax(fabs(tao[0]), fmax(fabs(tao[1]), fabs(tao[2]))) > 1e-7) {
        const double l = sqrt(dot3(tao, tao));
        for (int k = 0; k < 3; k++) tao[k] /= l;
        const double j = fmin(fmax(-dot3(v, tao) / contribution(r0, tao), -f0 * J), f0 * J);
        const double jt[3] = {j * tao[0], j * tao[1], j * tao[2]};
        apply_impulse(jt, r0);
      }
    }
  }
  enforce_axis(B);
  const double *T = M.script ? M.script + ((size_t)entry * R.n_bodies + b) * SCRIPT_STRIDE : nullptr;
  if (B.scripted_pos) {
    for (int k = 0; k < 3; k++) { B.pos[k] = T[k]; B.vel[k] = T[12 + k]; }
  } else {
    const double d = exp(-B.lin_damp * dt);
    for (int k = 0; k < 3; k++) { B.vel[k] *= d; B.pos[k] = B.pos[k] + B.vel[k] * dt; }
  }
  if (B.scripted_rot) {
    for (int k = 0; k < 9; k++) B.rot[k] = T[3 + k];
    for (int k = 0; k < 3; k++) B.ang[k] = T[15 + k];
  } else {
    const double d = exp(-B.ang_damp * dt);
    for (int k = 0; k < 3; k++) B.ang[k] *= d;
    const double w[3] = {B.ang[0] * dt, B.ang[1] * dt, B.ang[2] * dt};
    const double a = sqrt(dot3(w, w));
    if (a >= 1e-12) {   // exponential map: I + sin(a) K + (1 - cos(a)) K^2, K = [w / a]x
      const double k0 = w[0] / a, k1 = w[1] / a, k2 = w[2] / a;
      const double K[9] = {0, k2, -k1, -k2, 0, k0, k1, -k0, 0};   // column-major
      double K2[9], E[9], Rn[9];
      for (int c = 0; c < 3; c++)
        for (int r = 0; r < 3; r++) K2[c * 3 + r] = K[r] * K[c * 3] + K[3 + r] * K[c * 3 + 1] + K[6 + r] * K[c * 3 + 2];
      const double sa = sin(a), ca = 1.0 - cos(a);
      for (int k = 0; k < 9; k++) E[k] = (k % 4 == 0 ? 1.0 : 0.0) + sa * K[k] + ca * K2[k];
      for (int c = 0; c < 3; c++)
        for (int r = 0; r < 3; r++) Rn[c * 3 + r] = E[r] * B.rot[c * 3] + E[3 + r] * B.rot[c * 3 + 1] + E[6 + r] * B.rot[c * 3 + 2];
      for (int k = 0; k < 9; k++) B.rot[k] = Rn[k];
    }
  }
  const double gv[3] = {(double)gravity.x, (double)gravity.y, (double)gravity.z};
  for (int k = 0; k < 3; k++) B.vel[k] = B.vel[k] + gv[k] * (B.mass * dt) * B.inv_mass;   // apply_impulse(g m dt, position)
  enforce_axis(B);
  double Iw[9];
  rot_conj(B.rot, B.inv_inertia_body, Iw);
  for (int k = 0; k < 3; k++) { D.pos[k] = (float)B.pos[k]; D.vel[k] = (float)B.vel[k]; D.ang[k] = (float)B.ang[k]; }
  for (int k = 0; k < 9; k++) { D.rot[k] = (float)B.rot[k]; D.inv_inertia[k] = (float)Iw[k]; }
}

// block_op_rigid of resample_optimized (src/transfer.cpp:706-835) + what k_g2p does for the ordering (output rows, keys,
// movers, stay counts), for the tiles of rigid pages.  Launched BEFORE k_g2p, which commits the substep.  Owned tiles of
// `part` only, as k_p2g_rigid.
__global__ void __launch_bounds__(128) k_g2p_rigid(View V, Params P, RigidView R, int part) {
  __shared__ float4 s_vel[ARENA];
  __shared__ int s_nb[27];
  __shared__ uint32_t s_word[ARENA];
  __shared__ float s_acc[RIGID_MAX][6];
  __shared__ int s_stay;
  const int tid = threadIdx.x;
  const int n_tiles = V.cnt->n_tiles;
  const float scale = -4.0f * P.inv_dx * P.dt;
  const uint32_t epoch = *R.epoch;
  for (int slot = blockIdx.x; slot < n_tiles; slot += gridDim.x) {
    if (!R.tile_flag[slot]) continue;
    const TileMeta tm = V.meta[slot];
    const int tile = tm.tile;
    if (!tile_in_part(P, tile, part)) continue;
    MPMB_TILE_XYZ(P, tm, tx, ty, tz);
    if (tid < 27) s_nb[tid] = neighbour_slot(V, P, slot, tx, ty, tz, tid);
    __syncthreads();
    build_node_block<128>(V, P, tx, ty, tz, s_nb, s_vel);
    for (int n = tid; n < RIGID_MAX * 6; n += blockDim.x) (&s_acc[0][0])[n] = 0.f;
    load_tile_words(R, P, tx, ty, tz, s_word);
    if (tid == 0) s_stay = 0;
    __syncthreads();
    const int nrow = tm.run_len + tm.arr_len;
    int my_stay = 0;
    ImpulseAcc imp;
    imp.init();
    for (int g = tid; g < nrow; g += blockDim.x) {
      const uint32_t row = g < tm.run_len ? (uint32_t)(tm.run_begin + g) : V.arrivals_sorted[tm.arr_off + (g - tm.run_len)];
      const float4 q0 = V.q[0][row];
      if (g < tm.run_len && !(q0.w > 0.f)) continue;   // hole
      const float mass = fabsf(q0.w);
      const float4 q1 = V.q[1][row], q4 = V.q[4][row], q5 = V.q[5][row], q6 = V.q[6][row];
      const size_t o = V.outpos[row];
      if (o >= (size_t)V.cap_particles) { atomicOr(&V.cnt->error, DEVERR_PARTICLE_CAPACITY); continue; }
      const uint32_t tag = __float_as_uint(q6.w);
      const uint32_t id = (tag & TAG_ID_MASK) - R.id_base;
      const bool known = id < (uint32_t)R.id_cap;
      const uint32_t pst = known ? R.p_states[id] : 0u;
      const uint32_t mark = known ? R.p_mark[id] : 0u;
      const bool fresh = known && (mark >> 1) == epoch;   // gather_cdf saw this particle in this substep
      const float4 pc = fresh ? R.p_cdf[id] : make_float4(0.f, 0.f, 0.f, 0.f);
      const bool near = fresh && (mark & 1u);
      const float3 bn = make_float3(pc.x, pc.y, pc.z);
      // p.get_velocity() as rasterize left it: the gravity kick is stored back there (src/transfer.cpp:383-385)
      float3 pv = make_float3(q1.x, q1.y, q1.z);
      if (P.particle_gravity) { pv.x += P.gdt[0]; pv.y += P.gdt[1]; pv.z += P.gdt[2]; }
      int bx, by, bz;
      float rx, ry, rz;
      base_rel(q0.x, P.inv_dx, bx, rx);
      base_rel(q0.y, P.inv_dx, by, ry);
      base_rel(q0.z, P.inv_dx, bz, rz);
      const int lx = bx - tx * 4, ly = by - ty * 4, lz = bz - tz * 4;
      if ((unsigned)lx >= 4u || (unsigned)ly >= 4u || (unsigned)lz >= 4u) continue;
      float wx[3], wy[3], wz[3];
      bspline_weights(rx, wx); bspline_weights(ry, wy); bspline_weights(rz, wz);
      float3 v = make_float3(0.f, 0.f, 0.f);
      Mat3 B;
      for (int k = 0; k < 9; k++) B.m[k] = 0.f;
      int rigid_id = -1;
      for (int n = 0; n < 27; n++) {
        const int a = n / 9, b = (n / 3) % 3, c = n % 3;
        const int ln = ((lx + a) * 6 + (ly + b)) * 6 + (lz + c);
        const float w = (wx[a] * wy[b]) * wz[c];
        const float dp[3] = {rx - (float)a, ry - (float)b, rz - (float)c};
        float3 gv = make_float3(s_vel[ln].x, s_vel[ln].y, s_vel[ln].z);
        const uint32_t word = s_word[ln];
        if (!cdf_compatible(word, pst)) {   // different colour (761-785)
          float3 fake = pv, vg = make_float3(0.f, 0.f, 0.f);
          float friction = 0.f;
          const int rid = (int)(word >> 24) - 1;
          if (rid >= 0 && rid < R.n_bodies) {
            const RigidDev &Bd = R.bodies[rid];
            vg = rigid_velocity_at(Bd, make_float3((float)(bx + a) * P.dx, (float)(by + b) * P.dx, (float)(bz + c) * P.dx));
            rigid_id = rid;
            friction = Bd.fric[(pst >> (2 * rid)) & 1u];
          }
          if (near) {
            fake = friction_project_rel(pv, vg, bn, friction);
            const float push = P.dt * P.dx * R.pushing_force;
            fake.x += bn.x * push; fake.y += bn.y * push; fake.z += bn.z * push;
          }
          gv = fake;
        }
        v.x = fmaf(gv.x, w, v.x); v.y = fmaf(gv.y, w, v.y); v.z = fmaf(gv.z, w, v.z);                  // 788
        const float wgx = w * gv.x, wgy = w * gv.y, wgz = w * gv.z;
        for (int cc = 0; cc < 3; cc++) { B(0, cc) = fmaf(wgx, dp[cc], B(0, cc)); B(1, cc) = fmaf(wgy, dp[cc], B(1, cc)); B(2, cc) = fmaf(wgz, dp[cc], B(2, cc)); }   // 793-795
      }
      Mat3 cdg;  // 810-815
      for (int k = 0; k < 9; k++) cdg.m[k] = fmaf(scale, B.m[k], (k % 4 == 0) ? 1.f : 0.f);
      Mat3 Bst = B;  // p.apic_b: zero next to a boundary (800-804)
      if (near) for (int k = 0; k < 9; k++) Bst.m[k] = 0.f;
      Mat3 F;
      F.m[0] = q4.x; F.m[1] = q4.y; F.m[2] = q4.z; F.m[3] = q4.w; F.m[4] = q5.x; F.m[5] = q5.y; F.m[6] = q5.z; F.m[7] = q5.w; F.m[8] = q6.x;
      float ps = q6.y;
      const float vol = q6.z;
      Mat3 force, A;
      material_step<true>(P.mats[tag >> TAG_ID_BITS], cdg, F, ps, vol, force);
      make_affine(force, Bst, mass, scale, A);
      float3 x = make_float3(fmaf(v.x, P.dt, q0.x), fmaf(v.y, P.dt, q0.y), fmaf(v.z, P.dt, q0.z));   // 819
      if (near && pc.w < -0.05f * P.dx && pc.w > -P.dx * 0.3f) {   // 823-832: position correction
        const float3 dv = make_float3(pc.w * bn.x * R.penalty, pc.w * bn.y * R.penalty, pc.w * bn.z * R.penalty);
        v.x -= dv.x; v.y -= dv.y; v.z -= dv.z;
        if (rigid_id != -1) imp.add(s_acc, rigid_id, R.bodies[rigid_id], make_float3(dv.x * mass, dv.y * mass, dv.z * mass), x);
      }
      uint32_t key = make_key(P, x.x, x.y, x.z);
      if (P.clean_boundary && reference_deletes(P, x, v)) key = (uint32_t)(P.ntiles_total + SPECIAL_DEAD);
      if (!isfinite(x.x + x.y + x.z)) key = (uint32_t)(P.ntiles_total + SPECIAL_DEAD);
      store_particle<true>(V.qn, o, x, key == (uint32_t)tile ? mass : -mass, v, A, F, ps, vol, tag, Bst);
      V.keys_next[o] = key;
      if (key == (uint32_t)tile) {
        my_stay++;
      } else if (key != (uint32_t)(P.ntiles_total + SPECIAL_DEAD)) {
        const int m = atomicAdd(&V.cnt->n_movers_next, 1);
        if (m >= V.cap_particles) { atomicOr(&V.cnt->error, DEVERR_PARTICLE_CAPACITY); continue; }
        V.mover_dst_n[m] = key;
        V.mover_idx_n[m] = (uint32_t)o;
        MPMB_COUNT_ARRIVAL(V, P, key);
      }
    }
    if (my_stay) atomicAdd(&s_stay, my_stay);
    imp.flush(s_acc);
    __syncthreads();
    if (tid == 0) V.stay_next[tile] = s_stay;
    for (int n = tid; n < RIGID_MAX * 6; n += blockDim.x) {
      const float a = (&s_acc[0][0])[n];
      if (a != 0.f) atomicAdd(&R.bodies[n / 6].acc[n % 6], a);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------ debug grid
__global__ void k_dense_grid(View V, Params P, int which, float4 *dense) {
  size_t n = (size_t)P.nnode[0] * P.nnode[1] * P.nnode[2];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    int gz = (int)(i % P.nnode[2]), gy = (int)((i / P.nnode[2]) % P.nnode[1]), gx = (int)(i / ((size_t)P.nnode[2] * P.nnode[1]));
    int tx = gx >> 2, ty = gy >> 2, tz = gz >> 2;
    float4 g = gather_node(V.arena, V.cap_tiles, gx & 3, gy & 3, gz & 3, [&](int ox, int oy, int oz) {
      int x = tx - ox, y = ty - oy, z = tz - oz - P.tz_off;  // z: local layer
      if (x < 0 || y < 0 || z < 0 || x >= P.nt[0] || y >= P.nt[1] || z >= P.nt[2]) return -1;
      return V.slot_map[(x * P.nt[1] + y) * P.nt[2] + z];
    });
    if (which == 1) {
      float4 s;
      const bool has_s = node_sdf(P, V.sdf4, gx, gy, gz, s);
      g = node_update(P, g, has_s, s);
    }
    dense[i] = g;
  }
}

__global__ void k_planes_to_sdf(Params P, int n_planes, const float4 *planes, float4 *sdf4) {
  size_t n = (size_t)P.nnode[0] * P.nnode[1] * P.nnode[2];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    int gz = (int)(i % P.nnode[2]), gy = (int)((i / P.nnode[2]) % P.nnode[1]), gx = (int)(i / ((size_t)P.nnode[2] * P.nnode[1]));
    float best = 1e30f;
    float4 out = make_float4(1.f, 0.f, 0.f, 1e30f);
    for (int k = 0; k < n_planes; k++) {
      float4 pl = planes[k];
      float phi = pl.x * gx + pl.y * gy + pl.z * gz + pl.w;
      if (phi < best) { best = phi; out = make_float4(pl.x, pl.y, pl.z, phi); }
    }
    sdf4[i] = out;
  }
}

// Level set rasterised on the device from analytic solids (SURVEY §8f row 4; the scripts build theirs with
// levelset.add_plane / add_cuboid / add_sphere, scripts/mls-cpic/sand_sweep.py:13-19, scripts/async/sand.py:35,
// scripts/mls-cpic/sand_stir.py:9): phi = min over the shapes of their signed distance (grid units, negative inside the
// obstacle), n = the unit gradient of the minimiser.  inside_out turns a solid into a container.
//   plane   p = (n_x, n_y, n_z, d):      phi = n.X + d
//   sphere  p = (c_x, c_y, c_z, r):      phi = |X - c| - r
//   cuboid  p = (lo_xyz, hi_xyz):        phi = exact box distance (outside: to the nearest face/edge/corner; inside: -depth)
__device__ __forceinline__ float4 shape_sdf(const MpmbShape &S, float x, float y, float z) {
  float4 o;  // (n, phi)
  if (S.kind == MPMB_SHAPE_PLANE) {
    o = make_float4(S.p[0], S.p[1], S.p[2], S.p[0] * x + S.p[1] * y + S.p[2] * z + S.p[3]);
  } else if (S.kind == MPMB_SHAPE_SPHERE) {
    const float dx = x - S.p[0], dy = y - S.p[1], dz = z - S.p[2];
    const float r = sqrtf(dx * dx + dy * dy + dz * dz), inv = r > 1e-20f ? 1.0f / r : 0.f;
    o = make_float4(dx * inv, dy * inv, dz * inv, r - S.p[3]);
    if (!(r > 1e-20f)) o.x = 1.f;
  } else {
    const float X[3] = {x, y, z};
    float q[3], out2 = 0.f, depth = 1e30f;
    int amax = 0;
    float sgn[3];
    for (int a = 0; a < 3; a++) {
      const float c = 0.5f * (S.p[a] + S.p[3 + a]), hw = 0.5f * (S.p[3 + a] - S.p[a]);
      const float d = X[a] - c;
      sgn[a] = d < 0.f ? -1.f : 1.f;
      q[a] = fabsf(d) - hw;                  // > 0 outside along this axis
      if (q[a] > 0.f) out2 += q[a] * q[a];
      if (-q[a] < depth) { depth = -q[a]; amax = a; }
    }
    if (out2 > 0.f) {
      const float r = sqrtf(out2), inv = 1.0f / r;
      o = make_float4(q[0] > 0.f ? sgn[0] * q[0] * inv : 0.f, q[1] > 0.f ? sgn[1] * q[1] * inv : 0.f, q[2] > 0.f ? sgn[2] * q[2] * inv : 0.f, r);
    } else {
      o = make_float4(amax == 0 ? sgn[0] : 0.f, amax == 1 ? sgn[1] : 0.f, amax == 2 ? sgn[2] : 0.f, -depth);
    }
  }
  if (S.inside_out) o = make_float4(-o.x, -o.y, -o.z, -o.w);
  return o;
}
__global__ void k_shapes_to_sdf(Params P, int n_shapes, const MpmbShape *shapes, float4 *sdf4) {
  size_t n = (size_t)P.nnode[0] * P.nnode[1] * P.nnode[2];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    int gz = (int)(i % P.nnode[2]), gy = (int)((i / P.nnode[2]) % P.nnode[1]), gx = (int)(i / ((size_t)P.nnode[2] * P.nnode[1]));
    float4 best = make_float4(1.f, 0.f, 0.f, 1e30f);
    for (int k = 0; k < n_shapes; k++) {
      const float4 c = shape_sdf(shapes[k], (float)gx, (float)gy, (float)gz);
      if (c.w < best.w) best = c;
    }
    sdf4[i] = best;
  }
}

// ------------------------------------------------------------------------------ z-slab exchange
// Halo message: int4 header {count,0,0,0} | int tile_xy[cap_xy] | float4 arena[cap_xy][216].
// Packs the arenas of the owned tiles of one tile layer (the partial sums of (p,m) the neighbour
// rank's nodes need); the neighbour registers them as ghost tiles, so its grid update sums them in
// the same fixed order as a single-GPU run would.
// layer_z: LOCAL tile layer (global layer - P.tz_off)
__global__ void k_halo_pack(View V, Params P, int layer_z, int cap_xy, int *hdr, int *tile_xy, float4 *arenas) {
  __shared__ int s_idx;
  const int n_tiles = V.cnt->n_tiles;
  for (int slot = blockIdx.x; slot < n_tiles; slot += gridDim.x) {
    const int tile = V.meta[slot].tile;
    if (tile % P.nt[2] != layer_z) continue;  // uniform per CTA
    if (threadIdx.x == 0) {
      int idx = atomicAdd(&hdr[0], 1);
      if (idx >= cap_xy) { atomicOr(&V.cnt->error, DEVERR_TILE_CAPACITY); idx = -1; }
      else tile_xy[idx] = tile / P.nt[2];
      s_idx = idx;
    }
    __syncthreads();
    const int idx = s_idx;
    if (idx >= 0)
      for (int n = threadIdx.x; n < ARENA; n += blockDim.x) arenas[(size_t)idx * ARENA + n] = V.arena[(size_t)slot * ARENA + n];
    __syncthreads();
  }
}

__global__ void k_halo_unpack(View V, Params P, int layer_z, int cap_xy, const int *hdr, const int *tile_xy, const float4 *arenas) {
  __shared__ int s_slot;
  const int count = min(hdr[0], cap_xy);
  for (int e = blockIdx.x; e < count; e += gridDim.x) {
    if (threadIdx.x == 0) {
      int slot = V.cnt->n_tiles + atomicAdd(&V.cnt->n_ghost, 1);
      if (slot >= V.cap_tiles) { atomicOr(&V.cnt->error, DEVERR_TILE_CAPACITY); slot = -1; }
      else if (MPMB_CHK(V.cnt, (unsigned)tile_xy[e] < (unsigned)(P.nt[0] * P.nt[1]), 10, e, tile_xy[e], count)) V.slot_map[tile_xy[e] * P.nt[2] + layer_z] = slot;  // rewritten densely by the next ordering
      s_slot = slot;
    }
    __syncthreads();
    const int slot = s_slot;
    if (slot >= 0)
      for (int n = threadIdx.x; n < ARENA; n += blockDim.x) V.arena[(size_t)slot * ARENA + n] = arenas[(size_t)e * ARENA + n];
    __syncthreads();
  }
}

// CPIC colour state of the particles that change rank (z-slab ranks with rigid coupling; w == nullptr otherwise):
// MPMParticle::states, kept by ABSOLUTE particle id on z-slab ranks (w[id], id < n), travels in row 9 .y of the record
// (that row holds only apic_b[8] in .x), so the migration and re-cut records keep their size.  Without rigid coupling
// the records are the raw rows.
struct StateWords {
  uint32_t *w;
  int n;
};
__device__ __forceinline__ void copy_record(const StateWords &S, float4 *const *q, size_t i, float4 *rec, Counters *cnt) {
#pragma unroll
  for (int k = 0; k < N_Q - 1; k++) rec[k] = q[k][i];
  float4 r9 = q[N_Q - 1][i];
  if (S.w) {
    const uint32_t id = __float_as_uint(q[6][i].w) & TAG_ID_MASK;
    if (id < (uint32_t)S.n) r9.y = __uint_as_float(S.w[id]);
    else { r9.y = 0.f; atomicOr(&cnt->error, DEVERR_BAD_INPUT); }
  }
  rec[N_Q - 1] = r9;
}
__device__ __forceinline__ void record_state_in(const StateWords &S, const float4 *rec, Counters *cnt) {
  if (!S.w) return;
  const uint32_t id = __float_as_uint(rec[6].w) & TAG_ID_MASK;
  if (id < (uint32_t)S.n) S.w[id] = __float_as_uint(rec[N_Q - 1].y);
  else atomicOr(&cnt->error, DEVERR_BAD_INPUT);   // an id past the run's id range (include/mpmb.h, mpmb_set_rigid_samples)
}

// Migration message: int4 header {count,0,0,0} | float4 record[cap][N_Q].  Emigrants are the movers
// whose destination is the face's special key; their row in the (new) current storage is a hole
// for everybody else, the key is set dead so that downloads skip it.
__global__ void k_migrate_pack(View V, uint32_t key_face, uint32_t key_dead, int cap, int *hdr, float4 *rec, StateWords S) {
  const int n = V.cnt->n_movers;
  for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < n; m += gridDim.x * blockDim.x) {
    if (V.mover_dst[m] != key_face) continue;
    const uint32_t i = V.mover_idx[m];
    const int idx = atomicAdd(&hdr[0], 1);
    V.keys[i] = key_dead;
    V.mover_dst[m] = key_dead;
    if (idx >= cap) { atomicOr(&V.cnt->error, DEVERR_MIGRATE_CAPACITY); continue; }
    copy_record(S, V.q, i, rec + (size_t)idx * N_Q, V.cnt);
  }
}

// Immigrants are appended after the last row of the current storage and enter the mover list, so the
// next ordering bins them like any other particle that changed tile.
__global__ void k_migrate_unpack(View V, Params P, int cap, const int *hdr, const float4 *rec, StateWords S) {
  const int count = min(hdr[0], cap);
  const int base = V.cnt->n_store, mbase = V.cnt->n_movers;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < count; e += gridDim.x * blockDim.x) {
    const int dst = base + e;
    if (dst >= V.cap_particles) { atomicOr(&V.cnt->error, DEVERR_PARTICLE_CAPACITY); continue; }
    float4 r0 = rec[(size_t)e * N_Q];
#pragma unroll
    for (int k = 0; k < N_Q; k++) V.q[k][dst] = rec[(size_t)e * N_Q + k];
    record_state_in(S, rec + (size_t)e * N_Q, V.cnt);
    const uint32_t key = make_key(P, r0.x, r0.y, r0.z);
    V.keys[dst] = key;
    V.mover_dst[mbase + e] = key;
    V.mover_idx[mbase + e] = (uint32_t)dst;
    MPMB_COUNT_ARRIVAL(V, P, key);
  }
}
// ---- peer-memory exchange (no NCCL on the data path): the sending kernels store the payload straight into the neighbour
// GPU's receive buffer over NVLink and release {count, seq} system-wide; the receiving kernels acquire seq before they
// read.  One substep = one seq value; a bounded spin turns a lost peer into an error flag instead of a hung GPU.
// What mpmb_substep launches on a z-slab rank is fused:  one kernel per direction handles BOTH faces,
// resets its own counters and publishes from its last CTA; the receiving kernel waits for the neighbours' sequence
// numbers itself.  4 launches per substep instead of 22 (round 1: memset + pack + publish and wait + unpack (+ commit)
// per face and per message kind, each a 2-3 us launch on a stream whose real work is ~100 us at 8 ranks).
struct XFace {     // one face of one message kind, as the kernels see it
  char *tx;        // the neighbour's receive buffer (peer memory) — header | payload
  const char *rx;  // my receive buffer for this face
  int layer;       // halo: LOCAL tile layer packed (send) / registered as ghosts (recv)
  uint32_t key;    // migration: the special key of this face
};
__device__ __forceinline__ void xchg_spin(const int *hdr, int seq, Counters *cnt) {
  const long long t0 = clock64();
  for (;;) {
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(hdr + 1) : "memory");
    if (v >= seq) return;
    if (clock64() - t0 > 60000000000ll) {  // ~30 s: a lost peer becomes an error flag, not a hung GPU
      atomicOr(&cnt->error, DEVERR_PEER_TIMEOUT);
      return;
    }
    __nanosleep(200);
  }
}
// last CTA of a sending kernel: header {count, seq} of every face, counters back to zero for the next substep
__device__ __forceinline__ void xchg_publish_last(int *xcount, int *done, XFace f0, XFace f1, int mask, int seq) {
  __threadfence_system();  // my payload stores are visible system-wide before the CTA is counted as done
  __syncthreads();
  if (threadIdx.x == 0) {
    if (atomicAdd(done, 1) == (int)gridDim.x - 1) {
      __threadfence_system();
#pragma unroll
      for (int f = 0; f < 2; f++) {
        if (!((mask >> f) & 1)) continue;
        int *hdr = (int *)(f == 0 ? f0.tx : f1.tx);
        hdr[0] = atomicAdd(&xcount[4 * f], 0);
        __threadfence_system();
        asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(hdr + 1), "r"(seq) : "memory");
        xcount[4 * f] = 0;
      }
      *done = 0;
    }
  }
}

__global__ void __launch_bounds__(128) k_halo_send2(View V, Params P, int cap_xy, int idx_bytes, XFace f0, XFace f1, int mask, int *xcount, int *done) {
  __shared__ int s_idx[2];
  const int seq = V.cnt->xstep + 1;  // this substep's halo
  const int n_tiles = V.cnt->n_tiles;
  for (int slot = blockIdx.x; slot < n_tiles; slot += gridDim.x) {
    const int tile = V.meta[slot].tile, lz = tile % P.nt[2];
    const bool to0 = (mask & 1) && lz == f0.layer, to1 = (mask & 2) && lz == f1.layer;  // a one-layer slab sends the tile both ways
    if (!to0 && !to1) continue;                                                          // uniform per CTA
    if (threadIdx.x < 2) {
      int idx = -1;
      if (threadIdx.x == 0 ? to0 : to1) {
        idx = atomicAdd(&xcount[4 * threadIdx.x], 1);
        if (idx >= cap_xy) { atomicOr(&V.cnt->error, DEVERR_TILE_CAPACITY); idx = -1; }
        else ((int *)((threadIdx.x == 0 ? f0.tx : f1.tx) + 16))[idx] = tile / P.nt[2];
      }
      s_idx[threadIdx.x] = idx;
    }
    __syncthreads();
    const float4 *src = V.arena + (size_t)slot * ARENA;
#pragma unroll
    for (int f = 0; f < 2; f++) {
      const int idx = s_idx[f];
      if (idx < 0) continue;
      float4 *dst = (float4 *)((f == 0 ? f0.tx : f1.tx) + 16 + idx_bytes) + (size_t)idx * ARENA;
      for (int n = threadIdx.x; n < ARENA; n += blockDim.x) dst[n] = src[n];
    }
    __syncthreads();
  }
  xchg_publish_last(xcount, done, f0, f1, mask, seq);
}

__global__ void __launch_bounds__(128) k_halo_recv2(View V, Params P, int cap_xy, int idx_bytes, XFace f0, XFace f1, int mask) {
  __shared__ int s_slot;
  const int seq = V.cnt->xstep + 1;
  if (threadIdx.x == 0) {
    if (mask & 1) xchg_spin((const int *)f0.rx, seq, V.cnt);
    if (mask & 2) xchg_spin((const int *)f1.rx, seq, V.cnt);
  }
  __syncthreads();
  const int c0 = (mask & 1) ? min(((const int *)f0.rx)[0], cap_xy) : 0, c1 = (mask & 2) ? min(((const int *)f1.rx)[0], cap_xy) : 0;
  for (int e = blockIdx.x; e < c0 + c1; e += gridDim.x) {
    const bool lo = e < c0;
    const char *b = lo ? f0.rx : f1.rx;
    const int k = lo ? e : e - c0, layer = lo ? f0.layer : f1.layer;
    if (threadIdx.x == 0) {
      int slot = V.cnt->n_tiles + atomicAdd(&V.cnt->n_ghost, 1);
      if (slot >= V.cap_tiles) { atomicOr(&V.cnt->error, DEVERR_TILE_CAPACITY); slot = -1; }
      else if (MPMB_CHK(V.cnt, (unsigned)((const int *)(b + 16))[k] < (unsigned)(P.nt[0] * P.nt[1]), 11, k, ((const int *)(b + 16))[k], c0 + c1))
        V.slot_map[((const int *)(b + 16))[k] * P.nt[2] + layer] = slot;  // rewritten densely by the next ordering
      s_slot = slot;
    }
    __syncthreads();
    const int slot = s_slot;
    const float4 *src = (const float4 *)(b + 16 + idx_bytes) + (size_t)k * ARENA;
    if (slot >= 0)
      for (int n = threadIdx.x; n < ARENA; n += blockDim.x) V.arena[(size_t)slot * ARENA + n] = src[n];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) k_migrate_send2(View V, uint32_t key_dead, int cap, XFace f0, XFace f1, int mask, int *xcount, int *done, StateWords S) {
  const int n = V.cnt->n_movers;
  const int seq = V.cnt->xstep;  // k_g2p has committed this substep
  for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < n; m += gridDim.x * blockDim.x) {
    const uint32_t d = V.mover_dst[m];
    const int f = ((mask & 1) && d == f0.key) ? 0 : (((mask & 2) && d == f1.key) ? 1 : -1);
    if (f < 0) continue;
    const uint32_t i = V.mover_idx[m];
    const int idx = atomicAdd(&xcount[4 * f], 1);
    V.keys[i] = key_dead;
    V.mover_dst[m] = key_dead;
    if (idx >= cap) { atomicOr(&V.cnt->error, DEVERR_MIGRATE_CAPACITY); continue; }
    float4 *rec = (float4 *)((f == 0 ? f0.tx : f1.tx) + 16);
    copy_record(S, V.q, i, rec + (size_t)idx * N_Q, V.cnt);
  }
  xchg_publish_last(xcount, done, f0, f1, mask, seq);
}

// one CTA: waits for both neighbours, appends the immigrants of both faces after the last storage row, enters them in the
// mover list and commits the counts
__global__ void __launch_bounds__(1024) k_migrate_recv2(View V, Params P, int cap, XFace f0, XFace f1, int mask, StateWords S) {
  __shared__ int s_n[2];
  const int seq = V.cnt->xstep;
  if (threadIdx.x == 0) {
    if (mask & 1) xchg_spin((const int *)f0.rx, seq, V.cnt);
    if (mask & 2) xchg_spin((const int *)f1.rx, seq, V.cnt);
    int c0 = (mask & 1) ? min(((const int *)f0.rx)[0], cap) : 0, c1 = (mask & 2) ? min(((const int *)f1.rx)[0], cap) : 0;
    if (c0 > cap || c1 > cap) atomicOr(&V.cnt->error, DEVERR_MIGRATE_CAPACITY);
    const int room = max(V.cap_particles - V.cnt->n_store, 0);
    if (c0 + c1 > room) { atomicOr(&V.cnt->error, DEVERR_PARTICLE_CAPACITY); c0 = min(c0, room); c1 = min(c1, room - c0); }
    s_n[0] = c0; s_n[1] = c1;
  }
  __syncthreads();
  const int c0 = s_n[0], c1 = s_n[1];
  const int base = V.cnt->n_store, mbase = V.cnt->n_movers;
  for (int e = threadIdx.x; e < c0 + c1; e += blockDim.x) {
    const float4 *rec = (const float4 *)((e < c0 ? f0.rx : f1.rx) + 16) + (size_t)(e < c0 ? e : e - c0) * N_Q;
    const int dst = base + e;
    const float4 r0 = rec[0];
#pragma unroll
    for (int k = 0; k < N_Q; k++) V.q[k][dst] = rec[k];
    record_state_in(S, rec, V.cnt);
    const uint32_t key = make_key(P, r0.x, r0.y, r0.z);
    V.keys[dst] = key;
    V.mover_dst[mbase + e] = key;
    V.mover_idx[mbase + e] = (uint32_t)dst;
    MPMB_COUNT_ARRIVAL(V, P, key);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    V.cnt->n_store = base + c0 + c1;
    V.cnt->n_movers = mbase + c0 + c1;
  }
}

__global__ void k_migrate_commit(Counters *c, const int *hdr, int cap, int cap_particles) {
  const int n = min(min(hdr[0], cap), max(cap_particles - c->n_store, 0));
  c->n_store += n;
  c->n_movers += n;
}

// ---- rigid impulse mailboxes (z-slab ranks with rigid coupling, peer memory): every rank owns one mailbox of
// [2 transfers][world] slots that every other rank maps; a slot is {0, seq} (16 B) + one rank's RIGID_IMPULSE_FLOATS
// partial sums.  After transfer t a rank writes its partials into slot [t][rank] of EVERY mailbox, its own included, and
// releases seq system-wide; then it waits for all `world` slots [t][*] of its own mailbox and sums them in rank order.
// seq = the device exchange counter (+1 for the P2G transfer, which precedes k_g2p's commit), so a captured graph stays
// valid.  A slot is not overwritten before every rank has read it: the next write to [t][r] follows rank r's reduction of
// the other transfer, which waits for every rank's publication that follows its reduction of t.
constexpr int RMAIL_SLOT = 320;   // bytes: 16 + 4 * RIGID_IMPULSE_FLOATS, rounded up
static_assert(16 + 4 * RIGID_IMPULSE_FLOATS <= RMAIL_SLOT, "rigid mailbox slot");
__global__ void k_rigid_mail_send(RigidView R, char *const *boxes, int world, int rank, int transfer, int seq_off, const Counters *cnt) {
  const int seq = cnt->xstep + seq_off;
  const size_t off = ((size_t)transfer * world + rank) * RMAIL_SLOT;
  for (int j = 0; j < world; j++) {
    float *dst = (float *)(boxes[j] + off + 16);
    for (int n = threadIdx.x; n < RIGID_IMPULSE_FLOATS; n += blockDim.x) dst[n] = R.bodies[n / 6].acc[n % 6];
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0)
    for (int j = 0; j < world; j++) asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"((int *)(boxes[j] + off) + 1), "r"(seq) : "memory");
}
__global__ void k_rigid_mail_recv(RigidView R, const char *mine, int world, int transfer, int seq_off, Counters *cnt) {
  const int seq = cnt->xstep + seq_off;
  const char *box = mine + (size_t)transfer * world * RMAIL_SLOT;
  if (threadIdx.x == 0)
    for (int w = 0; w < world; w++) xchg_spin((const int *)(box + (size_t)w * RMAIL_SLOT), seq, cnt);
  __syncthreads();
  rigid_sum_apply(R, (const float *)(box + 16), RMAIL_SLOT / sizeof(float), world);
}

// ---- re-cut of the z slabs (mpmb_layer_counts, mpmb_recut_pack, mpmb_recut_apply), between substeps.  The GLOBAL tile layer
// of a row's base node, with make_key's arithmetic; a live row's layer lies in its rank's [tile_z0, tile_z1).
__device__ __forceinline__ int base_layer(float z, float inv_dx) {
  int bz;
  float r;
  base_rel(z, inv_dx, bz, r);
  return bz >> 2;
}
constexpr int RECUT_MAX_LAYERS = 1026;  // tile layers of a 4096-cell axis

// live rows of the current storage per global tile layer: a shared-memory histogram per CTA, one 64-bit integer atomic
// per non-empty bin into hist (zeroed by the caller)
__global__ void __launch_bounds__(256) k_layer_hist(const uint32_t *keys, const float4 *q0, uint32_t special_min, float inv_dx, int n_layers,
                                                    const Counters *cnt, unsigned long long *hist) {
  __shared__ int s_h[RECUT_MAX_LAYERS];
  for (int l = threadIdx.x; l < n_layers; l += blockDim.x) s_h[l] = 0;
  __syncthreads();
  const int n = cnt->n_store;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (keys[i] >= special_min) continue;
    const int l = base_layer(q0[i].z, inv_dx);
    if (l >= 0 && l < n_layers) atomicAdd(&s_h[l], 1);
  }
  __syncthreads();
  for (int l = threadIdx.x; l < n_layers; l += blockDim.x)
    if (s_h[l]) atomicAdd(&hist[l], (unsigned long long)s_h[l]);
}

// flags[i] = 1 for the live rows whose base layer lies in [lo, hi)
__global__ void k_layer_flags(const uint32_t *keys, const float4 *q0, int n, uint32_t special_min, float inv_dx, int lo, int hi, int *flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int f = 0;
  if (keys[i] < special_min) {
    const int l = base_layer(q0[i].z, inv_dx);
    f = l >= lo && l < hi;
  }
  flags[i] = f;
}

// the rows k_layer_flags marked (prefix = its exclusive scan), in storage order, as migration records: N_Q raw float4 rows
__global__ void k_recut_pack(View V, int n, const int *prefix, float4 *rec, StateWords S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || prefix[i + 1] == prefix[i]) return;
  const size_t o = (size_t)prefix[i];
  copy_record(S, V.q, i, rec + o * N_Q, V.cnt);
}

// the rows k_layer_flags marked, compacted in storage order into the other buffer and keyed under the new slicing P;
// *max_id = the largest id among them (warp maximum, one atomic per warp)
__global__ void __launch_bounds__(256) k_recut_keep(View V, Params P, int n, const int *prefix, int *max_id) {
  int m = -1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (prefix[i + 1] == prefix[i]) continue;
    const size_t o = (size_t)prefix[i];
#pragma unroll
    for (int k = 0; k < N_Q; k++) V.qn[k][o] = V.q[k][i];
    const float4 r0 = V.q[0][i];
    V.keys_next[o] = make_key(P, r0.x, r0.y, r0.z);
    m = max(m, (int)(__float_as_uint(V.q[6][i].w) & TAG_ID_MASK));
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m >= 0) atomicMax(max_id, m);
}

// the arriving records of a re-cut, before anything changes: *bad counts those the new slicing P does not own, *max_id
// receives their largest id
__global__ void __launch_bounds__(256) k_recut_check(Params P, int n, const float4 *rec, int *bad, int *max_id) {
  int m = -1, b = 0;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
    const float4 r0 = rec[(size_t)e * N_Q];
    b += make_key(P, r0.x, r0.y, r0.z) >= (uint32_t)P.ntiles_total;
    m = max(m, (int)(__float_as_uint(rec[(size_t)e * N_Q + 6].w) & TAG_ID_MASK));
  }
  if (b) atomicAdd(bad, b);
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m >= 0) atomicMax(max_id, m);
}

// the arriving records after row row0 of the current storage, keyed under P (as k_migrate_recv2 appends immigrants)
__global__ void k_recut_unpack(View V, Params P, int n, int row0, const float4 *rec, StateWords S) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int dst = row0 + e;
#pragma unroll
  for (int k = 0; k < N_Q; k++) V.q[k][dst] = rec[(size_t)e * N_Q + k];
  record_state_in(S, rec + (size_t)e * N_Q, V.cnt);
  const float4 r0 = rec[(size_t)e * N_Q];
  V.keys[dst] = make_key(P, r0.x, r0.y, r0.z);
}

// ------------------------------------------------------------------------------ AsyncMPM pools (mpmb_async_*)
// One pool of AsyncMPM particle records, SoA: x[3n] v[3n] F[9n] b[9n] mass vol scalar group id block (the linear index of
// the record's 4x4x8-node scheduler block).
struct ARec {
  float *x, *v, *F, *b, *mass, *vol, *scalar;
  int *group;
  uint32_t *id;
  int *block;
};
constexpr int AREC_WORDS = 30;  // 4-byte words per record
enum { ASYNC_SMALLER = MPMB_ASYNC_SMALLER, ASYNC_EQUAL = MPMB_ASYNC_EQUAL, ASYNC_LARGER = MPMB_ASYNC_LARGER, ASYNC_SWAP = MPMB_ASYNC_SWAP,
       ASYNC_CLEAR = MPMB_ASYNC_CLEAR };

__device__ __forceinline__ void arec_copy(const ARec &d, size_t j, const ARec &s, size_t i) {
#pragma unroll
  for (int k = 0; k < 3; k++) { d.x[3 * j + k] = s.x[3 * i + k]; d.v[3 * j + k] = s.v[3 * i + k]; }
#pragma unroll
  for (int k = 0; k < 9; k++) { d.F[9 * j + k] = s.F[9 * i + k]; d.b[9 * j + k] = s.b[9 * i + k]; }
  d.mass[j] = s.mass[i]; d.vol[j] = s.vol[i]; d.scalar[j] = s.scalar[i];
  d.group[j] = s.group[i]; d.id[j] = s.id[i]; d.block[j] = s.block[i];
}

// The scheduler block of a position, in the host scheduler's fp32 arithmetic with ITS 1/dx: base = int(x * inv_dx - 0.5),
// block = (base_x >> 2, base_y >> 2, base_z >> 3), linear (bx * nb1 + by) * nb2 + bz.  A block outside the grid counts in *bad.
__global__ void k_async_blocks(const float *x, int n, float inv_dx, int nb0, int nb1, int nb2, int *block, int *bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c[3];
#pragma unroll
  for (int a = 0; a < 3; a++) c[a] = (int)__fsub_rn(__fmul_rn(x[3 * (size_t)i + a], inv_dx), 0.5f);
  const int bx = c[0] >> 2, by = c[1] >> 2, bz = c[2] >> 3;
  const bool ok = bx >= 0 && by >= 0 && bz >= 0 && bx < nb0 && by < nb1 && bz < nb2;
  block[i] = ok ? (bx * nb1 + by) * nb2 + bz : 0;
  if (!ok) atomicAdd(bad, 1);
}

// MPMParticle::get_allowed_dt of the registered types (src/particles.cpp:136-153, 254-281, 480-494, 649-668, 734-753,
// 814-833) in the operation order of async_mpm.allowed_dt: fp32 with explicit rounding (no FMA contraction), the
// determinant and the transcendental functions in fp64 rounded once.  Types without a limit (linear, jelly) return -1.
__device__ __forceinline__ float async_allowed_dt(const Material &M, const float *F, float ps, float mass, float vol, float v2, float dx) {
  const double d = (double)F[0] * ((double)F[4] * F[8] - (double)F[5] * F[7]) - (double)F[1] * ((double)F[3] * F[8] - (double)F[5] * F[6]) +
                   (double)F[2] * ((double)F[3] * F[7] - (double)F[4] * F[6]);
  float J = (float)d;
  const float u = sqrtf(v2);
  const float rho0 = mass / vol;
  float c;
  if (M.kind == MAT_SNOW) {
    J = __fmul_rn(J, ps);
    const float hh = (float)exp((double)__fmul_rn(M.p[2], __fsub_rn(1.0f, ps)));
    const float mu = __fmul_rn(M.p[0], hh), lam = __fmul_rn(M.p[1], hh);
    c = sqrtf(__fadd_rn(lam, __fmul_rn(2.0f, mu)) / (rho0 / J));
  } else if (M.kind == MAT_WATER) {
    c = sqrtf(__fmul_rn(M.p[0], M.p[1]) / (float)pow((double)ps, (double)__fsub_rn(M.p[1], 1.0f)));
  } else if (M.kind == MAT_SAND || M.kind == MAT_VON_MISES || M.kind == MAT_ELASTIC || M.kind == MAT_VISCO) {
    const float mu = M.p[0], lam = M.p[1];
    const float K = __fadd_rn(__fmul_rn(2.0f, mu) / 3.0f, lam);
    const float c2 = __fadd_rn(__fmul_rn(4.0f, mu) / __fmul_rn(3.0f, rho0 / J), __fmul_rn(K, __fsub_rn(1.0f, (float)log((double)J))) / rho0);
    c = sqrtf(c2 != c2 ? c2 : fmaxf(c2, 1e-20f));  // np.maximum keeps a NaN
  } else {
    return -1.0f;
  }
  return dx / __fadd_rn(c, u);
}

// One pass over the particle pool: per block an occupied bit (1), and with limits min(0.1, allowed_dt) and max |v|^2 as
// the bits of non-negative floats read as signed integers (ordered like the floats), a NaN as a flag bit (2: the limit,
// 4: |v|^2).  A type without a limit counts in *bad; its block is still occupied.
__global__ void __launch_bounds__(256) k_async_limits(ARec R, int n, Params P, int with_limits, uint32_t *bflag, int *bmin, int *bmax, int *bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int blk = R.block[i];
  if (!with_limits) {
    if (bflag[blk] == 0u) atomicOr(&bflag[blk], 1u);
    return;
  }
  const float vx = R.v[3 * (size_t)i], vy = R.v[3 * (size_t)i + 1], vz = R.v[3 * (size_t)i + 2];
  const float v2 = __fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)), __fmul_rn(vz, vz));
  const int g = min(max(R.group[i], 0), MPMB_MAX_GROUPS - 1);
  float adt = async_allowed_dt(P.mats[g], R.F + 9 * (size_t)i, R.scalar[i], R.mass[i], R.vol[i], v2, P.dx);
  unsigned f = 1u;
  if (adt == -1.0f) {
    atomicAdd(bad, 1);
    atomicOr(&bflag[blk], f);
    return;
  }
  if (adt != adt) f |= 2u;
  else atomicMin(&bmin[blk], __float_as_int(fminf(0.1f, adt)));
  if (v2 != v2) f |= 4u;
  else atomicMax(&bmax[blk], __float_as_int(v2));
  atomicOr(&bflag[blk], f);
}

__global__ void k_async_occupied(const uint32_t *bflag, int nblk, int *flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nblk) flags[i] = (int)(bflag[i] & 1u);
}

// the occupied blocks in block order, with their limits
__global__ void k_async_block_out(const uint32_t *bflag, const int *bmin, const int *bmax, int nblk, const int *prefix, int *ob, float *omin,
                                  float *omax) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nblk || !(bflag[i] & 1u)) return;
  const int o = prefix[i];
  ob[o] = i;
  omin[o] = (bflag[i] & 2u) ? __uint_as_float(0x7fc00000u) : __int_as_float(bmin[i]);
  omax[o] = (bflag[i] & 4u) ? __uint_as_float(0x7fc00000u) : __int_as_float(bmax[i]);
}

// candidates of a gather: [0, np) pool entries of SMALLER blocks, [np, 2np) pool entries of EQUAL blocks, [2np, 2np + nbk)
// backup entries of LARGER blocks
__device__ __forceinline__ int async_cand_part(int c, int np, int &src) {
  if (c < np) { src = c; return 0; }
  if (c < 2 * np) { src = c - np; return 1; }
  src = c - 2 * np;
  return 2;
}

__global__ void k_async_cand_flags(const int *pblock, int np, const int *bblock, int nbk, const uint8_t *bfl, int *flags) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 2 * np + nbk) return;
  int s;
  const int part = async_cand_part(c, np, s);
  const int want = part == 0 ? ASYNC_SMALLER : part == 1 ? ASYNC_EQUAL : ASYNC_LARGER;
  flags[c] = (bfl[part == 2 ? bblock[s] : pblock[s]] & want) ? 1 : 0;
}

// SPGrid's page index of a block (async_mpm._morton): coordinate bits interleaved y, x, z from the least significant
__device__ __forceinline__ unsigned long long async_morton(int bx, int by, int bz) {
  unsigned long long m = 0;
#pragma unroll
  for (int i = 0; i < 12; i++)
    m |= ((unsigned long long)((by >> i) & 1) << (3 * i)) | ((unsigned long long)((bx >> i) & 1) << (3 * i + 1)) |
         ((unsigned long long)((bz >> i) & 1) << (3 * i + 2));
  return m;
}

// the flagged candidates in candidate order with the sort key (part, morton of the block)
__global__ void k_async_cand_keys(const int *pblock, int np, const int *bblock, int nbk, const int *flags, const int *prefix, int nb1, int nb2,
                                  unsigned long long *key, uint32_t *cand) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 2 * np + nbk || !flags[c]) return;
  int s;
  const int part = async_cand_part(c, np, s);
  const int blk = part == 2 ? bblock[s] : pblock[s];
  const int bz = blk % nb2, by = (blk / nb2) % nb1, bx = blk / (nb1 * nb2);
  const int o = prefix[c];
  key[o] = ((unsigned long long)part << 36) | async_morton(bx, by, bz);
  cand[o] = (uint32_t)c;
}

__global__ void k_async_cand_ids(const uint32_t *cand, int nc, const uint32_t *pid, int np, const uint32_t *bid, uint32_t *ids, uint32_t *pos) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nc) return;
  int s;
  const int part = async_cand_part((int)cand[k], np, s);
  ids[k] = part == 2 ? bid[s] : pid[s];
  pos[k] = (uint32_t)k;
}

// sorted by id (stable: ascending gather position within an id): the first entry of every id is the copy that is kept
__global__ void k_async_first(const uint32_t *ids_sorted, const uint32_t *pos_sorted, int nc, int *keep) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < nc) keep[pos_sorted[j]] = (j == 0 || ids_sorted[j] != ids_sorted[j - 1]) ? 1 : 0;
}

__global__ void k_async_gather(const uint32_t *cand, int nc, const int *keep, const int *prefix, ARec Pp, int np, ARec Bp, ARec G) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nc || !keep[k]) return;
  int s;
  const int part = async_cand_part((int)cand[k], np, s);
  arec_copy(G, (size_t)prefix[k], part == 2 ? Bp : Pp, (size_t)s);
}

__global__ void k_async_rec_flags(const int *block, int n, const uint8_t *bfl, int bit, int *flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = (bfl[block[i]] & bit) ? 1 : 0;
}

// stable partition: flagged records to dA[offA + rank among the flagged], the others to dB[offB + rank among the others];
// a side whose has* is 0 is dropped
__global__ void k_async_split(ARec src, int n, const int *flags, const int *prefix, ARec dA, int offA, int hasA, ARec dB, int offB, int hasB) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (flags[i]) {
    if (hasA) arec_copy(dA, (size_t)offA + prefix[i], src, (size_t)i);
  } else if (hasB) {
    arec_copy(dB, (size_t)offB + (i - prefix[i]), src, (size_t)i);
  }
}

// survivors of a substep: row of every gather index (-1: deleted)
__global__ void k_async_rank(const uint32_t *sid, int ns, int *rowk) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < ns) rowk[sid[r]] = r;
}

// in gather order: survivors whose new block is EQUAL (to_backup = 0), or CLEAR and not EQUAL (to_backup = 1)
__global__ void k_async_route_flags(const int *rowk, int ng, const int *sblock, const uint8_t *bfl, int to_backup, int *flags) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ng) return;
  const int r = rowk[k];
  int f = 0;
  if (r >= 0) {
    const uint8_t b = bfl[sblock[r]];
    f = to_backup ? (!(b & ASYNC_EQUAL) && (b & ASYNC_CLEAR)) : ((b & ASYNC_EQUAL) != 0);
  }
  flags[k] = f;
}

// the survivor of gather index k appended to a pool, with the particle id of its gathered record (the engine numbered it k)
__global__ void k_async_route(const int *rowk, int ng, const int *flags, const int *prefix, ARec S, const uint32_t *gid, ARec D, int off) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ng || !flags[k]) return;
  const size_t o = (size_t)off + prefix[k];
  arec_copy(D, o, S, (size_t)rowk[k]);
  D.id[o] = gid[k];
}

// ---- the block scheduler on the device (mpmb_async_schedule / mpmb_async_advance_level): async_mpm.update_dt_limits and
// the flag building of async_mpm.advance, per block instead of per numpy pass
struct ASched {
  int bad;      // pool particles of a type without a time-step limit (k_async_limits)
  int due;      // some occupied block is due
  int low;      // some due block's limit is below one unit
  int ne_max;   // max level over the occupied blocks after their update, 1 if there are none
  int lv_min, lv_max;   // over all blocks after the empty-block pass
  int sc;       // MPMB_ASYNC_SWAP | MPMB_ASYNC_CLEAR bits of the last flag set built on the device
};
// the schedule fails, and no block state changes: a type without a limit while a block is due (the host raises wherever in
// the pool that particle lies, async_mpm._pool_scan), or a due block's limit below one unit
__device__ __forceinline__ bool async_sched_failed(const ASched *S) { return S->low || (S->bad && S->due); }

__global__ void k_async_state_init(int nblk, int *level, long long *local_min, long long *particle_t, long long *backup_t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nblk) return;
  level[i] = 1;
  local_min[i] = 1;
  particle_t[i] = 0;
  backup_t[i] = 0;
}

// the block reductions of k_async_limits start empty (0.1 / 1e-16 as in mpmb_async_block_limits), the counters from nothing
__global__ void k_async_sched_reset(int nblk, uint32_t *bflag, int *bmin, int *bmax, ASched *S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *S = ASched{0, 0, 0, 1, 0x7fffffff, 0, 0};
  if (i >= nblk) return;
  bflag[i] = 0u;
  bmin[i] = 0x3dcccccd;   // 0.1f
  bmax[i] = 0x2539705f;   // 1e-16f
}

// float32 -> int64 as numpy's astype on x86 (cvttss2si): truncation, INT64_MIN for NaN and |x| >= 2^63
__device__ __forceinline__ long long async_f2i64(float x) { return fabsf(x) < 9223372036854775808.0f ? (long long)x : INT64_MIN; }

// occupied blocks (update_dt_limits, :95-131): a due block takes tmp = min(cdl, sdl, max_units) and moves its level toward it,
// into lv_new; strength limit sdl = (s min_adt) inv_unit, CFL limit cdl = ((c dx) inv_unit) (1 / sqrt(max_v2)), every
// operation rounded on its own as the host's fp32 numpy expressions
__global__ void k_async_sched_due(const uint32_t *bflag, const int *bmin, const int *bmax, const int *level, int *lv_new, int nblk, long long t,
                                  float smul, float cmul, float dx, float inv_unit, long long max_units, ASched *S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nblk) return;
  const uint32_t f = bflag[i];
  if (!(f & 1u)) return;
  long long lv = level[i];
  if ((t & (lv - 1)) == 0) {
    atomicOr(&S->due, 1);
    const float min_adt = (f & 2u) ? __uint_as_float(0x7fc00000u) : __int_as_float(bmin[i]);
    const float max_v2 = (f & 4u) ? __uint_as_float(0x7fc00000u) : __int_as_float(bmax[i]);
    const long long sdl = async_f2i64(__fmul_rn(__fmul_rn(smul, min_adt), inv_unit));
    const long long cdl = async_f2i64(__fmul_rn(__fmul_rn(__fmul_rn(cmul, dx), inv_unit), 1.0f / sqrtf(max_v2)));   // IEEE / and sqrt
    const long long tmp = min(min(cdl, sdl), max_units);
    if (tmp < 1) {
      atomicOr(&S->low, 1);
      return;
    }
    while (tmp < lv) lv >>= 1;
    while (tmp >= 2 * lv && (t & (2 * lv - 1)) == 0) lv <<= 1;
  }
  lv_new[i] = (int)lv;
  atomicMax(&S->ne_max, (int)lv);
}

// every block's level is committed: an occupied block's from lv_new, an aligned empty one moves toward the occupied blocks'
// max (:138-152); then min / max over all blocks
__global__ void k_async_sched_commit(const uint32_t *bflag, const int *lv_new, int *level, int nblk, long long t, ASched *S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nblk || async_sched_failed(S)) return;
  long long lv;
  if (bflag[i] & 1u) {
    lv = lv_new[i];
  } else {
    lv = level[i];
    if ((t & (lv - 1)) == 0) {
      const long long mx = S->ne_max;
      while (mx < lv) lv >>= 1;
      while (mx >= 2 * lv && (t & (2 * lv - 1)) == 0) lv <<= 1;
    }
  }
  level[i] = (int)lv;
  atomicMin(&S->lv_min, (int)lv);
  atomicMax(&S->lv_max, (int)lv);
}

// fn(j) for the linear index j of every in-range neighbour of block i (the scheduler's cached_neighbours,
// src/async/async_mpm.h:255-300)
template <class Fn>
__device__ __forceinline__ void async_neighbours(int i, int nb0, int nb1, int nb2, Fn fn) {
  const int bz = i % nb2, by = (i / nb2) % nb1, bx = i / (nb1 * nb2);
  for (int dx = -1; dx <= 1; dx++)
    for (int dy = -1; dy <= 1; dy++)
      for (int dz = -1; dz <= 1; dz++) {
        const int x = bx + dx, y = by + dy, z = bz + dz;
        if ((dx | dy | dz) == 0 || x < 0 || y < 0 || z < 0 || x >= nb0 || y >= nb1 || z >= nb2) continue;
        fn((x * nb1 + y) * nb2 + z);
      }
}

// local_min_dt_limit (:165-181): a block off the finest level takes the earliest time a neighbour is stepped next
__global__ void k_async_local_min(const int *level, const long long *particle_t, long long *local_min, int nb0, int nb1, int nb2, const ASched *S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb0 * nb1 * nb2 || async_sched_failed(S) || level[i] == S->lv_min) return;
  long long lm = 1ll << 31;
  async_neighbours(i, nb0, nb1, nb2, [&](int j) { lm = min(lm, particle_t[j] + level[j]); });
  local_min[i] = lm;
}

// the MPMB_ASYNC_* bits of every block for level `limit` at clock t (async_mpm.advance; the larger / smaller neighbour sets
// of :183-250 reduce to: a neighbour is on that level)
__global__ void k_async_level_flags(const int *level, const long long *particle_t, const long long *local_min, int nb0, int nb1, int nb2, long long t,
                                    int limit, uint8_t *bfl, ASched *S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb0 * nb1 * nb2) return;
  const int lv = level[i];
  int f;
  if (lv == limit) {
    f = ASYNC_EQUAL | (particle_t[i] == t ? ASYNC_SWAP : 0);
  } else {
    bool touch = false;
    async_neighbours(i, nb0, nb1, nb2, [&](int j) { touch |= level[j] == limit; });
    f = !touch ? 0 : lv < limit ? ASYNC_SMALLER : ASYNC_LARGER | (local_min[i] == t + limit ? ASYNC_CLEAR : 0);
  }
  bfl[i] = (uint8_t)f;
  if (f & (ASYNC_SWAP | ASYNC_CLEAR)) atomicOr(&S->sc, f & (ASYNC_SWAP | ASYNC_CLEAR));
}

// the blocks' clocks after an advance of level `limit` (:318-343), in the host's order
__global__ void k_async_level_clocks(const uint8_t *bfl, int nblk, long long t, int limit, long long *particle_t, long long *backup_t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nblk) return;
  const int f = bfl[i];
  if (f & ASYNC_SWAP) backup_t[i] = t;
  if (f & ASYNC_EQUAL) particle_t[i] = t + limit;
  if (f & ASYNC_CLEAR) backup_t[i] = t + limit;
}

}  // namespace mpmb

// =====================================================================================
// Host side
// =====================================================================================
using namespace mpmb;

// One device allocation of n elements of T, owned: freed by the destructor or by the next allocation.  Move-only, so every
// address has exactly one owner; kernels and their argument structs get the raw pointer (get()), never the buffer.
template <class T>
class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  DevBuf &operator=(DevBuf &&o) noexcept {   // frees what this buffer held
    if (this != &o) {
      reset();
      p_ = o.p_; n_ = o.n_;
      o.p_ = nullptr; o.n_ = 0;
    }
    return *this;
  }
  ~DevBuf() { reset(); }
  // exactly n elements, content undefined; the old allocation is freed first, so after a failure the buffer is empty
  cudaError_t alloc(size_t n) {
    reset();
    cudaError_t e = cudaMalloc(&p_, sizeof(T) * n);
    if (e != cudaSuccess) p_ = nullptr;
    else n_ = n;
    return e;
  }
  // at least n elements: a smaller buffer is replaced by one of exactly n, its content discarded
  cudaError_t reserve(size_t n) { return n <= n_ ? cudaSuccess : alloc(n); }
  void reset() {
    if (p_) cudaFree(p_);
    p_ = nullptr;
    n_ = 0;
  }
  T *get() const { return p_; }
  size_t size() const { return n_; }

 private:
  T *p_ = nullptr;
  size_t n_ = 0;
};

// fields of `cap` records laid out one after another in one allocation of AREC_WORDS * cap words
static ARec arec_layout(float *w, int64_t cap) {
  const size_t c = (size_t)cap;
  ARec r;
  r.x = w; r.v = w + 3 * c; r.F = w + 6 * c; r.b = w + 15 * c; r.mass = w + 24 * c; r.vol = w + 25 * c; r.scalar = w + 26 * c;
  r.group = (int *)(w + 27 * c); r.id = (uint32_t *)(w + 28 * c); r.block = (int *)(w + 29 * c);
  return r;
}
// a buffer of whole records and the layout of its records
static int64_t arec_cap(const DevBuf<float> &buf) { return (int64_t)(buf.size() / AREC_WORDS); }
static ARec arec_of(const DevBuf<float> &buf) { return arec_layout(buf.get(), arec_cap(buf)); }

struct Mpm2d;  // the 2-D engine (below, "The 2-D engine")

struct MpmbEngine {
  MpmbConfig cfg{};
  Mpm2d *m2 = nullptr;   // set on a 2-D handle (cfg.dim == 2): every entry point routes to it or refuses
  Params P{};
  cudaStream_t stream = nullptr;
  std::string err;
  bool sticky_cuda = false;

  int64_t cap = 0;       // particle rows allocated per buffer
  int cur = 0;           // which q/keys buffer is current
  int ord = 0;           // which (run,stay) set is current
  int mov = 0;           // which mover list the next ordering consumes
  bool fresh = false;    // storage was just uploaded: arrival lists come from the radix sort
  DevBuf<float4> q[2][N_Q];
  DevBuf<uint32_t> keys[2];       // tile of every row (cur / next)
  DevBuf<uint32_t> outpos;
  DevBuf<uint32_t> mover_dst[2], mover_idx[2];
  DevBuf<uint32_t> arrivals, arrivals_sorted;
  DevBuf<uint32_t> keys_sorted, iota;  // upload-time radix sort scratch
  uint32_t special_min = 0, key_dead = 0;
  DevBuf<unsigned char> cub_temp;
  int key_bits = 32;

  int cap_tiles = 0;
  int ntot = 0;           // tiles of the dense tile grid
  int ord_blocks = 0;
  DevBuf<int> run_begin[2], run_len[2], stay[2];  // [ord]: current / next
  DevBuf<int> arr_cnt, arr_off, arr_len, arr_cur, slot_map, blocksum;
  DevBuf<TileMeta> meta;
  DevBuf<float4> arena;
  DevBuf<float4> sdf4;
  DevBuf<Counters> cnt;

  int stage = 0;  // 0 idle/after resample, 1 after sort, 2 after rasterize
  int64_t mig_cap = 0;
  // peer-memory exchange: rx = my receive buffers [kind 0 halo / 1 migration][face], tx = the
  // neighbour's receive buffer I write into through face f
  DevBuf<char> rx[2][2];
  char *tx[2][2] = {};    // not owned: the neighbour's rx, mapped by IPC (closed by mpmb_destroy) or given by the same process
  bool tx_ipc[2][2] = {};
  DevBuf<int> xcount;     // local pack counters (int4 per [kind][face])
  int xstep = 0;          // substeps completed since the peers were connected
  bool skip_b = false;        // intermediate substeps of mpmb_substep do not store apic_b
  DevBuf<unsigned char> stage_buf;  // cached staging buffer of the host<->device marshalling
  // device image of the reference's AoS pool + index vector, kept from mpmb_upload_aos to mpmb_download_aos
  DevBuf<unsigned char> aos_pool;
  DevBuf<uint32_t> aos_idx;
  const void *aos_host_pool = nullptr;  // not owned: the host pool, kept only to identify the image (with slots and particle count)
  int64_t aos_slots = 0, aos_n = 0;
  // group -> material kind at the last mpmb_upload_aos: where per-kind scalars are read at upload and written at download
  int32_t aos_kinds[MPMB_MAX_GROUPS] = {};
  bool aos_kinds_valid = false;
  DevBuf<int> scan_a, scan_b;  // flags / prefix scratch (downloads, seeding)
  DevBuf<unsigned char> scan_tmp;
  uint32_t id_base = 0;
  int num_sms = 132;  // H100 SXM; queried from the device in mpmb_create
  int nt2_global = 0;  // tile layers of the whole domain (P.nt[2] is slab-local)
  DevBuf<unsigned long long> recut_buf;  // re-cut scratch: layer histogram [nt2_global], then two ints (bad arrivals, largest id)
  int grid_p2g = 132 * 4, grid_g2p = 132 * 4;  // persistent grids = SMs x resident CTAs (queried)
  int64_t launches = 0;

  // two substeps captured as one CUDA graph per buffer parity: mpmb_substep replays it instead of re-launching
  // 16 (1 GPU) / 24 (z-slab rank) kernels from the host; invalidated by anything that changes a kernel argument
  cudaGraphExec_t graph_exec[2] = {nullptr, nullptr};
  int graph_launches = 0;
  cudaStream_t cap_stream = nullptr;
  bool use_graph = true;

  // CPIC rigid coupling (enabled by mpmb_set_rigid_samples with at least one sample); rigid_view() hands it to the kernels
  bool rigid_on = false;
  int rigid_bodies = 0, rigid_samples = 0;
  int rigid_nb[3] = {};                // rigid_page_map blocks (4x4x8 nodes) per axis
  float penalty = 0.f, pushing_force = 0.f;
  DevBuf<RigidDev> bodies;             // [RIGID_MAX]
  DevBuf<float> rs_offset, rs_tri;     // boundary samples
  DevBuf<int> rs_rigid, s_base;
  DevBuf<unsigned long long> node_key; // colour field of the whole node grid
  DevBuf<uint32_t> node_tags;
  DevBuf<unsigned char> page, tile_flag;
  DevBuf<uint32_t> p_states;           // by particle id - id_base: its size is the number of ids tracked
  DevBuf<float4> p_cdf;
  DevBuf<uint32_t> p_mark;
  DevBuf<uint32_t> epoch;
  // bodies advanced on the device (mpmb_set_rigid_motion): master states, script table, contacts; motion_view() for the kernels
  bool motion_on = false;
  bool motion_scripted = false;        // some body follows the script table
  bool motion_collide = false;         // the level-set collision was asked for (it runs while a level set is set)
  RigidMaster h_master[RIGID_MAX] = {};  // host image: motion parameters (+ the state last written by the host)
  DevBuf<RigidMaster> master;          // [RIGID_MAX]
  DevBuf<int> cursor;                  // next script entry
  DevBuf<double> script;               // grow-only: its size is the capacity in doubles
  int64_t script_left = 0;             // entries not yet consumed (host-side count of the device cursor)
  DevBuf<int> s_order;                 // sample indices grouped by body; body b owns s_order[s_begin[b] .. s_begin[b + 1])
  int s_begin[RIGID_MAX + 1] = {};
  DevBuf<double> contact;
  // z-slab ranks: the bodies' impulses are summed over the ranks after each transfer (mpmb_rigid_impulse_* / mpmb_rigid_*)
  int rigid_pending = 0;               // 1 / 2: the P2G / G2P transfer has run here and its partial impulses await the reduction
  bool rigid_sent = false;             // ... and were published into the mailboxes (mpmb_rigid_send)
  DevBuf<char> rmail;                  // my impulse mailbox: [2 transfers][world] slots of RMAIL_SLOT bytes (allocated at create)
  std::vector<char *> rmail_tx;        // [rank] every rank's mailbox as mapped here ([my rank] = rmail); not owned
  std::vector<bool> rmail_ipc;         // [rank] rmail_tx was opened from an IPC handle (closed by mpmb_destroy)
  DevBuf<char *> rmail_dev;            // rmail_tx on the device
  int64_t id_span_pending = 0;
  int64_t id_span = 0;   // ids of the resident particles lie in [id_base, id_base + id_span): uploads number 0..n-1, the seeded
                         // lattice numbers by lattice index (gaps where the boundary band is skipped)
  int64_t id_end = 0;    // every id this engine has handed out or seen handed out lies below id_end (absolute, not relative to
                         // id_base): on a z-slab rank it covers the whole seeded lattice and every batch appended on any rank

  // AsyncMPM pools (mpmb_async_*): [0] particle_pool, [1] backup_pool, each double-buffered for the stable edits
  struct APool {
    DevBuf<float> buf[2];   // record layout (arec_of), both of the same capacity
    int cur = 0;
    int64_t n = 0;
    ARec rec(int b) const { return arec_of(buf[b]); }
  };
  bool async_on = false;
  int anb[3] = {};
  int nblk = 0;
  float a_inv_dx = 0.f;
  APool apool[2];
  DevBuf<uint8_t> a_bfl;                                            // [nblk] MPMB_ASYNC_* flags of the current advance
  DevBuf<uint32_t> a_bflag;                                         // [nblk] block reductions of mpmb_async_block_limits
  DevBuf<int> a_bmin, a_bmax;
  DevBuf<int> a_blk;                                                // [nblk] compacted block list
  DevBuf<float> a_lim;                                              // [2 nblk] compacted min_dt, max_v2
  DevBuf<int> a_bad;
  DevBuf<float> a_gbuf, a_sbuf;                                     // gathered set / survivors (record layout)
  DevBuf<unsigned long long> a_key[2];                              // gather: candidate keys, candidate / id / position lists
  DevBuf<uint32_t> a_u[4];
  DevBuf<int> a_rowk;                                               // its size is the candidate capacity
  DevBuf<unsigned char> a_cub;
  DevBuf<int> a_level, a_lvnew;                                     // [nblk] the device scheduler's block levels, their update
  DevBuf<long long> a_local_min, a_particle_t, a_backup_t;          // [nblk] its block clocks
  DevBuf<ASched> a_sched;                                           // its reductions and error word

  bool profiling = false;
  struct Ev { cudaEvent_t a, b; int stage; };
  std::vector<Ev> events;
  size_t events_used = 0;
  double prof_ms[MPMB_N_STAGES] = {};
  int64_t prof_launches[MPMB_N_STAGES] = {};
};

static thread_local std::string g_create_error;

static int fail(MpmbEngine *h, int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (h) h->err = buf;
  else g_create_error = buf;
  return code;
}

#define CUDA_TRY(h, expr)                                                                      \
  do {                                                                                         \
    cudaError_t e_ = (expr);                                                                   \
    if (e_ != cudaSuccess) {                                                                   \
      (h)->sticky_cuda = true;                                                                 \
      return fail((h), MPMB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
    }                                                                                          \
  } while (0)

#define CHECK_HANDLE(h)                                                       \
  do {                                                                        \
    if (!(h)) return fail(nullptr, MPMB_ERR_INVALID, "null handle");          \
    if ((h)->sticky_cuda) return MPMB_ERR_CUDA;                               \
    cudaError_t e0_ = cudaSetDevice((h)->cfg.device);                         \
    if (e0_ != cudaSuccess) return fail((h), MPMB_ERR_CUDA, "cudaSetDevice"); \
  } while (0)

static void graph_reset(MpmbEngine *h) {
  for (int p = 0; p < 2; p++)
    if (h->graph_exec[p]) { cudaGraphExecDestroy(h->graph_exec[p]); h->graph_exec[p] = nullptr; }
}

static View make_view(MpmbEngine *h) {
  View V{};
  for (int k = 0; k < N_Q; k++) {
    V.q[k] = h->q[h->cur][k].get();
    V.qn[k] = h->q[h->cur ^ 1][k].get();
  }
  V.keys = h->keys[h->cur].get();
  V.keys_next = h->keys[h->cur ^ 1].get();
  V.outpos = h->outpos.get();
  V.run_begin = h->run_begin[h->ord].get();
  V.run_len = h->run_len[h->ord].get();
  V.out_begin = h->run_begin[h->ord ^ 1].get();
  V.total = h->run_len[h->ord ^ 1].get();
  V.stay_cnt = h->stay[h->ord].get();
  V.stay_next = h->stay[h->ord ^ 1].get();
  V.arr_cnt = h->arr_cnt.get();
  V.arr_off = h->arr_off.get();
  V.arr_len = h->arr_len.get();
  V.arr_cur = h->arr_cur.get();
  V.slot_map = h->slot_map.get();
  V.meta = h->meta.get();
  V.mover_dst = h->mover_dst[h->mov].get();
  V.mover_idx = h->mover_idx[h->mov].get();
  V.mover_dst_n = h->mover_dst[h->mov ^ 1].get();
  V.mover_idx_n = h->mover_idx[h->mov ^ 1].get();
  V.arrivals = h->arrivals.get();
  V.arrivals_sorted = h->arrivals_sorted.get();
  V.blocksum = h->blocksum.get();
  V.arena = h->arena.get();
  V.sdf4 = h->sdf4.get();
  V.cnt = h->cnt.get();
  V.cap_tiles = h->cap_tiles;
  V.cap_particles = (int)h->cap;
  V.rigid_flag = h->rigid_on ? h->tile_flag.get() : nullptr;
  return V;
}

// The by-id colour arrays (p_states, p_cdf, p_mark) are indexed by id - rigid_id0 and must cover rigid_ids ids.  One engine:
// the ids of its resident set, relative to id_base.  z-slab rank: ABSOLUTE ids below the id end, because a rank also holds
// immigrants whose ids lie below its own id_base; the id end then has to cover the run's ids (include/mpmb.h).
static uint32_t rigid_id0(const MpmbEngine *h) { return h->cfg.world > 1 ? 0u : h->id_base; }
static int64_t rigid_ids(const MpmbEngine *h) { return h->cfg.world > 1 ? std::max<int64_t>(h->id_end, h->id_base) : h->id_span; }
static StateWords state_words(MpmbEngine *h) {   // what the migration and re-cut records carry (nothing without rigid coupling)
  StateWords S{};
  if (h->rigid_on && h->p_states.get()) { S.w = h->p_states.get(); S.n = (int)h->p_states.size(); }
  return S;
}

// the rigid coupling and the device-advanced bodies as the kernels take them, built at every launch as make_view is
static RigidView rigid_view(MpmbEngine *h) {
  RigidView R{};
  R.bodies = h->bodies.get();
  R.n_bodies = h->rigid_bodies;
  R.n_samples = h->rigid_samples;
  R.s_offset = h->rs_offset.get(); R.s_tri = h->rs_tri.get(); R.s_rigid = h->rs_rigid.get();
  R.s_base = h->s_base.get();
  R.node_key = h->node_key.get();
  R.node_tags = h->node_tags.get();
  R.page = h->page.get();
  for (int d = 0; d < 3; d++) R.nb[d] = h->rigid_nb[d];
  R.tile_flag = h->tile_flag.get();
  R.p_states = h->p_states.get(); R.p_cdf = h->p_cdf.get(); R.p_mark = h->p_mark.get();
  R.epoch = h->epoch.get();
  R.id_base = rigid_id0(h);
  R.id_cap = (int)h->p_states.size();
  R.penalty = h->penalty;
  R.pushing_force = h->pushing_force;
  return R;
}
static MotionView motion_view(MpmbEngine *h) {
  MotionView M{};
  M.m = h->master.get();
  M.script = h->script.get();
  M.cursor = h->cursor.get();
  M.s_order = h->s_order.get();
  for (int b = 0; b <= RIGID_MAX; b++) M.s_begin[b] = h->s_begin[b];
  M.contact = h->contact.get();
  M.collide = h->motion_collide && h->P.has_sdf;   // without a level set there are no contacts: the advance must not read the buffer
  return M;                                        // (changing the level set resets the captured graphs)
}

static void prof_begin(MpmbEngine *h, int stage) {
  if (!h->profiling) return;
  if (h->events_used == h->events.size()) {
    MpmbEngine::Ev e{};
    cudaEventCreate(&e.a);
    cudaEventCreate(&e.b);
    h->events.push_back(e);
  }
  h->events[h->events_used].stage = stage;
  cudaEventRecord(h->events[h->events_used].a, h->stream);
}
static void prof_end(MpmbEngine *h, int n_launches) {
  if (!h->profiling) return;
  cudaEventRecord(h->events[h->events_used].b, h->stream);
  h->prof_launches[h->events[h->events_used].stage] += n_launches;
  h->events_used++;
}
static void prof_collect(MpmbEngine *h) {
  for (size_t i = 0; i < h->events_used; i++) {
    float ms = 0.f;
    cudaEventSynchronize(h->events[i].b);
    cudaEventElapsedTime(&ms, h->events[i].a, h->events[i].b);
    h->prof_ms[h->events[i].stage] += ms;
  }
  h->events_used = 0;
}

// Frees every particle-row buffer, then allocates them for `cap` rows: a reallocation never holds the old and the new set.
static int alloc_particles(MpmbEngine *h, int64_t cap) {
  graph_reset(h);
  for (int b = 0; b < 2; b++) {
    for (auto &q : h->q[b]) q.reset();
    h->keys[b].reset(); h->mover_dst[b].reset(); h->mover_idx[b].reset();
  }
  h->outpos.reset(); h->arrivals.reset(); h->arrivals_sorted.reset(); h->keys_sorted.reset(); h->iota.reset(); h->cub_temp.reset();
  h->cap = 0;
  if (cap >= (1ll << 30)) return fail(h, MPMB_ERR_CAPACITY, "capacity %lld exceeds 2^30 particle rows per GPU", (long long)cap);
  if (cap < 1) cap = 1;
  for (int b = 0; b < 2; b++) {
    for (auto &q : h->q[b]) CUDA_TRY(h, q.alloc(cap));
    CUDA_TRY(h, h->keys[b].alloc(cap));
    CUDA_TRY(h, h->mover_dst[b].alloc(cap));
    CUDA_TRY(h, h->mover_idx[b].alloc(cap));
  }
  CUDA_TRY(h, h->outpos.alloc(cap + 8));  // the bulk copy of a run's words is widened to 16-byte bounds
  CUDA_TRY(h, h->arrivals.alloc(cap));
  CUDA_TRY(h, h->arrivals_sorted.alloc(cap));
  CUDA_TRY(h, h->keys_sorted.alloc(cap));
  CUDA_TRY(h, h->iota.alloc(cap));
  k_iota<<<(unsigned)((cap + 255) / 256), 256, 0, h->stream>>>(h->iota.get(), (int)cap);
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, h->keys[0].get(), h->keys_sorted.get(), h->iota.get(), h->arrivals_sorted.get(), (int)cap, 0, 32, h->stream);
  CUDA_TRY(h, h->cub_temp.alloc(cub_bytes));
  h->cap = cap;
  return MPMB_OK;
}

// The dense tile grid of an engine that owns tile layers [z0, z1) of the domain: on a z-slab rank its own layers plus one
// ghost layer on each side, on world == 1 the whole domain; the keys of that grid and the ordering's block count.
// mpmb_create sizes an engine with it, mpmb_recut_apply re-slices one.
struct Slicing {
  int tz_off, nt2, tile_z0, tile_z1, ntot, key_bits, ord_blocks;
};
static bool slab_slicing(const Params &P, int nt2_global, int world, int z0, int z1, Slicing *s) {
  s->tz_off = 0; s->nt2 = nt2_global; s->tile_z0 = 0; s->tile_z1 = nt2_global;
  if (world > 1) {
    s->tz_off = z0 - 1;    // one ghost layer below ...
    s->nt2 = z1 - z0 + 2;  // ... and one above the owned layers
    s->tile_z0 = z0; s->tile_z1 = z1;
  }
  const unsigned long long ntot = (unsigned long long)P.nt[0] * P.nt[1] * s->nt2;
  s->key_bits = 1;
  while ((1ull << s->key_bits) <= ntot + SPECIAL_DEAD) s->key_bits++;
  if (s->key_bits > 31) return false;  // tile grid too large for 32-bit keys
  s->ntot = (int)ntot;
  s->ord_blocks = (int)((ntot + ORD_TILE - 1) / ORD_TILE);
  return true;
}
static void set_slicing(MpmbEngine *h, const Slicing &s) {
  Params &P = h->P;
  P.tz_off = s.tz_off; P.nt[2] = s.nt2; P.tile_z0 = s.tile_z0; P.tile_z1 = s.tile_z1; P.ntiles_total = s.ntot;
  h->ntot = s.ntot;
  h->special_min = (uint32_t)s.ntot;
  h->key_dead = (uint32_t)s.ntot + SPECIAL_DEAD;
  h->key_bits = s.key_bits;
  h->ord_blocks = s.ord_blocks;
}

// Dense per-tile arrays, active-tile records, arenas (plus the all-zero arena read for absent neighbours, past the last
// slot) and the ordering's block sums for `cap_tiles` tiles.  All or nothing: on failure the engine keeps
// the arrays it had.
static int alloc_tile_arrays(MpmbEngine *h, int64_t cap_tiles) {
  DevBuf<int> dense[11], blocksum;
  DevBuf<TileMeta> meta;
  DevBuf<float4> arena;
  const int64_t blocks = (cap_tiles + ORD_TILE - 1) / ORD_TILE;
  bool ok = true;
  for (auto &d : dense) ok = ok && d.alloc(cap_tiles) == cudaSuccess;
  ok = ok && blocksum.alloc(3 * (blocks + 1)) == cudaSuccess;
  ok = ok && meta.alloc(cap_tiles) == cudaSuccess;
  ok = ok && arena.alloc((size_t)ARENA * (cap_tiles + 1)) == cudaSuccess;
  if (!ok) return fail(h, MPMB_ERR_CUDA, "cudaMalloc of the tile arrays (%lld tiles): %s", (long long)cap_tiles, cudaGetErrorString(cudaGetLastError()));
  for (auto &d : dense) cudaMemsetAsync(d.get(), 0, sizeof(int) * cap_tiles, h->stream);
  cudaMemsetAsync(arena.get() + (size_t)ARENA * cap_tiles, 0, sizeof(float4) * ARENA, h->stream);
  DevBuf<int> *mine[] = {&h->run_begin[0], &h->run_begin[1], &h->run_len[0], &h->run_len[1], &h->stay[0], &h->stay[1],
                         &h->arr_cnt, &h->arr_off, &h->arr_len, &h->arr_cur, &h->slot_map};
  for (int k = 0; k < 11; k++) *mine[k] = std::move(dense[k]);
  cudaMemsetAsync(h->slot_map.get(), 0xFF, sizeof(int) * cap_tiles, h->stream);
  h->blocksum = std::move(blocksum); h->meta = std::move(meta); h->arena = std::move(arena);
  h->cap_tiles = (int)cap_tiles;
  return MPMB_OK;
}

// entry points that a 2-D handle does not have (include/mpmb.h lists what it has)
#define NOT_2D(h) \
  if ((h)->m2) return fail((h), MPMB_ERR_STATE, "%s is not available on a 2-D handle (dim = 2)", __func__)

// =====================================================================================
// The 2-D engine (MpmbConfig.dim == 2): MPM<2>::substep() of the reference (src/mpm.cpp:452-575) with the scalar
// transfers MPM<2> runs (rasterize / resample, src/transfer.cpp:193-284, 585-701).  It sits after the handle type; the
// C-ABI entry points route a 2-D handle here.  None of the 3-D tiles, arenas or orderings is used.
//
// Layout (DESIGN.md §10): particles are SoA, double buffered: x float2, v float2, F float4 and b float4
// (column-major 2x2), aux float4 = (mass, vol, scalar, tag) with tag = group << 28 | id.  One substep is
//   ordering  radix sort of the rows by the cell of their base node (dead rows last), a permutation into the other
//             buffer and the [begin, end) row range of every cell;
//   P2G       one thread per particle forms (X, m v, A = apic_b (4 m) - stress (4 dt / dx)); then one thread per node
//             sums the particles of the 3x3 cells whose stencil covers it, in storage order, and finishes the node in
//             place: normalise, gravity, level-set boundary.  No atomics: results are bit-reproducible;
//   G2P       one thread per particle: gather, apic_b (damped), the 2x2 constitutive step, advection, the position
//             clamp and the deletion rule, which writes the next ordering's key.
// Nothing crosses the bus between substeps; mpmb_substep replays one captured substep per buffer parity.

namespace mpmb {

constexpr int M2_TILE = 16;  // node tile edge of the grid kernel (16 x 16 nodes = 256 threads)

struct Params2 {
  int res[2], nnode[2];
  int ncells;  // res0 * res1; the key of a dead row
  float dx, inv_dx, dt;
  float gdt[2];  // gravity * dt
  int particle_gravity, clean_boundary;
  float friction;
  int has_sdf;
  float apic_damping, rpic_damping;
  Material mats[MPMB_MAX_GROUPS];
};

struct Counters2 {
  int n_alive;  // live rows after the last ordering
  int n_live;   // scratch of mpmb_num_particles
  int error;
  int aos_error;  // error bits of the running mpmb_upload_aos / mpmb_download_aos: that call reports them and changes nothing
  unsigned long long updates;
};

struct View2 {
  float2 *x, *v;
  float4 *F, *b, *aux;
  float2 *xn, *vn;  // the other buffer (written by the ordering)
  float4 *Fn, *bn, *auxn;
  uint32_t *keys, *keys_sorted, *perm;
  int *cell_begin, *cell_end;
  float4 *pa, *pb;  // P2G records: (X, Y, m vx, m vy), affine (column-major)
  float *pm;
  float4 *graw;     // (p_x, p_y, 0, m) after P2G
  float2 *gv;       // node velocity after normalise + boundary
  const float4 *sdf4;
  Counters2 *cnt;
};

__device__ __forceinline__ uint32_t cell_key2(const Params2 &P, float2 x) {
  const float X = __fmul_rn(x.x, P.inv_dx), Y = __fmul_rn(x.y, P.inv_dx);
  if (!isfinite(X) || !isfinite(Y)) return (uint32_t)P.ncells;
  const int bx = (int)__fsub_rn(X, 0.5f), by = (int)__fsub_rn(Y, 0.5f);
  // the 9-node stencil [base, base+2] must stay on the node grid
  if (bx < 0 || by < 0 || bx + 2 > P.res[0] || by + 2 > P.res[1]) return (uint32_t)P.ncells;
  return (uint32_t)(bx * P.res[1] + by);
}

__global__ void k2_pack(View2 V, Params2 P, int n, const float *x, const float *v, const float *F, const float *b, const float *mass,
                        const float *vol, const float *scalar, const int *group, uint32_t id0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int g = group ? group[i] : 0;
  float m = mass[i];
  if (g < 0 || g >= MPMB_MAX_GROUPS || !(m > 0.f)) {
    atomicOr(&V.cnt->error, DEVERR_BAD_INPUT);
    g = min(max(g, 0), MPMB_MAX_GROUPS - 1);
    m = 1e-30f;
  }
  float ps;
  if (scalar) ps = scalar[i];
  else ps = (P.mats[g].kind == MAT_SNOW || P.mats[g].kind == MAT_WATER) ? 1.0f : 0.0f;  // Jp = 1, j = 1, logJp = 0
  const float2 xx = make_float2(x[2 * (size_t)i], x[2 * (size_t)i + 1]);
  V.x[i] = xx;
  V.v[i] = make_float2(v[2 * (size_t)i], v[2 * (size_t)i + 1]);
  V.F[i] = F ? make_float4(F[4 * (size_t)i], F[4 * (size_t)i + 1], F[4 * (size_t)i + 2], F[4 * (size_t)i + 3]) : make_float4(1.f, 0.f, 0.f, 1.f);
  V.b[i] = b ? make_float4(b[4 * (size_t)i], b[4 * (size_t)i + 1], b[4 * (size_t)i + 2], b[4 * (size_t)i + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
  V.aux[i] = make_float4(m, vol[i], ps, __uint_as_float(((uint32_t)g << TAG_ID_BITS) | (id0 + (uint32_t)i)));
  V.keys[i] = cell_key2(P, xx);
}

// ---------------------------------------------------------------- AoS pools
// mpmb_upload_aos: slot indices[k] of the device image of the reference's pool (MPMParticle<2>: pos float[2], v_and_m
// float[3] = (vx, vy, mass), dg_e and apic_b as two columns of two floats col_pitch apart) -> row k, the row k2_pack makes
// of the same particle given field-wise.  The rows go to the spare buffers and the keys to keys_sorted; the host keeps them
// only when no slot lies outside the pool.  Every error bit goes to cnt->aos_error.
__global__ void k2_pack_aos(View2 V, Params2 P, int n, const unsigned char *pool, int64_t pool_slots, const uint32_t *indices, MpmbAosLayout L,
                            AosScalars S, const int *group, uint32_t id0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t slot = indices[i];
  if ((int64_t)slot >= pool_slots) { atomicOr(&V.cnt->aos_error, DEVERR_BAD_SLOT); return; }
  const unsigned char *s = pool + (size_t)slot * L.stride;
  const float *pos = (const float *)(s + L.off_pos), *vm = (const float *)(s + L.off_v_and_m);
  const float *f0 = (const float *)(s + L.off_dg_e), *f1 = (const float *)(s + L.off_dg_e + L.col_pitch);
  const float *b0 = (const float *)(s + L.off_apic_b), *b1 = (const float *)(s + L.off_apic_b + L.col_pitch);
  int g = group ? group[i] : 0;
  float m = vm[2];
  if (g < 0 || g >= MPMB_MAX_GROUPS || !(m > 0.f)) {
    atomicOr(&V.cnt->aos_error, DEVERR_BAD_INPUT);
    g = min(max(g, 0), MPMB_MAX_GROUPS - 1);
    m = 1e-30f;
  }
  float ps;
  if (S.on) ps = S.off[g] >= 0 ? *(const float *)(s + S.off[g]) : S.dflt[g];
  else ps = L.off_scalar >= 0 ? *(const float *)(s + L.off_scalar) : 0.f;
  const float2 xx = make_float2(pos[0], pos[1]);
  V.xn[i] = xx;
  V.vn[i] = make_float2(vm[0], vm[1]);
  V.Fn[i] = make_float4(f0[0], f0[1], f1[0], f1[1]);
  V.bn[i] = make_float4(b0[0], b0[1], b1[0], b1[1]);
  V.auxn[i] = make_float4(m, *(const float *)(s + L.off_vol), ps, __uint_as_float(((uint32_t)g << TAG_ID_BITS) | (id0 + (uint32_t)i)));
  V.keys_sorted[i] = cell_key2(P, xx);
}

// mpmb_download_aos: every live row back into its slot of the device image (slot = indices[id - id_base]) and the alive
// flag of its id; the survivors' slots in id order are then one stream compaction away (k_compact_survivors).  Dead rows
// write nothing.  An id or slot outside the vectors sets DEVERR_BAD_SLOT in cnt->aos_error and writes nothing.
__global__ void k2_aos_scatter(View2 V, Params2 P, int n, unsigned char *pool, const uint32_t *indices, int64_t n_indices, int64_t pool_slots,
                               MpmbAosLayout L, AosScalars S, uint32_t id_base, int *alive_flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || V.keys[i] >= (uint32_t)P.ncells) return;
  const float4 aux = V.aux[i];
  const uint32_t tag = __float_as_uint(aux.w), id = (tag & TAG_ID_MASK) - id_base;
  if ((int64_t)id >= n_indices) { atomicOr(&V.cnt->aos_error, DEVERR_BAD_SLOT); return; }
  const uint32_t slot = indices[id];
  if ((int64_t)slot >= pool_slots) { atomicOr(&V.cnt->aos_error, DEVERR_BAD_SLOT); return; }
  alive_flag[id] = 1;
  const float2 x = V.x[i], v = V.v[i];
  const float4 F = V.F[i], b = V.b[i];
  unsigned char *sl = pool + (size_t)slot * L.stride;
  float *pos = (float *)(sl + L.off_pos), *vm = (float *)(sl + L.off_v_and_m);
  float *f0 = (float *)(sl + L.off_dg_e), *f1 = (float *)(sl + L.off_dg_e + L.col_pitch);
  float *b0 = (float *)(sl + L.off_apic_b), *b1 = (float *)(sl + L.off_apic_b + L.col_pitch);
  pos[0] = x.x; pos[1] = x.y;
  vm[0] = v.x; vm[1] = v.y; vm[2] = aux.x;
  f0[0] = F.x; f0[1] = F.y; f1[0] = F.z; f1[1] = F.w;
  b0[0] = b.x; b0[1] = b.y; b1[0] = b.z; b1[1] = b.w;
  if (S.on) {
    const int32_t off = S.off[tag >> TAG_ID_BITS];
    if (off >= 0) *(float *)(sl + off) = aux.z;
  } else if (L.off_scalar >= 0) {
    *(float *)(sl + L.off_scalar) = aux.z;
  }
}

// ---------------------------------------------------------------- ordering
__global__ void k2_permute(View2 V, Params2 P, int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t key = V.keys_sorted[j];
  V.keys[j] = key;
  if (key >= (uint32_t)P.ncells) return;
  const uint32_t s = V.perm[j];
  V.xn[j] = V.x[s];
  V.vn[j] = V.v[s];
  V.Fn[j] = V.F[s];
  V.bn[j] = V.b[s];
  V.auxn[j] = V.aux[s];
}
// [begin, end) of every cell from the sorted keys (cells without particles keep the memset 0, 0) and the live count
__global__ void k2_cells(View2 V, Params2 P, int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t dead = (uint32_t)P.ncells, k = V.keys_sorted[j];
  const uint32_t prev = j > 0 ? V.keys_sorted[j - 1] : 0xffffffffu;
  const uint32_t next = j + 1 < n ? V.keys_sorted[j + 1] : dead;
  if (k < dead) {
    if (k != prev) V.cell_begin[k] = j;
    if (k != next) V.cell_end[k] = j + 1;
    if (next >= dead) V.cnt->n_alive = j + 1;
  } else if (j == 0) {
    V.cnt->n_alive = 0;
  }
}

// ---------------------------------------------------------------- P2G
// MPM<2>::rasterize(dt, true) (src/transfer.cpp:193-278) without rigid bodies: the particle gravity kick, then per node
// w (m v + apic_b (inv_D m) dpos - (dt force) dpos 4 inv_dx, m) with dpos = X - node in grid units
__global__ void __launch_bounds__(256) k2_p2g_particles(View2 V, Params2 P, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) V.cnt->updates += (unsigned long long)V.cnt->n_alive;  // update_counter += particles.size() (src/mpm.cpp:436)
  if (i >= n || V.keys[i] >= (uint32_t)P.ncells) return;
  const float2 x = V.x[i];
  float2 v = V.v[i];
  const float4 f = V.F[i], b = V.b[i], aux = V.aux[i];
  if (P.particle_gravity) v = make_float2(v.x + P.gdt[0], v.y + P.gdt[1]);
  const int g = (int)(__float_as_uint(aux.w) >> TAG_ID_BITS);
  const Mat2 F = {{f.x, f.y, f.z, f.w}};
  const Mat2 force = calculate_force2(P.mats[g], F, aux.z, aux.y);
  const float m = aux.x, bm = 4.0f * m, S = -4.0f * P.inv_dx * P.dt;  // Kernel::inv_D() = 4
  V.pa[i] = make_float4(__fmul_rn(x.x, P.inv_dx), __fmul_rn(x.y, P.inv_dx), m * v.x, m * v.y);
  V.pb[i] = make_float4(fmaf(force.m[0], S, b.x * bm), fmaf(force.m[1], S, b.y * bm), fmaf(force.m[2], S, b.z * bm), fmaf(force.m[3], S, b.w * bm));
  V.pm[i] = m;
}

// One thread per node: the fixed-order sum over the particles of cells [i-2, i] x [j-2, j], then
// normalize_grid_and_apply_external_force and apply_grid_boundary_conditions (src/mpm.cpp:277-372), static level set.
__global__ void __launch_bounds__(256) k2_grid(View2 V, Params2 P, int tiles1) {
  const int t = threadIdx.x;
  const int i = (blockIdx.x / tiles1) * M2_TILE + (t >> 4), j = (blockIdx.x % tiles1) * M2_TILE + (t & 15);
  if (i >= P.nnode[0] || j >= P.nnode[1]) return;
  float px = 0.f, py = 0.f, m = 0.f;
  for (int cx = max(i - 2, 0); cx <= min(i, P.res[0] - 1); cx++)
    for (int cy = max(j - 2, 0); cy <= min(j, P.res[1] - 1); cy++) {
      const int c = cx * P.res[1] + cy, e = V.cell_end[c];
      for (int r = V.cell_begin[c]; r < e; r++) {
        const float4 a = V.pa[r], A = V.pb[r];
        int bx, by;
        float wx[3], wy[3];
        quadratic_weights2(a.x, bx, wx);
        quadratic_weights2(a.y, by, wy);
        const float w = wx[i - cx] * wy[j - cy];
        const float dx = a.x - (float)i, dy = a.y - (float)j;
        px += w * fmaf(A.z, dy, fmaf(A.x, dx, a.z));
        py += w * fmaf(A.w, dy, fmaf(A.y, dx, a.w));
        m += w * V.pm[r];
      }
    }
  const size_t node = (size_t)i * P.nnode[1] + j;
  V.graw[node] = make_float4(px, py, 0.f, m);
  float2 vel = make_float2(px, py);
  if (m > 0.f) {
    const float inv = 1.0f / m;
    const float ix = P.particle_gravity ? 0.f : P.gdt[0], iy = P.particle_gravity ? 0.f : P.gdt[1];
    vel = make_float2(fmaf(px, inv, ix), fmaf(py, inv, iy));
  }
  if (P.has_sdf && m != 0.f) {
    const float4 s = V.sdf4[node];
    if (!(s.w < -3.f || 0.f < s.w)) vel = friction_project2(vel, make_float2(s.x, s.y), P.friction);
  }
  V.gv[node] = vel;
}

// ---------------------------------------------------------------- G2P
// MPM<2>::resample() (src/transfer.cpp:585-687) without rigid bodies, then the deletion rule: clean_boundary = 1 deletes
// in the 7-cell band (near_boundary, src/mpm.h:269-276) and non-finite particles (src/mpm.cpp:583-633); clean_boundary = 0
// deletes a particle whose 9-node stencil leaves the node grid or whose position or velocity is not finite.
__global__ void __launch_bounds__(256) k2_g2p(View2 V, Params2 P, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || V.keys[i] >= (uint32_t)P.ncells) return;
  float2 x = V.x[i];
  const float4 f = V.F[i];
  float4 aux = V.aux[i];
  const float X = __fmul_rn(x.x, P.inv_dx), Y = __fmul_rn(x.y, P.inv_dx);
  int bx, by;
  float wx[3], wy[3];
  quadratic_weights2(X, bx, wx);
  quadratic_weights2(Y, by, wy);
  float vx = 0.f, vy = 0.f;
  Mat2 B = {{0.f, 0.f, 0.f, 0.f}};
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const float2 gv = V.gv[(size_t)(bx + a) * P.nnode[1] + (by + c)];
      const float w = wx[a] * wy[c];
      const float dx = X - (float)(bx + a), dy = Y - (float)(by + c);
      const float wgx = w * gv.x, wgy = w * gv.y;
      vx += wgx;
      vy += wgy;
      B.m[0] = fmaf(wgx, dx, B.m[0]);
      B.m[1] = fmaf(wgy, dx, B.m[1]);
      B.m[2] = fmaf(wgx, dy, B.m[2]);
      B.m[3] = fmaf(wgy, dy, B.m[3]);
    }
  // apic_b = damp_affine_momemtum(b) = (1 - rpic) sym(b) + (1 - apic) skew(b) (src/mpm.h:465-469)
  const float sym_o = 0.5f * (B.m[1] + B.m[2]);
  const float kr = 1.f - P.rpic_damping, ka = 1.f - P.apic_damping;
  const float4 bd = make_float4(kr * B.m[0], kr * sym_o + ka * (B.m[1] - sym_o), kr * sym_o + ka * (B.m[2] - sym_o), kr * B.m[3]);
  // cdg = I + dt (b (-4 inv_dx)) of the undamped b
  const float S = -4.f * P.inv_dx;
  Mat2 cdg;
  cdg.m[0] = 1.f + P.dt * (B.m[0] * S);
  cdg.m[1] = P.dt * (B.m[1] * S);
  cdg.m[2] = P.dt * (B.m[2] * S);
  cdg.m[3] = 1.f + P.dt * (B.m[3] * S);
  const int g = (int)(__float_as_uint(aux.w) >> TAG_ID_BITS);
  Mat2 F = {{f.x, f.y, f.z, f.w}};
  plasticity2(P.mats[g], cdg, F, aux.z);
  x = make_float2(x.x + P.dt * vx, x.y + P.dt * vy);
  const bool finite = isfinite(x.x) && isfinite(x.y) && isfinite(vx) && isfinite(vy);
  // position correction: (pos inv_dx).clamp(0, res - eps) dx, eps = 1e-6
  x.x = fminf(fmaxf(x.x * P.inv_dx, 0.f), (float)P.res[0] - 1e-6f) * P.dx;
  x.y = fminf(fmaxf(x.y * P.inv_dx, 0.f), (float)P.res[1] - 1e-6f) * P.dx;
  bool dead = !finite;
  if (P.clean_boundary) {
    const float Xn = x.x * P.inv_dx, Yn = x.y * P.inv_dx;
    dead |= fminf(Xn, Yn) < 7.0f || fmaxf(Xn - (float)P.res[0], Yn - (float)P.res[1]) > -7.0f;
  }
  V.x[i] = x;
  V.v[i] = make_float2(vx, vy);
  V.F[i] = make_float4(F.m[0], F.m[1], F.m[2], F.m[3]);
  V.b[i] = bd;
  V.aux[i] = aux;
  V.keys[i] = dead ? (uint32_t)P.ncells : cell_key2(P, x);
}

__global__ void __launch_bounds__(256) k2_count_live(const uint32_t *keys, int n, uint32_t dead, Counters2 *cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && keys[i] < dead) atomicAdd(&cnt->n_live, 1);
}

// the level set of 2-D solids: mpmb_set_planes / mpmb_set_levelset_shapes with zero z parts, node (n_x, n_y, 0, phi)
__global__ void k2_shapes_to_sdf(Params2 P, int n_shapes, const MpmbShape *shapes, float4 *sdf4) {
  const size_t n = (size_t)P.nnode[0] * P.nnode[1];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int gx = (int)(i / P.nnode[1]), gy = (int)(i % P.nnode[1]);
    float4 best = make_float4(1.f, 0.f, 0.f, 1e30f);
    for (int k = 0; k < n_shapes; k++) {
      const float4 c = shape_sdf(shapes[k], (float)gx, (float)gy, 0.f);
      if (c.w < best.w) best = c;
    }
    sdf4[i] = best;
  }
}

}  // namespace mpmb

// ================================================================================================ host side
struct Mpm2d {
  Params2 P{};
  int64_t cap = 0;   // rows allocated per buffer
  int64_t rows = 0;  // rows of the current storage (the last upload's n); dead rows keep the dead key
  int cur = 0;
  int stage = 0;     // 0 idle / after G2P, 1 after the ordering, 2 after P2G
  int key_bits = 32;
  uint32_t id_base = 0;
  DevBuf<float2> x[2], v[2];
  DevBuf<float4> F[2], b[2], aux[2];
  DevBuf<uint32_t> keys, keys_sorted, perm, iota;
  DevBuf<unsigned char> cub_temp;
  DevBuf<int> cell_begin, cell_end;
  DevBuf<float4> pa, pb, graw, sdf4;
  DevBuf<float> pm;
  DevBuf<float2> gv;
  DevBuf<Counters2> cnt;
  DevBuf<float> stage_buf;
  cudaGraphExec_t graph[2] = {nullptr, nullptr};
  int graph_launches = 0;
};

static void m2_graph_reset(Mpm2d *m) {
  for (int p = 0; p < 2; p++)
    if (m->graph[p]) { cudaGraphExecDestroy(m->graph[p]); m->graph[p] = nullptr; }
}

static View2 m2_view(MpmbEngine *h) {
  Mpm2d *m = h->m2;
  View2 V{};
  const int c = m->cur, o = c ^ 1;
  V.x = m->x[c].get(); V.v = m->v[c].get(); V.F = m->F[c].get(); V.b = m->b[c].get(); V.aux = m->aux[c].get();
  V.xn = m->x[o].get(); V.vn = m->v[o].get(); V.Fn = m->F[o].get(); V.bn = m->b[o].get(); V.auxn = m->aux[o].get();
  V.keys = m->keys.get(); V.keys_sorted = m->keys_sorted.get(); V.perm = m->perm.get();
  V.cell_begin = m->cell_begin.get(); V.cell_end = m->cell_end.get();
  V.pa = m->pa.get(); V.pb = m->pb.get(); V.pm = m->pm.get();
  V.graw = m->graw.get(); V.gv = m->gv.get();
  V.sdf4 = m->sdf4.get();
  V.cnt = m->cnt.get();
  return V;
}

static unsigned m2_blocks(int64_t n, int t) { return (unsigned)std::max<int64_t>(1, (n + t - 1) / t); }

static int m2_create(MpmbEngine *h, const MpmbConfig *cfg) {
  Mpm2d *m = new Mpm2d();
  h->m2 = m;
  Params2 &P = m->P;
  for (int d = 0; d < 2; d++) {
    P.res[d] = cfg->res[d];
    P.nnode[d] = cfg->res[d] + 1;
    P.gdt[d] = cfg->gravity[d] * cfg->dt;
  }
  P.ncells = cfg->res[0] * cfg->res[1];
  P.dx = cfg->dx;
  P.inv_dx = 1.0f / cfg->dx;
  P.dt = cfg->dt;
  P.particle_gravity = cfg->particle_gravity;
  P.clean_boundary = cfg->clean_boundary;
  P.apic_damping = cfg->apic_damping;
  P.rpic_damping = cfg->rpic_damping;
  for (int g = 0; g < MPMB_MAX_GROUPS; g++) P.mats[g] = h->P.mats[g];  // the default material of mpmb_create
  m->key_bits = 1;
  while ((1ll << m->key_bits) <= (int64_t)P.ncells) m->key_bits++;
  const size_t nodes = (size_t)P.nnode[0] * P.nnode[1];
  if (m->cell_begin.alloc(P.ncells) != cudaSuccess || m->cell_end.alloc(P.ncells) != cudaSuccess || m->graw.alloc(nodes) != cudaSuccess ||
      m->gv.alloc(nodes) != cudaSuccess || m->cnt.alloc(1) != cudaSuccess)
    return fail(nullptr, MPMB_ERR_CUDA, "cudaMalloc of the 2-D grid (%lld nodes): %s", (long long)nodes, cudaGetErrorString(cudaGetLastError()));
  cudaMemset(m->cnt.get(), 0, sizeof(Counters2));
  return MPMB_OK;
}

static void m2_destroy(MpmbEngine *h) {
  if (!h->m2) return;
  m2_graph_reset(h->m2);
  delete h->m2;
  h->m2 = nullptr;
}

static int m2_alloc_rows(MpmbEngine *h, int64_t cap) {
  Mpm2d *m = h->m2;
  m2_graph_reset(m);
  if (cap >= (1ll << 30)) return fail(h, MPMB_ERR_CAPACITY, "capacity %lld exceeds 2^30 particle rows per GPU", (long long)cap);
  cap = std::max<int64_t>(cap, 1);
  for (int b = 0; b < 2; b++) {
    CUDA_TRY(h, m->x[b].alloc(cap)); CUDA_TRY(h, m->v[b].alloc(cap)); CUDA_TRY(h, m->F[b].alloc(cap));
    CUDA_TRY(h, m->b[b].alloc(cap)); CUDA_TRY(h, m->aux[b].alloc(cap));
  }
  CUDA_TRY(h, m->keys.alloc(cap)); CUDA_TRY(h, m->keys_sorted.alloc(cap)); CUDA_TRY(h, m->perm.alloc(cap)); CUDA_TRY(h, m->iota.alloc(cap));
  CUDA_TRY(h, m->pa.alloc(cap)); CUDA_TRY(h, m->pb.alloc(cap)); CUDA_TRY(h, m->pm.alloc(cap));
  k_iota<<<m2_blocks(cap, 256), 256, 0, h->stream>>>(m->iota.get(), (int)cap);
  h->launches++;
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, m->keys.get(), m->keys_sorted.get(), m->iota.get(), m->perm.get(), (int)cap, 0, m->key_bits, h->stream);
  CUDA_TRY(h, m->cub_temp.alloc(std::max<size_t>(bytes, 16)));
  m->cap = cap;
  return MPMB_OK;
}

static int m2_upload(MpmbEngine *h, int64_t n, const float *x, const float *v, const float *F, const float *b, const float *mass,
                     const float *vol, const float *scalar, const int32_t *group) {
  Mpm2d *m = h->m2;
  if (n < 0 || (n > 0 && (!x || !v || !mass || !vol))) return fail(h, MPMB_ERR_INVALID, "x, v, mass, vol are required");
  if ((int64_t)m->id_base + n > (1ll << TAG_ID_BITS)) return fail(h, MPMB_ERR_CAPACITY, "particle ids exceed 2^%d", TAG_ID_BITS);
  if (m->stage != 0) return fail(h, MPMB_ERR_STATE, "upload between substeps, not inside one");
  if (h->cfg.capacity > 0 && n > m->cap) return fail(h, MPMB_ERR_CAPACITY, "%lld particles exceed the configured capacity %lld", (long long)n, (long long)m->cap);
  if (n > m->cap) { int rc = m2_alloc_rows(h, n); if (rc != MPMB_OK) return rc; }
  m2_graph_reset(m);
  h->aos_host_pool = nullptr;   // the resident set is no longer the AoS pool's (mpmb_download_aos needs a new upload)
  h->aos_kinds_valid = false;
  const size_t words = (size_t)n * (2 + 2 + (F ? 4 : 0) + (b ? 4 : 0) + 1 + 1 + (scalar ? 1 : 0) + (group ? 1 : 0));
  CUDA_TRY(h, m->stage_buf.reserve(std::max<size_t>(words, 1)));
  float *p = m->stage_buf.get();
  auto put = [&](const void *src, size_t count) -> float * {
    if (!src) return nullptr;
    float *dst = p;
    cudaMemcpyAsync(dst, src, count * sizeof(float), cudaMemcpyHostToDevice, h->stream);
    p += count;
    return dst;
  };
  const float *dx = put(x, 2 * n), *dv = put(v, 2 * n), *dF = put(F, 4 * n), *db = put(b, 4 * n), *dm = put(mass, n), *dvol = put(vol, n);
  const float *ds = put(scalar, n);
  const int *dg = (const int *)put(group, n);
  CUDA_TRY(h, cudaMemsetAsync(m->cnt.get(), 0, sizeof(int) * 4, h->stream));  // n_alive, n_live, error (updates are kept)
  if (n > 0) {
    k2_pack<<<m2_blocks(n, 128), 128, 0, h->stream>>>(m2_view(h), m->P, (int)n, dx, dv, dF, db, dm, dvol, ds, dg, m->id_base);
    h->launches++;
  }
  m->rows = n;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

// ---- the three stages
static int m2_order(MpmbEngine *h) {
  Mpm2d *m = h->m2;
  if (m->stage != 0) return fail(h, MPMB_ERR_STATE, "stages run in the order sort, rasterize, resample");
  const int n = (int)m->rows;
  prof_begin(h, 0);
  int nl = 0;
  CUDA_TRY(h, cudaMemsetAsync(m->cell_begin.get(), 0, sizeof(int) * (size_t)m->P.ncells, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(m->cell_end.get(), 0, sizeof(int) * (size_t)m->P.ncells, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(m->cnt.get(), 0, sizeof(int), h->stream));  // n_alive
  if (n > 0) {
    size_t bytes = m->cub_temp.size();
    CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(m->cub_temp.get(), bytes, m->keys.get(), m->keys_sorted.get(), m->iota.get(), m->perm.get(), n, 0,
                                                 m->key_bits, h->stream));
    const View2 V = m2_view(h);
    k2_permute<<<m2_blocks(n, 256), 256, 0, h->stream>>>(V, m->P, n);
    k2_cells<<<m2_blocks(n, 256), 256, 0, h->stream>>>(V, m->P, n);
    nl += 3;
  }
  h->launches += nl;
  prof_end(h, nl);
  CUDA_TRY(h, cudaGetLastError());
  m->cur ^= 1;
  m->stage = 1;
  return MPMB_OK;
}

static int m2_rasterize(MpmbEngine *h) {
  Mpm2d *m = h->m2;
  if (m->stage != 1) return fail(h, MPMB_ERR_STATE, "stages run in the order sort, rasterize, resample");
  const int n = (int)m->rows;
  const View2 V = m2_view(h);
  const int t0 = (m->P.nnode[0] + M2_TILE - 1) / M2_TILE, t1 = (m->P.nnode[1] + M2_TILE - 1) / M2_TILE;
  prof_begin(h, 1);
  k2_p2g_particles<<<m2_blocks(n, 256), 256, 0, h->stream>>>(V, m->P, n);
  k2_grid<<<(unsigned)(t0 * t1), 256, 0, h->stream>>>(V, m->P, t1);
  h->launches += 2;
  prof_end(h, 2);
  CUDA_TRY(h, cudaGetLastError());
  m->stage = 2;
  return MPMB_OK;
}

static int m2_resample(MpmbEngine *h) {
  Mpm2d *m = h->m2;
  if (m->stage != 2) return fail(h, MPMB_ERR_STATE, "stages run in the order sort, rasterize, resample");
  const int n = (int)m->rows;
  prof_begin(h, 2);
  if (n > 0) k2_g2p<<<m2_blocks(n, 256), 256, 0, h->stream>>>(m2_view(h), m->P, n);
  h->launches += n > 0;
  prof_end(h, n > 0);
  CUDA_TRY(h, cudaGetLastError());
  m->stage = 0;
  return MPMB_OK;
}

static int m2_substep_once(MpmbEngine *h) {
  int rc;
  if ((rc = m2_order(h)) != MPMB_OK) return rc;
  if ((rc = m2_rasterize(h)) != MPMB_OK) return rc;
  return m2_resample(h);
}

// Captures one substep at the current buffer parity (graph[cur]) and leaves the host state as before; any failure turns
// graphs off for this handle, and the substeps then run from the host with the same kernels.
static void m2_capture(MpmbEngine *h) {
  Mpm2d *m = h->m2;
  if (!h->cap_stream && cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking) != cudaSuccess) { h->use_graph = false; cudaGetLastError(); return; }
  const int cur0 = m->cur;
  const int64_t l0 = h->launches;
  cudaStream_t user = h->stream;
  h->stream = h->cap_stream;
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal);
  int rc = MPMB_OK;
  if (e == cudaSuccess) {
    rc = m2_substep_once(h);
    e = cudaStreamEndCapture(h->cap_stream, &g);
  }
  h->stream = user;
  if (e == cudaSuccess && rc == MPMB_OK && g) e = cudaGraphInstantiate(&m->graph[cur0], g, 0);
  if (g) cudaGraphDestroy(g);
  if (e != cudaSuccess || rc != MPMB_OK || !m->graph[cur0]) {
    cudaGetLastError();
    m->graph[cur0] = nullptr;
    h->use_graph = false;
    h->sticky_cuda = false;
  }
  m->graph_launches = (int)(h->launches - l0);
  m->cur = cur0;
  m->stage = 0;
  h->launches = l0;
}

static int m2_substep(MpmbEngine *h, int nsub) {
  Mpm2d *m = h->m2;
  if (m->stage != 0) return fail(h, MPMB_ERR_STATE, "mpmb_substep runs between substeps (the stage calls left one open)");
  for (int s = 0; s < nsub; s++) {
    if (h->use_graph && !h->profiling && m->rows > 0) {
      if (!m->graph[m->cur]) m2_capture(h);
      if (m->graph[m->cur]) {
        CUDA_TRY(h, cudaGraphLaunch(m->graph[m->cur], h->stream));
        h->launches += m->graph_launches;
        m->cur ^= 1;
        continue;
      }
    }
    int rc = m2_substep_once(h);
    if (rc != MPMB_OK) return rc;
  }
  return MPMB_OK;
}

static int m2_synchronize(MpmbEngine *h) {
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  Counters2 c;
  CUDA_TRY(h, cudaMemcpy(&c, h->m2->cnt.get(), sizeof(c), cudaMemcpyDeviceToHost));
  if (c.error & DEVERR_BAD_INPUT) return fail(h, MPMB_ERR_INVALID, "uploaded particles with group outside [0,%d) or mass <= 0", MPMB_MAX_GROUPS);
  return MPMB_OK;
}

static int m2_num_particles(MpmbEngine *h, int64_t *n) {
  Mpm2d *m = h->m2;
  int rc = m2_synchronize(h);
  if (rc != MPMB_OK) return rc;
  CUDA_TRY(h, cudaMemsetAsync(&m->cnt.get()->n_live, 0, sizeof(int), h->stream));
  if (m->rows > 0) {
    k2_count_live<<<m2_blocks(m->rows, 256), 256, 0, h->stream>>>(m->keys.get(), (int)m->rows, (uint32_t)m->P.ncells, m->cnt.get());
    h->launches++;
  }
  int live = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&live, &m->cnt.get()->n_live, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  *n = live;
  return MPMB_OK;
}

// The live rows of the current storage on the host, in storage order: keys, x, v, F, b, aux (staging for the downloads;
// a download is not on the substep's path).
struct M2Rows {
  std::vector<uint32_t> keys;
  std::vector<float2> x, v;
  std::vector<float4> F, b, aux;
  std::vector<int64_t> live;  // row indices
};
static int m2_read_rows(MpmbEngine *h, M2Rows *r) {
  Mpm2d *m = h->m2;
  int rc = m2_synchronize(h);
  if (rc != MPMB_OK) return rc;
  const size_t n = (size_t)m->rows;
  r->keys.resize(n); r->x.resize(n); r->v.resize(n); r->F.resize(n); r->b.resize(n); r->aux.resize(n);
  r->live.clear();
  if (n == 0) return MPMB_OK;
  const int c = m->cur;
  CUDA_TRY(h, cudaMemcpy(r->keys.data(), m->keys.get(), sizeof(uint32_t) * n, cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(r->x.data(), m->x[c].get(), sizeof(float2) * n, cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(r->v.data(), m->v[c].get(), sizeof(float2) * n, cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(r->F.data(), m->F[c].get(), sizeof(float4) * n, cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(r->b.data(), m->b[c].get(), sizeof(float4) * n, cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(r->aux.data(), m->aux[c].get(), sizeof(float4) * n, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < n; i++)
    if (r->keys[i] < (uint32_t)m->P.ncells) r->live.push_back((int64_t)i);
  return MPMB_OK;
}

static uint32_t m2_bits(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}

static int m2_download(MpmbEngine *h, int64_t cap, int64_t *n_out, uint32_t *id, float *x, float *v, float *F, float *b, float *mass, float *vol,
                       float *scalar, int32_t *group) {
  if (!n_out) return fail(h, MPMB_ERR_INVALID, "null n_out");
  M2Rows r;
  int rc = m2_read_rows(h, &r);
  if (rc != MPMB_OK) return rc;
  const int64_t n = (int64_t)r.live.size();
  if (n > cap) return fail(h, MPMB_ERR_CAPACITY, "%lld live particles do not fit in %lld rows", (long long)n, (long long)cap);
  for (int64_t k = 0; k < n; k++) {
    const int64_t i = r.live[k];
    const uint32_t tag = m2_bits(r.aux[i].w);
    if (id) id[k] = tag & TAG_ID_MASK;
    if (x) { x[2 * k] = r.x[i].x; x[2 * k + 1] = r.x[i].y; }
    if (v) { v[2 * k] = r.v[i].x; v[2 * k + 1] = r.v[i].y; }
    if (F) { F[4 * k] = r.F[i].x; F[4 * k + 1] = r.F[i].y; F[4 * k + 2] = r.F[i].z; F[4 * k + 3] = r.F[i].w; }
    if (b) { b[4 * k] = r.b[i].x; b[4 * k + 1] = r.b[i].y; b[4 * k + 2] = r.b[i].z; b[4 * k + 3] = r.b[i].w; }
    if (mass) mass[k] = r.aux[i].x;
    if (vol) vol[k] = r.aux[i].y;
    if (scalar) scalar[k] = r.aux[i].z;
    if (group) group[k] = (int32_t)(tag >> TAG_ID_BITS);
  }
  *n_out = n;
  return MPMB_OK;
}

// The 48-byte point records of write_partio (src/visualize.cpp:16-100) for MPM<2>: the dim loops fill x, y and v_x, v_y
// and leave the third components 0.  In id order.
static int m2_bgeo_points(MpmbEngine *h, int64_t id_range, void *records, int64_t cap_records, int64_t *n_out) {
  Mpm2d *m = h->m2;
  M2Rows r;
  int rc = m2_read_rows(h, &r);
  if (rc != MPMB_OK) return rc;
  std::vector<std::pair<uint32_t, int64_t>> order;
  order.reserve(r.live.size());
  for (int64_t i : r.live) {
    const uint32_t gid = m2_bits(r.aux[i].w) & TAG_ID_MASK;
    if ((int64_t)(gid - m->id_base) >= id_range || gid < m->id_base) return fail(h, MPMB_ERR_INVALID, "particle id %u outside [id_base, id_base + id_range)", gid);
    order.push_back({gid, i});
  }
  std::sort(order.begin(), order.end());
  if ((int64_t)order.size() > cap_records) return fail(h, MPMB_ERR_CAPACITY, "%lld live particles do not fit in the %lld records provided", (long long)order.size(), (long long)cap_records);
  auto be = [](uint32_t v) { return (v >> 24) | ((v >> 8) & 0xff00u) | ((v << 8) & 0xff0000u) | (v << 24); };
  uint32_t *out = (uint32_t *)records;
  for (size_t k = 0; k < order.size(); k++) {
    const int64_t i = order[k].second;
    uint32_t *w = out + 12 * k;
    w[0] = be(m2_bits(r.x[i].x)); w[1] = be(m2_bits(r.x[i].y)); w[2] = 0u; w[3] = be(m2_bits(1.0f));
    w[4] = 0u; w[5] = be(order[k].first); w[6] = be(1u); w[7] = be(1u);
    w[8] = be(1u); w[9] = be(m2_bits(r.v[i].x)); w[10] = be(m2_bits(r.v[i].y)); w[11] = 0u;
  }
  *n_out = (int64_t)order.size();
  return MPMB_OK;
}

static int m2_download_grid(MpmbEngine *h, int which, float *dense4) {
  Mpm2d *m = h->m2;
  if (m->stage != 2) return fail(h, MPMB_ERR_STATE, "the grid exists between rasterize and resample");
  if (!dense4 || which < 0 || which > 1) return fail(h, MPMB_ERR_INVALID, "bad argument");
  const size_t n = (size_t)m->P.nnode[0] * m->P.nnode[1];
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaMemcpy(dense4, m->graw.get(), sizeof(float4) * n, cudaMemcpyDeviceToHost));
  if (which == 1) {
    std::vector<float2> gv(n);
    CUDA_TRY(h, cudaMemcpy(gv.data(), m->gv.get(), sizeof(float2) * n, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; i++) { dense4[4 * i] = gv[i].x; dense4[4 * i + 1] = gv[i].y; }
  }
  return MPMB_OK;
}

static int m2_set_material(MpmbEngine *h, int group, int kind, const float *params, int n_params) {
  Mpm2d *m = h->m2;
  m->P.mats[group].kind = kind;
  for (int k = 0; k < 8; k++) m->P.mats[group].p[k] = k < n_params ? params[k] : 0.f;
  m2_graph_reset(m);
  return MPMB_OK;
}

static int m2_set_delta_t(MpmbEngine *h, float dt) {
  Mpm2d *m = h->m2;
  if (m->stage != 0) return fail(h, MPMB_ERR_STATE, "delta_t changes between substeps, not inside one");
  h->cfg.dt = dt;
  m->P.dt = dt;
  for (int d = 0; d < 2; d++) m->P.gdt[d] = h->cfg.gravity[d] * dt;
  m2_graph_reset(m);
  return MPMB_OK;
}

// shapes with zero z parts only (a 2-D solid): planes n_z = 0, circles c_z = 0, rectangles lo_z = hi_z = 0
static int m2_set_shapes(MpmbEngine *h, int n_shapes, const MpmbShape *shapes, float friction) {
  Mpm2d *m = h->m2;
  for (int k = 0; k < n_shapes; k++) {
    const MpmbShape &s = shapes[k];
    const bool flat = s.kind == MPMB_SHAPE_CUBOID ? (s.p[2] == 0.f && s.p[5] == 0.f) : s.p[2] == 0.f;
    if (!flat) return fail(h, MPMB_ERR_INVALID, "shape %d of a 2-D level set has a z part (must be 0)", k);
  }
  std::vector<MpmbShape> flat(shapes, shapes + n_shapes);
  for (auto &s : flat)  // a rectangle is the cuboid unbounded along z
    if (s.kind == MPMB_SHAPE_CUBOID) { s.p[2] = -1e30f; s.p[5] = 1e30f; }
  const size_t n = (size_t)m->P.nnode[0] * m->P.nnode[1];
  CUDA_TRY(h, m->sdf4.reserve(n));
  DevBuf<MpmbShape> d;
  CUDA_TRY(h, d.alloc(n_shapes));
  CUDA_TRY(h, cudaMemcpyAsync(d.get(), flat.data(), sizeof(MpmbShape) * n_shapes, cudaMemcpyHostToDevice, h->stream));
  k2_shapes_to_sdf<<<h->num_sms * 8, 256, 0, h->stream>>>(m->P, n_shapes, d.get(), m->sdf4.get());
  h->launches++;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  m->P.has_sdf = 1;
  m->P.friction = friction;
  m2_graph_reset(m);
  return MPMB_OK;
}

static int m2_set_planes(MpmbEngine *h, int n_planes, const float *planes4, float friction) {
  std::vector<MpmbShape> s(n_planes);
  for (int k = 0; k < n_planes; k++) {
    s[k] = MpmbShape{};
    s[k].kind = MPMB_SHAPE_PLANE;
    for (int c = 0; c < 4; c++) s[k].p[c] = planes4[4 * k + c];
  }
  return m2_set_shapes(h, n_planes, s.data(), friction);
}

static int m2_set_sdf(MpmbEngine *h, const float *sdf4, float friction) {
  Mpm2d *m = h->m2;
  m2_graph_reset(m);
  if (!sdf4) {
    m->P.has_sdf = 0;
    return MPMB_OK;
  }
  const size_t n = (size_t)m->P.nnode[0] * m->P.nnode[1];
  CUDA_TRY(h, m->sdf4.reserve(n));
  CUDA_TRY(h, cudaMemcpyAsync(m->sdf4.get(), sdf4, sizeof(float4) * n, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  m->P.has_sdf = 1;
  m->P.friction = friction;
  return MPMB_OK;
}
// ===================================================================================== end of the 2-D engine

// mpmb_create of a 2-D handle (cfg->dim == 2, validated): the 2-D engine and the handle's shared parts (stream, profiling,
// default materials, CUDA-graph switch)
static int create_2d(MpmbEngine *h, const MpmbConfig *cfg, MpmbHandle *out) {
  for (int g = 0; g < MPMB_MAX_GROUPS; g++) {
    h->P.mats[g].kind = MAT_JELLY;  // JellyParticle defaults E=1e5, nu=0.3 (src/particles.cpp:383-389)
    for (int k = 0; k < 8; k++) h->P.mats[g].p[k] = 0.f;
    h->P.mats[g].p[0] = 1e5f / (2.f * 1.3f);
    h->P.mats[g].p[1] = 1e5f * 0.3f / (1.3f * 0.4f);
  }
  h->use_graph = cfg->no_graph == 0;
  if (cudaSetDevice(cfg->device) != cudaSuccess) { delete h; return fail(nullptr, MPMB_ERR_CUDA, "cudaSetDevice failed"); }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, cfg->device);
  h->num_sms = prop.multiProcessorCount;
  int rc = m2_create(h, cfg);
  if (rc == MPMB_OK && cfg->capacity > 0) {
    rc = m2_alloc_rows(h, cfg->capacity);
    if (rc != MPMB_OK) g_create_error = h->err;
  }
  if (rc != MPMB_OK) {
    mpmb_destroy(h);
    return rc;
  }
  *out = h;
  return MPMB_OK;
}

extern "C" {

static int read_n_store(MpmbEngine *h, int *n_store);

int mpmb_version(void) { return MPMB_VERSION; }

const char *mpmb_last_error(MpmbHandle h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int mpmb_create(const MpmbConfig *cfg, MpmbHandle *out) {
  if (!cfg || !out) return fail(nullptr, MPMB_ERR_INVALID, "null argument");
  *out = nullptr;
  if (cfg->dim != 0 && cfg->dim != 2 && cfg->dim != 3) return fail(nullptr, MPMB_ERR_INVALID, "dim=%d: 0 or 3 (MPM<3>) or 2 (MPM<2>)", cfg->dim);
  const bool two_d = cfg->dim == 2;
  for (int d = 0; d < (two_d ? 2 : 3); d++)
    if (cfg->res[d] < 16 || cfg->res[d] > 4096) return fail(nullptr, MPMB_ERR_INVALID, "res[%d]=%d out of range [16,4096]", d, cfg->res[d]);
  if (two_d && (cfg->res[2] != 0 || cfg->gravity[2] != 0.f || cfg->world > 1))
    return fail(nullptr, MPMB_ERR_INVALID, "dim=2 needs res[2] == 0, gravity[2] == 0 and world == 1");
  if (!two_d && (cfg->apic_damping != 0.f || cfg->rpic_damping != 0.f))
    return fail(nullptr, MPMB_ERR_INVALID, "apic_damping / rpic_damping are supported with dim=2 only");
  if (two_d && (!std::isfinite(cfg->apic_damping) || !std::isfinite(cfg->rpic_damping)))
    return fail(nullptr, MPMB_ERR_INVALID, "apic_damping / rpic_damping must be finite");
  if (!(cfg->dx > 0.f) || !(cfg->dt > 0.f)) return fail(nullptr, MPMB_ERR_INVALID, "dx and dt must be positive");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return fail(nullptr, MPMB_ERR_CUDA, "no CUDA device: %s", cudaGetErrorString(e));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, MPMB_ERR_INVALID, "device %d not in [0,%d)", cfg->device, ndev);
  MpmbEngine *h = new MpmbEngine();
  h->cfg = *cfg;
  if (h->cfg.world <= 0) h->cfg.world = 1;
  if (two_d) return create_2d(h, cfg, out);
  Params &P = h->P;
  for (int d = 0; d < 3; d++) {
    P.res[d] = cfg->res[d];
    P.nnode[d] = cfg->res[d] + 1;
    P.nt[d] = (P.nnode[d] + 3) / 4 + 1;
    P.gdt[d] = cfg->gravity[d] * cfg->dt;
  }
  h->nt2_global = P.nt[2];
  if (h->cfg.world > 1 && (cfg->tile_z0 < 0 || cfg->tile_z1 > P.nt[2] || cfg->tile_z0 >= cfg->tile_z1)) {
    const int n2 = P.nt[2];
    delete h;
    return fail(nullptr, MPMB_ERR_INVALID, "bad slab [%d,%d) for %d tile layers", cfg->tile_z0, cfg->tile_z1, n2);
  }
  Slicing sl;
  if (!slab_slicing(P, h->nt2_global, h->cfg.world, cfg->tile_z0, cfg->tile_z1, &sl)) { delete h; return fail(nullptr, MPMB_ERR_INVALID, "tile grid too large for 32-bit keys"); }
  set_slicing(h, sl);
  P.dx = cfg->dx;
  P.inv_dx = 1.0f / cfg->dx;
  P.dt = cfg->dt;
  P.particle_gravity = cfg->particle_gravity;
  P.clean_boundary = cfg->clean_boundary;
  P.friction = 0.f;
  P.has_sdf = 0;
  P.world = h->cfg.world;
  for (int g = 0; g < MPMB_MAX_GROUPS; g++) {
    P.mats[g].kind = MAT_JELLY;  // JellyParticle defaults E=1e5, nu=0.3 (src/particles.cpp:383-389)
    for (int k = 0; k < 8; k++) P.mats[g].p[k] = 0.f;
    P.mats[g].p[0] = 1e5f / (2.f * 1.3f);
    P.mats[g].p[1] = 1e5f * 0.3f / (1.3f * 0.4f);
  }
  h->use_graph = cfg->no_graph == 0;
  if (const char *g = getenv("MPMB_GRAPH")) h->use_graph = g[0] != '0';   // MPMB_GRAPH=0: launch every kernel from the host (A/B, debugging)
  if (cudaSetDevice(cfg->device) != cudaSuccess) { delete h; return fail(nullptr, MPMB_ERR_CUDA, "cudaSetDevice failed"); }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, cfg->device);
  h->num_sms = prop.multiProcessorCount;
  // MPMB_NUM_SMS=k (tests): size every persistent and grid-stride launch for min(k, SMs) SMs, so that a small scene
  // still makes each CTA walk many tiles
  if (const char *s = getenv("MPMB_NUM_SMS")) { const int k = atoi(s); if (k > 0) h->num_sms = std::min(k, h->num_sms); }
  {
    int occ = 0;
    cudaFuncSetAttribute(k_p2g, cudaFuncAttributeMaxDynamicSharedMemorySize, P2G_DYN_BYTES);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_p2g, P2G_T, P2G_DYN_BYTES) == cudaSuccess && occ > 0) h->grid_p2g = h->num_sms * occ;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_g2p<128, true, true>, 128, 0) == cudaSuccess && occ > 0) h->grid_g2p = h->num_sms * occ;
  }
  auto bail = [&](const char *what) {
    std::string msg = std::string(what) + ": " + cudaGetErrorString(cudaGetLastError());
    mpmb_destroy(h);
    return fail(nullptr, MPMB_ERR_CUDA, "%s", msg.c_str());
  };
  // tiles: every tile of the (slab of the) domain can be active
  if (alloc_tile_arrays(h, sl.ntot) != MPMB_OK) {
    g_create_error = h->err;
    mpmb_destroy(h);
    return MPMB_ERR_CUDA;
  }
  if (h->cnt.alloc(1) != cudaSuccess) return bail("cudaMalloc counters");
  cudaMemset(h->cnt.get(), 0, sizeof(Counters));
  h->mig_cap = h->cfg.world > 1 ? (cfg->migrate_capacity > 0 ? cfg->migrate_capacity : 65536) : 0;
  if (h->cfg.world > 1) {
    const int64_t bytes[2] = {mpmb_halo_bytes(h), mpmb_migrate_bytes(h)};
    for (int k = 0; k < 2; k++)
      for (int f = 0; f < 2; f++) {
        if (h->rx[k][f].alloc(bytes[k]) != cudaSuccess) return bail("cudaMalloc exchange buffer");
        cudaMemset(h->rx[k][f].get(), 0, 16);
      }
    if (h->xcount.alloc(32) != cudaSuccess) return bail("cudaMalloc exchange counters");
    cudaMemset(h->xcount.get(), 0, sizeof(int) * 32);  // [0],[4] halo counts, [8],[12] migration counts, [16],[20] finished-CTA counters
    const size_t mail = (size_t)2 * h->cfg.world * RMAIL_SLOT;
    if (h->rmail.alloc(mail) != cudaSuccess || h->rmail_dev.alloc(h->cfg.world) != cudaSuccess) return bail("cudaMalloc rigid mailbox");
    cudaMemset(h->rmail.get(), 0, mail);
    h->rmail_tx.assign(h->cfg.world, nullptr);
    h->rmail_ipc.assign(h->cfg.world, false);
    h->rmail_tx[h->cfg.rank] = h->rmail.get();
  }
  if (cfg->capacity > 0) {
    int rc = alloc_particles(h, cfg->capacity);
    if (rc != MPMB_OK) { g_create_error = h->err; mpmb_destroy(h); return rc; }
  }
  *out = h;
  return MPMB_OK;
}

int mpmb_destroy(MpmbHandle h) {
  if (!h) return MPMB_OK;
  cudaSetDevice(h->cfg.device);
  cudaDeviceSynchronize();
  m2_destroy(h);
  // memory is freed by the buffers' destructors (with this device current); here go the handles that are not memory
  for (int k = 0; k < 2; k++)
    for (int f = 0; f < 2; f++)
      if (h->tx_ipc[k][f] && h->tx[k][f]) cudaIpcCloseMemHandle(h->tx[k][f]);
  for (size_t r = 0; r < h->rmail_tx.size(); r++)
    if (h->rmail_ipc[r] && h->rmail_tx[r]) cudaIpcCloseMemHandle(h->rmail_tx[r]);
  for (auto &e : h->events) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
  graph_reset(h);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  delete h;
  return MPMB_OK;
}

int mpmb_set_stream(MpmbHandle h, void *s) {
  CHECK_HANDLE(h);
  h->stream = (cudaStream_t)s;
  return MPMB_OK;
}

int mpmb_synchronize(MpmbHandle h) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_synchronize(h);
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  Counters c;
  CUDA_TRY(h, cudaMemcpy(&c, h->cnt.get(), sizeof(c), cudaMemcpyDeviceToHost));
  if (c.error & DEVERR_TILE_CAPACITY) return fail(h, MPMB_ERR_CAPACITY, "active tile capacity exceeded");
  if (c.error & DEVERR_MIGRATE_CAPACITY) return fail(h, MPMB_ERR_CAPACITY, "migration buffer capacity exceeded");
  if (c.error & DEVERR_PARTICLE_CAPACITY) return fail(h, MPMB_ERR_CAPACITY, "particle capacity exceeded");
  if (c.error & DEVERR_PEER_TIMEOUT) return fail(h, MPMB_ERR_STATE, "peer exchange timed out (neighbour rank not stepping)");
  if (c.error & DEVERR_BAD_INPUT) return fail(h, MPMB_ERR_INVALID, "uploaded particles with group outside [0,%d) or mass <= 0", MPMB_MAX_GROUPS);
  return MPMB_OK;
}

int mpmb_set_material(MpmbHandle h, int32_t group, int32_t kind, const float *params, int32_t n_params) {
  CHECK_HANDLE(h);
  if (group < 0 || group >= MPMB_MAX_GROUPS) return fail(h, MPMB_ERR_INVALID, "group %d out of range", group);
  if (kind < MPMB_MAT_LINEAR || kind > MPMB_MAT_VISCO) return fail(h, MPMB_ERR_INVALID, "unknown material kind %d", kind);
  if (n_params < 0 || n_params > MPMB_MAT_PARAMS || (n_params > 0 && !params)) return fail(h, MPMB_ERR_INVALID, "bad parameter vector");
  if (h->m2) return m2_set_material(h, group, kind, params, n_params);
  h->P.mats[group].kind = kind;
  for (int k = 0; k < 8; k++) h->P.mats[group].p[k] = k < n_params ? params[k] : 0.f;
  graph_reset(h);
  // particles of this group already resident: their cached affine matrix belongs to the old material
  if (h->cap > 0 && h->stage == 0) {
    int ns = 0;
    int rc = read_n_store(h, &ns);
    if (rc != MPMB_OK) return rc;
    if (ns > 0) {
      View V = make_view(h);
      k_refresh_affine<<<(ns + 127) / 128, 128, 0, h->stream>>>(V, h->P, h->keys[h->cur].get(), ns, h->special_min, group);
      h->launches++;
      CUDA_TRY(h, cudaGetLastError());
    }
  }
  return MPMB_OK;
}

// the step of the following substeps (dt and the gravity kick it scales); returns whether it changed
static bool apply_delta_t(MpmbEngine *h, float dt) {
  if (dt == h->P.dt) return false;
  h->cfg.dt = dt;
  h->P.dt = dt;
  for (int d = 0; d < 3; d++) h->P.gdt[d] = h->cfg.gravity[d] * dt;
  graph_reset(h);
  return true;
}

int mpmb_set_delta_t(MpmbHandle h, float dt) {
  CHECK_HANDLE(h);
  if (!(dt > 0.f) || !std::isfinite(dt)) return fail(h, MPMB_ERR_INVALID, "delta_t must be positive and finite");
  if (h->m2) return m2_set_delta_t(h, dt);
  if (h->stage != 0) return fail(h, MPMB_ERR_STATE, "delta_t changes between substeps, not inside one");
  if (!apply_delta_t(h, dt)) return MPMB_OK;
  // resident particles: the affine matrix cached for the next rasterize carries the old dt (stress * (-4 dt / dx))
  if (h->cap > 0) {
    int ns = 0;
    int rc = read_n_store(h, &ns);
    if (rc != MPMB_OK) return rc;
    if (ns > 0) {
      View V = make_view(h);
      for (int g = 0; g < MPMB_MAX_GROUPS; g++) {
        k_refresh_affine<<<(ns + 127) / 128, 128, 0, h->stream>>>(V, h->P, h->keys[h->cur].get(), ns, h->special_min, g);
        h->launches++;
      }
      CUDA_TRY(h, cudaGetLastError());
    }
  }
  return MPMB_OK;
}

int mpmb_set_id_base(MpmbHandle h, int64_t base) {
  CHECK_HANDLE(h);
  if (base < 0 || base >= (1ll << TAG_ID_BITS)) return fail(h, MPMB_ERR_INVALID, "id base %lld outside [0, 2^%d)", (long long)base, TAG_ID_BITS);
  if (h->m2) { h->m2->id_base = (uint32_t)base; return MPMB_OK; }
  if ((uint32_t)base != h->id_base) graph_reset(h);   // the captured rigid kernels take id_base by value
  h->id_base = (uint32_t)base;
  return MPMB_OK;
}

int mpmb_set_sdf(MpmbHandle h, const float *sdf4, float friction) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_set_sdf(h, sdf4, friction);
  size_t n = (size_t)h->P.nnode[0] * h->P.nnode[1] * h->P.nnode[2];
  if (!sdf4) {
    h->P.has_sdf = 0;
    graph_reset(h);
    return MPMB_OK;
  }
  CUDA_TRY(h, h->sdf4.reserve(n));
  CUDA_TRY(h, cudaMemcpyAsync(h->sdf4.get(), sdf4, sizeof(float4) * n, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->P.has_sdf = 1;
  h->P.friction = friction;
  graph_reset(h);
  return MPMB_OK;
}

int mpmb_set_planes(MpmbHandle h, int32_t n_planes, const float *planes4, float friction) {
  CHECK_HANDLE(h);
  if (n_planes <= 0 || n_planes > 64 || !planes4) return fail(h, MPMB_ERR_INVALID, "need 1..64 planes");
  if (h->m2) return m2_set_planes(h, n_planes, planes4, friction);
  size_t n = (size_t)h->P.nnode[0] * h->P.nnode[1] * h->P.nnode[2];
  CUDA_TRY(h, h->sdf4.reserve(n));
  DevBuf<float4> d_planes;
  CUDA_TRY(h, d_planes.alloc(n_planes));
  CUDA_TRY(h, cudaMemcpyAsync(d_planes.get(), planes4, sizeof(float4) * n_planes, cudaMemcpyHostToDevice, h->stream));
  k_planes_to_sdf<<<h->num_sms * 8, 256, 0, h->stream>>>(h->P, n_planes, d_planes.get(), h->sdf4.get());
  h->launches++;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->P.has_sdf = 1;
  h->P.friction = friction;
  graph_reset(h);
  return MPMB_OK;
}

int mpmb_set_levelset_shapes(MpmbHandle h, int32_t n_shapes, const MpmbShape *shapes, float friction) {
  CHECK_HANDLE(h);
  if (n_shapes <= 0 || n_shapes > 64 || !shapes) return fail(h, MPMB_ERR_INVALID, "need 1..64 shapes");
  for (int k = 0; k < n_shapes; k++)
    if (shapes[k].kind < MPMB_SHAPE_PLANE || shapes[k].kind > MPMB_SHAPE_CUBOID) return fail(h, MPMB_ERR_INVALID, "unknown shape kind %d", shapes[k].kind);
  if (h->m2) return m2_set_shapes(h, n_shapes, shapes, friction);
  size_t n = (size_t)h->P.nnode[0] * h->P.nnode[1] * h->P.nnode[2];
  CUDA_TRY(h, h->sdf4.reserve(n));
  DevBuf<MpmbShape> d_shapes;
  CUDA_TRY(h, d_shapes.alloc(n_shapes));
  CUDA_TRY(h, cudaMemcpyAsync(d_shapes.get(), shapes, sizeof(MpmbShape) * n_shapes, cudaMemcpyHostToDevice, h->stream));
  k_shapes_to_sdf<<<h->num_sms * 8, 256, 0, h->stream>>>(h->P, n_shapes, d_shapes.get(), h->sdf4.get());
  h->launches++;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->P.has_sdf = 1;
  h->P.friction = friction;
  graph_reset(h);
  return MPMB_OK;
}

static int ensure_capacity(MpmbEngine *h, int64_t n) {
  int64_t want = n;
  if (h->cfg.world > 1) want = n + n / 4 + 16 * h->mig_cap;
  if (h->cfg.capacity > 0) {
    if (n > h->cap) return fail(h, MPMB_ERR_CAPACITY, "%lld particles exceed the configured capacity %lld", (long long)n, (long long)h->cap);
    return MPMB_OK;
  }
  if (want > h->cap) return alloc_particles(h, want);
  return MPMB_OK;
}

// Room for `need` rows that keeps rows [0, n_keep) of the current storage (an append onto a resident set).  With a
// configured capacity that is too small nothing changes; otherwise the buffers grow by at least half, so that a source
// that appends every frame reallocates rarely.  On z-slab ranks growth keeps the migration headroom of ensure_capacity
// (immigrants are appended after the last row).  The exchange buffers (rx / tx) are not particle rows: they survive.
static int grow_keeping_rows(MpmbEngine *h, int64_t need, int n_keep) {
  if (h->cfg.capacity > 0) {
    if (need <= h->cap) return MPMB_OK;
    return fail(h, MPMB_ERR_CAPACITY, "%lld particle rows exceed the configured capacity %lld", (long long)need, (long long)h->cap);
  }
  const int64_t room = h->cfg.world > 1 ? need + need / 4 + 16 * h->mig_cap : need;
  if (room <= h->cap) return MPMB_OK;
  const int64_t want = std::max<int64_t>(room, std::min<int64_t>(h->cap + h->cap / 2, (1ll << 30) - 1));
  DevBuf<float4> old_q[N_Q];   // the current rows survive the reallocation here
  for (int k = 0; k < N_Q; k++) old_q[k] = std::move(h->q[h->cur][k]);
  DevBuf<uint32_t> old_keys = std::move(h->keys[h->cur]);
  int rc = alloc_particles(h, want);   // frees everything else (scratch, the other buffer) and resets the graphs
  if (rc == MPMB_OK && n_keep > 0) {
    for (int k = 0; k < N_Q; k++)
      CUDA_TRY(h, cudaMemcpyAsync(h->q[h->cur][k].get(), old_q[k].get(), sizeof(float4) * n_keep, cudaMemcpyDeviceToDevice, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->keys[h->cur].get(), old_keys.get(), sizeof(uint32_t) * n_keep, cudaMemcpyDeviceToDevice, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  return rc;
}

// Orders rows [0, n_rows) of the current storage from scratch: no runs yet, every live row is an "arrival" of its tile.
// One radix sort groups the rows by tile (dead keys sort past every tile, so rows killed since the last ordering drop
// out here); the ordinary ordering scan then lays out the first runs.  The next substep runs outside the graph.
static int reorder_from_scratch(MpmbEngine *h, int64_t n_rows) {
  View V = make_view(h);
  const size_t dense = sizeof(int) * (size_t)h->ntot;
  CUDA_TRY(h, cudaMemsetAsync(h->run_begin[h->ord].get(), 0, dense, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->run_len[h->ord].get(), 0, dense, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->stay[h->ord].get(), 0, dense, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->arr_cnt.get(), 0, dense, h->stream));
  Counters c{};
  c.n_store = (int)n_rows;
  CUDA_TRY(h, cudaMemcpyAsync(h->cnt.get(), &c, sizeof(int) * 3, cudaMemcpyHostToDevice, h->stream));          // n_store, n_tiles, n_ghost
  CUDA_TRY(h, cudaMemsetAsync(&h->cnt.get()->n_movers, 0, sizeof(int) * 3, h->stream));                          // n_movers, n_movers_next, n_alive
  if (n_rows > 0) {
    size_t cub_bytes = h->cub_temp.size();
    cub::DeviceRadixSort::SortPairs(h->cub_temp.get(), cub_bytes, h->keys[h->cur].get(), h->keys_sorted.get(), h->iota.get(), h->arrivals_sorted.get(), (int)n_rows, 0, h->key_bits, h->stream);
    k_count_sorted<<<(unsigned)((n_rows + 255) / 256), 256, 0, h->stream>>>(V, h->keys_sorted.get(), (int)n_rows, h->ntot);
    h->launches++;
  }
  h->fresh = true;
  h->stage = 0;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

static int rigid_reserve_ids(MpmbEngine *h, int64_t n_ids);
// A new resident set of n rows (upload, seeding): its id span, fresh rigid colours, then the ordering.
static int finish_upload(MpmbEngine *h, int64_t n) {
  h->aos_kinds_valid = false;   // mpmb_upload_aos takes its snapshot after this
  h->id_span = std::max<int64_t>(h->id_span_pending, n);
  h->id_span_pending = 0;
  h->id_end = (int64_t)h->id_base + h->id_span;
  if (h->rigid_on) {  // new particles start with MPMParticle::states = 0 (mpmb_set_particle_states overrides)
    int rc = rigid_reserve_ids(h, std::max<int64_t>(rigid_ids(h), h->cap));
    if (rc != MPMB_OK) return rc;
    CUDA_TRY(h, cudaMemsetAsync(h->p_states.get(), 0, sizeof(uint32_t) * h->p_states.size(), h->stream));
  }
  return reorder_from_scratch(h, n);
}

// Packs n field-wise particles held in DEVICE arrays into rows row0.. with ids id0.. of the current storage (F, b, scalar,
// group may be NULL).  The one packing path of uploads, appends and AsyncMPM advances.  With `prefix` only the particles
// k_owned_flags marked, compacted (k_pack_particles).
static int pack_rows(MpmbEngine *h, int64_t n, const float *x, const float *v, const float *F, const float *b, const float *mass,
                     const float *vol, const float *scalar, const int *group, int row0, uint32_t id0, const int *prefix = nullptr) {
  View V = make_view(h);
  k_pack_particles<<<(unsigned)((n + 127) / 128), 128, 0, h->stream>>>(V, h->P, (int)n, x, v, F, b, mass, vol, scalar, group, h->keys[h->cur].get(), row0, id0,
                                                                         prefix);
  h->launches++;
  cudaError_t e = cudaStreamSynchronize(h->stream);
  CUDA_TRY(h, e);
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

// n field-wise particles staged on the device (F, b, scalar, group NULL where the caller gave none)
struct StagedFields {
  float *x, *v, *F, *b, *mass, *vol, *scalar;
  int *group;
};

// Copies n field-wise host particles into the staging buffer (one allocation, grow-only); asynchronous.
static int stage_fields(MpmbEngine *h, int64_t n, const float *x, const float *v, const float *F, const float *b, const float *mass,
                        const float *vol, const float *scalar, const int32_t *group, StagedFields *s) {
  size_t fl = (size_t)n * (3 + 3 + (F ? 9 : 0) + (b ? 9 : 0) + 1 + 1 + (scalar ? 1 : 0)) + (group ? (size_t)n : 0);
  CUDA_TRY(h, h->stage_buf.reserve(fl * sizeof(float)));
  float *p = (float *)h->stage_buf.get();
  auto put = [&](const void *src, size_t count) -> float * {
    if (!src) return nullptr;
    float *dst = p;
    cudaMemcpyAsync(dst, src, count * sizeof(float), cudaMemcpyHostToDevice, h->stream);
    p += count;
    return dst;
  };
  s->x = put(x, 3 * n); s->v = put(v, 3 * n); s->F = put(F, 9 * n); s->b = put(b, 9 * n); s->mass = put(mass, n); s->vol = put(vol, n);
  s->scalar = put(scalar, n);
  s->group = (int *)put(group, n);
  return MPMB_OK;
}

// Stages n field-wise particles on the device and packs them into rows row0.. with ids id0.. of the current storage.
static int pack_fields(MpmbEngine *h, int64_t n, const float *x, const float *v, const float *F, const float *b, const float *mass,
                       const float *vol, const float *scalar, const int32_t *group, int row0, uint32_t id0) {
  StagedFields s;
  int rc = stage_fields(h, n, x, v, F, b, mass, vol, scalar, group, &s);
  if (rc != MPMB_OK) return rc;
  return pack_rows(h, n, s.x, s.v, s.F, s.b, s.mass, s.vol, s.scalar, s.group, row0, id0);
}

int mpmb_upload_particles(MpmbHandle h, int64_t n, const float *x, const float *v, const float *F, const float *b,
                          const float *mass, const float *vol, const float *scalar, const int32_t *group) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_upload(h, n, x, v, F, b, mass, vol, scalar, group);
  if (n < 0 || (n > 0 && (!x || !v || !mass || !vol))) return fail(h, MPMB_ERR_INVALID, "x, v, mass, vol are required");
  if ((int64_t)h->id_base + n > (1ll << TAG_ID_BITS)) return fail(h, MPMB_ERR_CAPACITY, "particle ids exceed 2^%d", TAG_ID_BITS);
  h->aos_host_pool = nullptr;
  int rc = ensure_capacity(h, n);
  if (rc != MPMB_OK) return rc;
  if (n > 0 && (rc = pack_fields(h, n, x, v, F, b, mass, vol, scalar, group, 0, h->id_base)) != MPMB_OK) return rc;
  return finish_upload(h, n);
}

// Edits of the resident set between substeps (single-GPU engines): the rows already there keep their state, ids and
// CPIC colours; the whole set is ordered again from scratch, as after an upload.
static int edit_allowed(MpmbEngine *h, const char *what) {
  if (h->cfg.world > 1) return fail(h, MPMB_ERR_STATE, "%s is implemented for single-GPU engines (world == 1)", what);
  if (h->stage != 0) return fail(h, MPMB_ERR_STATE, "%s runs between substeps, not inside one", what);
  return MPMB_OK;
}

int mpmb_append_particles(MpmbHandle h, int64_t n, const float *x, const float *v, const float *F, const float *b,
                          const float *mass, const float *vol, const float *scalar, const int32_t *group, int64_t *first_id) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (n < 0 || (n > 0 && (!x || !v || !mass || !vol))) return fail(h, MPMB_ERR_INVALID, "x, v, mass, vol are required");
  int rc = edit_allowed(h, "append");
  if (rc != MPMB_OK) return rc;
  const int64_t id0 = h->id_span;
  if ((int64_t)h->id_base + id0 + n > (1ll << TAG_ID_BITS)) return fail(h, MPMB_ERR_CAPACITY, "particle ids exceed 2^%d", TAG_ID_BITS);
  if (first_id) *first_id = (int64_t)h->id_base + id0;
  if (n == 0) return MPMB_OK;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  int ns = 0;
  if ((rc = read_n_store(h, &ns)) != MPMB_OK) return rc;
  if ((rc = grow_keeping_rows(h, (int64_t)ns + n, ns)) != MPMB_OK) return rc;
  h->aos_host_pool = nullptr;   // the AoS index vector does not cover the new ids: mpmb_download_aos needs a new upload
  if ((rc = pack_fields(h, n, x, v, F, b, mass, vol, scalar, group, ns, h->id_base + (uint32_t)id0)) != MPMB_OK) return rc;
  h->id_span = id0 + n;
  h->id_end = std::max<int64_t>(h->id_end, (int64_t)h->id_base + h->id_span);
  if (h->rigid_on && (rc = rigid_reserve_ids(h, std::max<int64_t>(rigid_ids(h), h->cap))) != MPMB_OK) return rc;   // keeps the colours
  return reorder_from_scratch(h, (int64_t)ns + n);
}

static int scan_reserve(MpmbEngine *h, size_t n);
static int scan_flags(MpmbEngine *h, size_t n, int *total, const int *word = nullptr, int *word_out = nullptr);

int mpmb_append_owned_particles(MpmbHandle h, int64_t n, const float *x, const float *v, const float *F, const float *b,
                                const float *mass, const float *vol, const float *scalar, const int32_t *group, int64_t first_id,
                                int64_t *n_kept) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!n_kept) return fail(h, MPMB_ERR_INVALID, "null argument");
  *n_kept = 0;
  if (n < 0 || (n > 0 && (!x || !v || !mass || !vol))) return fail(h, MPMB_ERR_INVALID, "x, v, mass, vol are required");
  if (h->stage != 0 || h->rigid_pending) return fail(h, MPMB_ERR_STATE, "append_owned runs between substeps, not inside one");
  const int64_t end = std::max<int64_t>(h->id_end, h->id_base);
  if (first_id < end) return fail(h, MPMB_ERR_INVALID, "first_id %lld lies below the id end %lld", (long long)first_id, (long long)end);
  if (first_id + n > (1ll << TAG_ID_BITS)) return fail(h, MPMB_ERR_CAPACITY, "particle ids exceed 2^%d", TAG_ID_BITS);
  int kept = 0, ns = 0, rc;
  if (n > 0) {
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if ((rc = read_n_store(h, &ns)) != MPMB_OK) return rc;
    StagedFields s;
    if ((rc = stage_fields(h, n, x, v, F, b, mass, vol, scalar, group, &s)) != MPMB_OK) return rc;
    if ((rc = scan_reserve(h, (size_t)n)) != MPMB_OK) return rc;
    k_owned_flags<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(h->P, (int)n, s.x, h->scan_a.get());
    h->launches++;
    if ((rc = scan_flags(h, (size_t)n, &kept)) != MPMB_OK) return rc;
    if (kept > 0) {
      if ((rc = grow_keeping_rows(h, (int64_t)ns + kept, ns)) != MPMB_OK) return rc;
      h->aos_host_pool = nullptr;   // as mpmb_append_particles: the AoS index vector does not cover the new ids
      if ((rc = pack_rows(h, n, s.x, s.v, s.F, s.b, s.mass, s.vol, s.scalar, s.group, ns, (uint32_t)first_id, h->scan_b.get())) != MPMB_OK) return rc;
    }
  }
  // the whole batch consumes its ids on every rank, kept or not
  h->id_end = std::max<int64_t>(h->id_end, first_id + n);
  h->id_span = std::max<int64_t>(h->id_span, h->id_end - (int64_t)h->id_base);
  *n_kept = kept;
  if (h->rigid_on) {   // keeps the colours; the new ids start with MPMParticle::states = 0, as after mpmb_append_particles
    if ((rc = rigid_reserve_ids(h, std::max<int64_t>(rigid_ids(h), h->cap))) != MPMB_OK) return rc;
    if (n > 0) CUDA_TRY(h, cudaMemsetAsync(h->p_states.get() + (first_id - rigid_id0(h)), 0, sizeof(uint32_t) * n, h->stream));
  }
  return kept > 0 ? reorder_from_scratch(h, (int64_t)ns + kept) : MPMB_OK;
}

int mpmb_id_end(MpmbHandle h, int64_t *id_end) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!id_end) return fail(h, MPMB_ERR_INVALID, "null argument");
  *id_end = std::max<int64_t>(h->id_end, h->id_base);
  return MPMB_OK;
}

// the device part of both level-set deletions: every live row of this engine is sampled against the whole node grid
// (the level set is not sliced on z-slab ranks), the rows inside get the dead key, the set is ordered again
static int delete_inside(MpmbEngine *h, int64_t *n_deleted) {
  int rc;
  h->aos_host_pool = nullptr;
  if (!h->P.has_sdf || h->cap == 0) return MPMB_OK;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  int ns = 0;
  if ((rc = read_n_store(h, &ns)) != MPMB_OK) return rc;
  if (ns == 0) return MPMB_OK;
  CUDA_TRY(h, cudaMemsetAsync(&h->cnt.get()->n_live, 0, sizeof(int), h->stream));
  View V = make_view(h);
  k_delete_inside<<<(unsigned)((ns + 255) / 256), 256, 0, h->stream>>>(V, h->P, ns, h->special_min, h->key_dead);
  h->launches++;
  int killed = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&killed, &h->cnt.get()->n_live, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  *n_deleted = killed;
  return killed > 0 ? reorder_from_scratch(h, ns) : MPMB_OK;
}

int mpmb_delete_inside_levelset(MpmbHandle h, int64_t *n_deleted) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!n_deleted) return fail(h, MPMB_ERR_INVALID, "null argument");
  *n_deleted = 0;
  int rc = edit_allowed(h, "delete_inside_levelset");
  if (rc != MPMB_OK) return rc;
  return delete_inside(h, n_deleted);
}

int mpmb_delete_owned_inside_levelset(MpmbHandle h, int64_t *n_deleted) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!n_deleted) return fail(h, MPMB_ERR_INVALID, "null argument");
  *n_deleted = 0;
  if (h->stage != 0 || h->rigid_pending) return fail(h, MPMB_ERR_STATE, "delete_owned_inside_levelset runs between substeps, not inside one");
  return delete_inside(h, n_deleted);
}

// flags / exclusive prefix scratch for n items (grow-only) and the CUB scan over them
static int scan_reserve(MpmbEngine *h, size_t n) {
  CUDA_TRY(h, h->scan_a.reserve(n + 1));
  CUDA_TRY(h, h->scan_b.reserve(n + 1));
  size_t need = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, need, h->scan_a.get(), h->scan_b.get(), (int)(n + 1), h->stream);
  CUDA_TRY(h, h->scan_tmp.reserve(need));
  return MPMB_OK;
}
// prefix = exclusive scan of flags over n (+1 so that prefix[n] is the total); returns the total.  With `word`, that device
// int comes back in the same read-back (it is copied behind the total: scan_reserve(n + 1) leaves the room).
static int scan_flags(MpmbEngine *h, size_t n, int *total, const int *word, int *word_out) {
  CUDA_TRY(h, cudaMemsetAsync(h->scan_a.get() + n, 0, sizeof(int), h->stream));
  size_t bytes = h->scan_tmp.size();
  cub::DeviceScan::ExclusiveSum(h->scan_tmp.get(), bytes, h->scan_a.get(), h->scan_b.get(), (int)(n + 1), h->stream);
  int out[2] = {0, 0};
  if (word) CUDA_TRY(h, cudaMemcpyAsync(h->scan_b.get() + n + 1, word, sizeof(int), cudaMemcpyDeviceToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(out, h->scan_b.get() + n, sizeof(int) * (word ? 2 : 1), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  *total = out[0];
  if (word) *word_out = out[1];
  return MPMB_OK;
}

// byte range [lo, hi) of a slot that the layout's fields occupy: only that window of every slot crosses the bus (a 2-D
// copy with the slot stride as pitch) — 204 of the reference's 320 bytes.  dim 3: pos float[3], v_and_m float[4], three
// columns of three floats; dim 2: pos float[2], v_and_m float[3], two columns of two floats.
static void aos_window(const MpmbAosLayout *L, int dim, int *lo, int *hi) {
  const int mat = (dim - 1) * L->col_pitch + 4 * dim;  // padded columns, the last one dim floats long
  int a = std::min(std::min(L->off_pos, L->off_v_and_m), std::min(L->off_dg_e, L->off_apic_b));
  int b = std::max(std::max(L->off_pos + 4 * dim, L->off_v_and_m + 4 * (dim + 1)), std::max(L->off_dg_e + mat, L->off_apic_b + mat));
  a = std::min(a, L->off_vol);
  b = std::max(b, L->off_vol + 4);
  if (L->off_scalar >= 0) { a = std::min(a, L->off_scalar); b = std::max(b, L->off_scalar + 4); }
  for (int k = 0; k < 4; k++)
    if (L->off_scalar_by_kind[k] > 0) { a = std::min(a, L->off_scalar_by_kind[k]); b = std::max(b, L->off_scalar_by_kind[k] + 4); }
  *lo = std::max(0, a & ~15);
  *hi = std::min(L->stride, (b + 15) & ~15);
}

// the layout's scalar mode: per kind when any off_scalar_by_kind entry is set, checked (MpmbAosLayout in mpmb.h)
static int aos_scalar_mode(MpmbEngine *h, const MpmbAosLayout *L, bool *per_kind) {
  *per_kind = false;
  for (int k = 0; k < 4; k++) *per_kind |= L->off_scalar_by_kind[k] != 0;
  if (!*per_kind) return MPMB_OK;
  if (L->off_scalar != -1) return fail(h, MPMB_ERR_INVALID, "per-kind scalar offsets need off_scalar = -1");
  for (int k = 0; k < 4; k++) {
    const int32_t o = L->off_scalar_by_kind[k];
    if (o != -1 && (o <= 0 || o > L->stride - 4 || (o & 3)))
      return fail(h, MPMB_ERR_INVALID, "off_scalar_by_kind[%d] = %d is not -1 or a 4-aligned offset in (0, stride - 4]", k, o);
  }
  return MPMB_OK;
}

// per-group scalar offsets and defaults from a group -> kind table (the snapshot of mpmb_upload_aos)
static AosScalars aos_scalars(const MpmbAosLayout *L, const int32_t *kinds, bool per_kind) {
  AosScalars S{};
  S.on = per_kind ? 1 : 0;
  for (int g = 0; g < MPMB_MAX_GROUPS; g++) {
    const int kind = kinds[g];
    const int k = kind == MAT_SNOW ? 0 : kind == MAT_WATER ? 1 : kind == MAT_SAND ? 2 : kind == MAT_VISCO ? 3 : -1;
    S.off[g] = k >= 0 ? L->off_scalar_by_kind[k] : -1;
    S.dflt[g] = (kind == MAT_SNOW || kind == MAT_WATER) ? 1.0f : 0.0f;   // as mpmb_upload_particles with scalar = NULL
  }
  return S;
}

static int aos_reserve(MpmbEngine *h, size_t pool_bytes, size_t n_idx) {
  CUDA_TRY(h, h->aos_pool.reserve(pool_bytes));
  CUDA_TRY(h, h->aos_idx.reserve(n_idx));
  return MPMB_OK;
}

// ---- the AoS calls of a 2-D handle (kernels k2_pack_aos / k2_aos_scatter in the 2-D engine's section)
// MpmbAosLayout against MPMParticle<2>'s extents: every field inside the slot, 4-aligned (the kernels read floats)
static int m2_aos_layout_check(MpmbEngine *h, const MpmbAosLayout *L, bool *per_kind) {
  const int32_t st = L->stride, cp = L->col_pitch;
  if (st <= 0 || (st & 3)) return fail(h, MPMB_ERR_INVALID, "2-D handle: layout stride %d is not a positive multiple of 4", st);
  if (cp < 8 || (cp & 3)) return fail(h, MPMB_ERR_INVALID, "2-D handle: col_pitch %d is not a multiple of 4 >= 8", cp);
  const int32_t off[5] = {L->off_pos, L->off_v_and_m, L->off_dg_e, L->off_apic_b, L->off_vol};
  const int32_t len[5] = {8, 12, cp + 8, cp + 8, 4};
  static const char *name[5] = {"off_pos", "off_v_and_m", "off_dg_e", "off_apic_b", "off_vol"};
  for (int k = 0; k < 5; k++)
    if (off[k] < 0 || (off[k] & 3) || off[k] > st - len[k])
      return fail(h, MPMB_ERR_INVALID, "2-D handle: %s = %d with %d bytes is not a 4-aligned field inside the %d-byte slot", name[k], off[k], len[k], st);
  if (L->off_scalar != -1 && (L->off_scalar < 0 || (L->off_scalar & 3) || L->off_scalar > st - 4))
    return fail(h, MPMB_ERR_INVALID, "2-D handle: off_scalar = %d is not -1 or a 4-aligned offset inside the slot", L->off_scalar);
  return aos_scalar_mode(h, L, per_kind);
}

static int m2_upload_aos(MpmbEngine *h, int64_t n, const void *pool, int64_t pool_slots, const uint32_t *indices, const MpmbAosLayout *L,
                         const int32_t *group) {
  Mpm2d *m = h->m2;
  if (n < 0 || !pool || !indices || !L || pool_slots < 0) return fail(h, MPMB_ERR_INVALID, "2-D handle: pool, indices and layout are required");
  bool per_kind;
  int rc = m2_aos_layout_check(h, L, &per_kind);
  if (rc != MPMB_OK) return rc;
  if ((int64_t)m->id_base + n > (1ll << TAG_ID_BITS)) return fail(h, MPMB_ERR_CAPACITY, "particle ids exceed 2^%d", TAG_ID_BITS);
  if (m->stage != 0) return fail(h, MPMB_ERR_STATE, "upload between substeps, not inside one");
  if (h->cfg.capacity > 0 && n > m->cap) return fail(h, MPMB_ERR_CAPACITY, "%lld particles exceed the configured capacity %lld", (long long)n, (long long)m->cap);
  if (n > m->cap) {
    if ((rc = m2_alloc_rows(h, n)) != MPMB_OK) return rc;
    m->rows = 0;   // the new storage holds nothing yet
  }
  h->aos_host_pool = nullptr;   // the device image is rewritten below
  int32_t kinds[MPMB_MAX_GROUPS];
  for (int g = 0; g < MPMB_MAX_GROUPS; g++) kinds[g] = m->P.mats[g].kind;
  const size_t pool_bytes = (size_t)pool_slots * L->stride;
  if (n > 0 && (rc = aos_reserve(h, pool_bytes, (size_t)n)) != MPMB_OK) return rc;
  CUDA_TRY(h, cudaMemsetAsync(&m->cnt.get()->aos_error, 0, sizeof(int), h->stream));
  if (n > 0) {
    const int *d_grp = nullptr;
    if (group) {
      CUDA_TRY(h, m->stage_buf.reserve((size_t)n));
      d_grp = (const int *)m->stage_buf.get();
      CUDA_TRY(h, cudaMemcpyAsync(m->stage_buf.get(), group, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
    }
    CUDA_TRY(h, cudaMemcpyAsync(h->aos_idx.get(), indices, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, h->stream));
    if (pool_slots > 0) {
      int lo, hi;
      aos_window(L, 2, &lo, &hi);
      CUDA_TRY(h, cudaMemcpy2DAsync(h->aos_pool.get() + lo, (size_t)L->stride, (const char *)pool + lo, (size_t)L->stride, (size_t)(hi - lo),
                                    (size_t)pool_slots, cudaMemcpyHostToDevice, h->stream));
    }
    k2_pack_aos<<<m2_blocks(n, 128), 128, 0, h->stream>>>(m2_view(h), m->P, (int)n, h->aos_pool.get(), pool_slots, h->aos_idx.get(), *L,
                                                           aos_scalars(L, kinds, per_kind), d_grp, m->id_base);
    h->launches++;
  }
  int err = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&err, &m->cnt.get()->aos_error, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  if (err & DEVERR_BAD_SLOT)   // the packed rows are in the spare buffers: the resident set stays as it was
    return fail(h, MPMB_ERR_INVALID, "2-D handle: a slot index is outside the pool of %lld slots", (long long)pool_slots);
  // keep the new rows: the spare buffers become the current ones and keys_sorted the keys; the counters restart as after
  // mpmb_upload_particles, with a bad group or mass reported by the next synchronize
  m2_graph_reset(m);
  m->cur ^= 1;
  std::swap(m->keys, m->keys_sorted);
  m->rows = n;
  const int c3[3] = {0, 0, err & DEVERR_BAD_INPUT};   // n_alive, n_live, error
  CUDA_TRY(h, cudaMemcpy(m->cnt.get(), c3, sizeof(c3), cudaMemcpyHostToDevice));
  if (n > 0) {
    h->aos_host_pool = pool;
    h->aos_slots = pool_slots;
    h->aos_n = n;
  }
  std::copy(kinds, kinds + MPMB_MAX_GROUPS, h->aos_kinds);
  h->aos_kinds_valid = true;
  return MPMB_OK;
}

static int m2_download_aos(MpmbEngine *h, void *pool, int64_t pool_slots, uint32_t *indices, int64_t n_indices, const MpmbAosLayout *L,
                           int64_t *n_alive) {
  Mpm2d *m = h->m2;
  if (!pool || !indices || !L || !n_alive || n_indices < 0 || pool_slots < 0)
    return fail(h, MPMB_ERR_INVALID, "2-D handle: pool, indices, layout and n_alive are required");
  bool per_kind;
  int rc = m2_aos_layout_check(h, L, &per_kind);
  if (rc != MPMB_OK) return rc;
  if (per_kind && !h->aos_kinds_valid)
    return fail(h, MPMB_ERR_STATE, "per-kind scalar offsets need the group kinds of an mpmb_upload_aos of the resident set");
  if ((rc = m2_synchronize(h)) != MPMB_OK) return rc;
  *n_alive = 0;
  if (n_indices == 0) return MPMB_OK;
  if (m->cap < n_indices) return fail(h, MPMB_ERR_CAPACITY, "index vector longer than the particle capacity");
  // the device image of the pool: still resident from mpmb_upload_aos of the same pool, else brought in now
  const bool resident = h->aos_host_pool == pool && h->aos_slots == pool_slots && h->aos_n == n_indices && h->aos_pool.get();
  h->aos_host_pool = nullptr;   // the image is written below: the next download reads the host pool again
  if (!resident) {
    if ((rc = aos_reserve(h, (size_t)pool_slots * L->stride, (size_t)n_indices)) != MPMB_OK) return rc;
    CUDA_TRY(h, cudaMemcpyAsync(h->aos_idx.get(), indices, sizeof(uint32_t) * n_indices, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->aos_pool.get(), pool, (size_t)pool_slots * L->stride, cudaMemcpyHostToDevice, h->stream));
  }
  if ((rc = scan_reserve(h, (size_t)n_indices + 1)) != MPMB_OK) return rc;   // + 1: the room for aos_error behind the total
  CUDA_TRY(h, cudaMemsetAsync(h->scan_a.get(), 0, sizeof(int) * (size_t)n_indices, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(&m->cnt.get()->aos_error, 0, sizeof(int), h->stream));
  if (m->rows > 0) {
    k2_aos_scatter<<<m2_blocks(m->rows, 128), 128, 0, h->stream>>>(m2_view(h), m->P, (int)m->rows, h->aos_pool.get(), h->aos_idx.get(), n_indices,
                                                                    pool_slots, *L, aos_scalars(L, h->aos_kinds, per_kind), m->id_base, h->scan_a.get());
    h->launches++;
  }
  int alive = 0, err = 0;
  if ((rc = scan_flags(h, (size_t)n_indices, &alive, &m->cnt.get()->aos_error, &err)) != MPMB_OK) return rc;
  if (err & DEVERR_BAD_SLOT)   // nothing has reached the host pool or the index vector yet
    return fail(h, MPMB_ERR_INVALID, "2-D handle: a particle id or slot index is outside the index vector of %lld or the pool of %lld slots",
                (long long)n_indices, (long long)pool_slots);
  // survivors' slots in id order == what clear_boundary_particles leaves in MPM::particles (src/mpm.cpp:618-622); the
  // scratch is keys_sorted, which the next ordering rewrites
  uint32_t *d_surv = m->keys_sorted.get();
  k_compact_survivors<<<(unsigned)((n_indices + 255) / 256), 256, 0, h->stream>>>(h->aos_idx.get(), h->scan_a.get(), h->scan_b.get(), n_indices, d_surv);
  h->launches++;
  if (pool_slots > 0) {  // only the window of every slot that holds the layout's fields comes back
    int lo, hi;
    aos_window(L, 2, &lo, &hi);
    CUDA_TRY(h, cudaMemcpy2DAsync((char *)pool + lo, (size_t)L->stride, h->aos_pool.get() + lo, (size_t)L->stride, (size_t)(hi - lo), (size_t)pool_slots,
                                  cudaMemcpyDeviceToHost, h->stream));
  }
  if (alive > 0) CUDA_TRY(h, cudaMemcpyAsync(indices, d_surv, sizeof(uint32_t) * (size_t)alive, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  *n_alive = alive;
  return MPMB_OK;
}

int mpmb_upload_aos(MpmbHandle h, int64_t n, const void *pool, int64_t pool_slots, const uint32_t *indices,
                    const MpmbAosLayout *L, const int32_t *group) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_upload_aos(h, n, pool, pool_slots, indices, L, group);
  if (n < 0 || !pool || !indices || !L || L->stride <= 0) return fail(h, MPMB_ERR_INVALID, "pool, indices and layout are required");
  if ((int64_t)h->id_base + n > (1ll << TAG_ID_BITS)) return fail(h, MPMB_ERR_CAPACITY, "particle ids exceed 2^%d", TAG_ID_BITS);
  bool per_kind;
  int rc = aos_scalar_mode(h, L, &per_kind);
  if (rc != MPMB_OK) return rc;
  if ((rc = ensure_capacity(h, n)) != MPMB_OK) return rc;
  h->aos_host_pool = nullptr;
  int32_t kinds[MPMB_MAX_GROUPS];
  for (int g = 0; g < MPMB_MAX_GROUPS; g++) kinds[g] = h->P.mats[g].kind;
  if (n == 0) {
    if ((rc = finish_upload(h, 0)) != MPMB_OK) return rc;
    std::copy(kinds, kinds + MPMB_MAX_GROUPS, h->aos_kinds);
    h->aos_kinds_valid = true;
    return MPMB_OK;
  }
  // the pool's device image and the index vector stay resident (grow-only buffers): mpmb_download_aos scatters the
  // results into the image and returns it with one contiguous copy
  const size_t pool_bytes = (size_t)pool_slots * L->stride;
  if ((rc = aos_reserve(h, pool_bytes, (size_t)n)) != MPMB_OK) return rc;
  int *d_grp = nullptr;
  if (group) {
    CUDA_TRY(h, h->stage_buf.reserve(sizeof(int) * (size_t)n));
    d_grp = (int *)h->stage_buf.get();
    CUDA_TRY(h, cudaMemcpyAsync(d_grp, group, sizeof(int) * n, cudaMemcpyHostToDevice, h->stream));
  }
  CUDA_TRY(h, cudaMemcpyAsync(h->aos_idx.get(), indices, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, h->stream));
  {
    int lo, hi;
    aos_window(L, 3, &lo, &hi);
    CUDA_TRY(h, cudaMemcpy2DAsync(h->aos_pool.get() + lo, (size_t)L->stride, (const char *)pool + lo, (size_t)L->stride, (size_t)(hi - lo), (size_t)pool_slots,
                                  cudaMemcpyHostToDevice, h->stream));
  }
  View V = make_view(h);
  k_pack_aos<<<(unsigned)((n + 127) / 128), 128, 0, h->stream>>>(V, h->P, (int)n, h->aos_pool.get(), h->aos_idx.get(), *L, aos_scalars(L, kinds, per_kind),
                                                                  d_grp, h->keys[h->cur].get(), h->id_base);
  h->launches++;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  h->aos_host_pool = pool;
  h->aos_slots = pool_slots;
  h->aos_n = n;
  if ((rc = finish_upload(h, n)) != MPMB_OK) return rc;
  std::copy(kinds, kinds + MPMB_MAX_GROUPS, h->aos_kinds);
  h->aos_kinds_valid = true;
  return MPMB_OK;
}

int mpmb_seed_lattice(MpmbHandle h, const int32_t lo_cell[3], const int32_t hi_cell[3], float vol, float mass, float jitter, uint32_t seed,
                      int32_t group, const float v0[3], int64_t *n_seeded) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!lo_cell || !hi_cell) return fail(h, MPMB_ERR_INVALID, "null argument");
  if (group < 0 || group >= MPMB_MAX_GROUPS || !(mass > 0.f) || !(vol > 0.f)) return fail(h, MPMB_ERR_INVALID, "bad group, mass or volume");
  SeedBox B{};
  size_t cells = 1;
  for (int d = 0; d < 3; d++) {
    B.lo[d] = lo_cell[d];
    B.n[d] = hi_cell[d] - lo_cell[d];
    if (B.n[d] <= 0 || lo_cell[d] < 0 || hi_cell[d] > h->P.res[d]) return fail(h, MPMB_ERR_INVALID, "empty or out-of-domain cell block");
    cells *= (size_t)B.n[d];
    B.v0[d] = v0 ? v0[d] : 0.f;
  }
  if (cells * 8 + (size_t)h->id_base > (size_t)(1ll << TAG_ID_BITS)) return fail(h, MPMB_ERR_CAPACITY, "lattice ids exceed 2^%d", TAG_ID_BITS);
  // candidate cell layers: a particle of cell layer kz has its base node in layer kz-1 or kz (|jitter| < 0.25)
  B.z_first = 0;
  B.z_count = B.n[2];
  if (h->cfg.world > 1) {
    const int c0 = std::max(B.lo[2], 4 * h->P.tile_z0 - 1), c1 = std::min(B.lo[2] + B.n[2], 4 * h->P.tile_z1 + 2);
    B.z_first = c0 - B.lo[2];
    B.z_count = std::max(0, c1 - c0);
  }
  B.jitter = jitter; B.vol = vol; B.mass = mass; B.seed = seed; B.id_base = h->id_base; B.group = group;
  const int kind = h->P.mats[group].kind;
  B.ps = (kind == MAT_SNOW || kind == MAT_WATER) ? 1.0f : 0.0f;
  const size_t n_cand = (size_t)B.n[0] * B.n[1] * (size_t)B.z_count * 8;
  h->aos_host_pool = nullptr;
  if (n_cand >= (size_t)0x7fffffff) return fail(h, MPMB_ERR_CAPACITY, "too many candidate particles for one rank");
  int total = 0, rc;
  if (n_cand > 0) {
    if ((rc = scan_reserve(h, n_cand)) != MPMB_OK) return rc;
    k_seed_flags<<<h->num_sms * 8, 256, 0, h->stream>>>(h->P, B, n_cand, h->scan_a.get());
    if ((rc = scan_flags(h, n_cand, &total)) != MPMB_OK) return rc;
  }
  if ((rc = ensure_capacity(h, total)) != MPMB_OK) return rc;
  if (total > 0) {
    View V = make_view(h);
    k_seed_write<<<h->num_sms * 8, 256, 0, h->stream>>>(V, h->P, B, n_cand, h->scan_a.get(), h->scan_b.get(), h->keys[h->cur].get());
    h->launches += 2;
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    CUDA_TRY(h, cudaGetLastError());
  }
  if (n_seeded) *n_seeded = total;
  h->id_span_pending = (int64_t)n_cand;   // ids = lattice index
  rc = finish_upload(h, total);
  h->id_end = (int64_t)h->id_base + (int64_t)cells * 8;   // the whole lattice's ids, whichever of them this rank created
  return rc;
}

static int read_n_store(MpmbEngine *h, int *n_store) {
  Counters c;
  CUDA_TRY(h, cudaMemcpy(&c, h->cnt.get(), sizeof(c), cudaMemcpyDeviceToHost));
  *n_store = c.n_store;
  return MPMB_OK;
}

int mpmb_num_particles(MpmbHandle h, int64_t *n) {
  CHECK_HANDLE(h);
  if (!n) return fail(h, MPMB_ERR_INVALID, "null argument");
  *n = 0;
  if (h->m2) return m2_num_particles(h, n);
  if (h->cap == 0) return MPMB_OK;
  CUDA_TRY(h, cudaMemsetAsync(&h->cnt.get()->n_live, 0, sizeof(int), h->stream));
  k_count_live<<<h->num_sms * 4, 256, 0, h->stream>>>(h->keys[h->cur].get(), h->special_min, h->cnt.get());
  h->launches++;
  int rc = mpmb_synchronize(h);
  if (rc != MPMB_OK) return rc;
  int live = 0;
  CUDA_TRY(h, cudaMemcpy(&live, &h->cnt.get()->n_live, sizeof(int), cudaMemcpyDeviceToHost));
  *n = live;
  return MPMB_OK;
}

int mpmb_get_update_count(MpmbHandle h, int64_t *updates) {
  CHECK_HANDLE(h);
  if (!updates) return fail(h, MPMB_ERR_INVALID, "null argument");
  int rc = mpmb_synchronize(h);
  if (rc != MPMB_OK) return rc;
  if (h->m2) {
    unsigned long long u = 0;
    CUDA_TRY(h, cudaMemcpy(&u, &h->m2->cnt.get()->updates, sizeof(u), cudaMemcpyDeviceToHost));
    *updates = (int64_t)u;
    return MPMB_OK;
  }
  unsigned long long u = 0;
  CUDA_TRY(h, cudaMemcpy(&u, &h->cnt.get()->updates, sizeof(u), cudaMemcpyDeviceToHost));
  *updates = (int64_t)u;
  return MPMB_OK;
}

// The live rows among the n rows of the current storage: alive flags and their exclusive prefix (scan_a / scan_b), *alive
// their number.  Followed by unpack_live: the one unpacking path of downloads and AsyncMPM advances.
static int live_prefix(MpmbEngine *h, int n, int64_t *alive) {
  int rc, total = 0;
  if ((rc = scan_reserve(h, (size_t)n)) != MPMB_OK) return rc;
  k_alive_flags<<<(n + 255) / 256, 256, 0, h->stream>>>(h->keys[h->cur].get(), n, h->special_min, h->scan_a.get());
  if ((rc = scan_flags(h, (size_t)n, &total)) != MPMB_OK) return rc;
  *alive = total;
  return MPMB_OK;
}

// The live rows, compacted in storage order, into DEVICE arrays (any may be NULL); id = the engine's particle id.
static void unpack_live(MpmbEngine *h, int n, uint32_t *id, float *x, float *v, float *F, float *b, float *mass, float *vol, float *scalar, int *group) {
  View V = make_view(h);
  k_unpack_particles<<<(n + 127) / 128, 128, 0, h->stream>>>(V, h->keys[h->cur].get(), n, h->special_min, id, x, v, F, b, mass, vol, scalar, group, h->scan_b.get());
  h->launches += 2;
}

int mpmb_download_particles(MpmbHandle h, int64_t cap, int64_t *n_out, uint32_t *id, float *x, float *v, float *F, float *b,
                            float *mass, float *vol, float *scalar, int32_t *group) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_download(h, cap, n_out, id, x, v, F, b, mass, vol, scalar, group);
  if (!n_out) return fail(h, MPMB_ERR_INVALID, "n_out is required");
  int rc = mpmb_synchronize(h);
  if (rc != MPMB_OK) return rc;
  int n = 0;
  if ((rc = read_n_store(h, &n)) != MPMB_OK) return rc;
  *n_out = 0;
  if (n == 0 || h->cap == 0) return MPMB_OK;
  int64_t alive = 0;
  if ((rc = live_prefix(h, n, &alive)) != MPMB_OK) return rc;
  if (alive > cap) return fail(h, MPMB_ERR_CAPACITY, "%lld live particles do not fit in the %lld rows provided", (long long)alive, (long long)cap);
  size_t fl = (size_t)alive * ((x ? 3 : 0) + (v ? 3 : 0) + (F ? 9 : 0) + (b ? 9 : 0) + (mass ? 1 : 0) + (vol ? 1 : 0) + (scalar ? 1 : 0) +
                               (id ? 1 : 0) + (group ? 1 : 0));
  CUDA_TRY(h, h->stage_buf.reserve(fl * sizeof(float)));
  float *p = (float *)h->stage_buf.get();
  auto take = [&](bool want, size_t per) -> float * {
    if (!want) return nullptr;
    float *r = p;
    p += per * alive;
    return r;
  };
  float *dx_ = take(x, 3), *dv = take(v, 3), *dF = take(F, 9), *db = take(b, 9), *dm = take(mass, 1), *dvol = take(vol, 1), *ds = take(scalar, 1);
  uint32_t *did = (uint32_t *)take(id, 1);
  int *dg = (int *)take(group, 1);
  unpack_live(h, n, did, dx_, dv, dF, db, dm, dvol, ds, dg);
  auto get = [&](void *dst, const void *src, size_t per) {
    if (dst) cudaMemcpyAsync(dst, src, per * alive * sizeof(float), cudaMemcpyDeviceToHost, h->stream);
  };
  get(x, dx_, 3); get(v, dv, 3); get(F, dF, 9); get(b, db, 9); get(mass, dm, 1); get(vol, dvol, 1); get(scalar, ds, 1);
  get(id, did, 1); get(group, dg, 1);
  cudaError_t e = cudaStreamSynchronize(h->stream);
  CUDA_TRY(h, e);
  CUDA_TRY(h, cudaGetLastError());
  *n_out = alive;
  return MPMB_OK;
}

int mpmb_download_aos(MpmbHandle h, void *pool, int64_t pool_slots, uint32_t *indices, int64_t n_indices, const MpmbAosLayout *L,
                      int64_t *n_alive) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_download_aos(h, pool, pool_slots, indices, n_indices, L, n_alive);
  if (!pool || !indices || !L || !n_alive || L->stride <= 0 || n_indices < 0) return fail(h, MPMB_ERR_INVALID, "null argument");
  bool per_kind;
  int ns = 0, rc = aos_scalar_mode(h, L, &per_kind);
  if (rc != MPMB_OK) return rc;
  if (per_kind && !h->aos_kinds_valid)
    return fail(h, MPMB_ERR_STATE, "per-kind scalar offsets need the group kinds of an mpmb_upload_aos of the resident set");
  if ((rc = mpmb_synchronize(h)) != MPMB_OK) return rc;
  if ((rc = read_n_store(h, &ns)) != MPMB_OK) return rc;
  *n_alive = 0;
  if (n_indices == 0) return MPMB_OK;
  const size_t pool_bytes = (size_t)pool_slots * L->stride;
  // the device image of the pool: still resident from mpmb_upload_aos of the same pool, else brought in now
  const bool resident = h->aos_host_pool == pool && h->aos_slots == pool_slots && h->aos_n == n_indices && h->aos_pool.get();
  if (!resident) {
    if ((rc = aos_reserve(h, pool_bytes, (size_t)n_indices)) != MPMB_OK) return rc;
    CUDA_TRY(h, cudaMemcpyAsync(h->aos_idx.get(), indices, sizeof(uint32_t) * n_indices, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->aos_pool.get(), pool, pool_bytes, cudaMemcpyHostToDevice, h->stream));
  }
  (void)pool_bytes;
  if ((rc = scan_reserve(h, (size_t)n_indices)) != MPMB_OK) return rc;
  CUDA_TRY(h, cudaMemsetAsync(h->scan_a.get(), 0, sizeof(int) * (size_t)n_indices, h->stream));
  if (ns > 0 && h->cap > 0) {
    View V = make_view(h);
    k_aos_scatter<<<(ns + 127) / 128, 128, 0, h->stream>>>(V, h->keys[h->cur].get(), ns, h->special_min, h->aos_pool.get(), h->aos_idx.get(), n_indices, pool_slots, *L,
                                                           aos_scalars(L, h->aos_kinds, per_kind), h->id_base, h->scan_a.get(), h->cnt.get());
    h->launches++;
  }
  int alive = 0;
  if ((rc = scan_flags(h, (size_t)n_indices, &alive)) != MPMB_OK) return rc;
  // survivors' slots in id order == what clear_boundary_particles leaves in MPM::particles (src/mpm.cpp:618-622)
  uint32_t *d_surv = (uint32_t *)h->keys_sorted.get();  // upload-time scratch, free between uploads; cap >= n rows
  if ((int64_t)h->cap < n_indices) return fail(h, MPMB_ERR_CAPACITY, "index vector longer than the particle capacity");
  k_compact_survivors<<<(unsigned)((n_indices + 255) / 256), 256, 0, h->stream>>>(h->aos_idx.get(), h->scan_a.get(), h->scan_b.get(), n_indices, d_surv);
  h->launches++;
  {  // only the window of every slot that holds the layout's fields comes back; the rest of the host pool is untouched
    int lo, hi;
    aos_window(L, 3, &lo, &hi);
    CUDA_TRY(h, cudaMemcpy2DAsync((char *)pool + lo, (size_t)L->stride, h->aos_pool.get() + lo, (size_t)L->stride, (size_t)(hi - lo), (size_t)pool_slots,
                                  cudaMemcpyDeviceToHost, h->stream));
  }
  if (alive > 0) CUDA_TRY(h, cudaMemcpyAsync(indices, d_surv, sizeof(uint32_t) * (size_t)alive, cudaMemcpyDeviceToHost, h->stream));
  if ((rc = mpmb_synchronize(h)) != MPMB_OK) return rc;   // also surfaces ids / slots outside the vectors
  CUDA_TRY(h, cudaGetLastError());
  h->aos_host_pool = nullptr;   // the host owns the pool again: the next upload refreshes the image
  *n_alive = alive;
  return MPMB_OK;
}

int mpmb_download_bgeo_points(MpmbHandle h, int64_t id_range, void *records, int64_t cap_records, int64_t *n_out) {
  CHECK_HANDLE(h);
  if (!records || !n_out || id_range <= 0) return fail(h, MPMB_ERR_INVALID, "bad argument");
  if (h->m2) return m2_bgeo_points(h, id_range, records, cap_records, n_out);
  int ns = 0, rc;
  if ((rc = mpmb_synchronize(h)) != MPMB_OK) return rc;
  if ((rc = read_n_store(h, &ns)) != MPMB_OK) return rc;
  *n_out = 0;
  if (ns == 0 || h->cap == 0) return MPMB_OK;
  if ((rc = scan_reserve(h, (size_t)id_range)) != MPMB_OK) return rc;
  CUDA_TRY(h, cudaMemsetAsync(h->scan_a.get(), 0, sizeof(int) * (size_t)id_range, h->stream));
  View V = make_view(h);
  k_id_flags<<<(ns + 255) / 256, 256, 0, h->stream>>>(V, h->keys[h->cur].get(), ns, h->special_min, h->id_base, id_range, h->scan_a.get(), h->cnt.get());
  int alive = 0;
  if ((rc = scan_flags(h, (size_t)id_range, &alive)) != MPMB_OK) return rc;
  if (alive > cap_records) return fail(h, MPMB_ERR_CAPACITY, "%d live particles do not fit in the %lld records provided", alive, (long long)cap_records);
  const size_t bytes = (size_t)alive * 48;
  CUDA_TRY(h, h->stage_buf.reserve(bytes));
  k_bgeo_points<<<(ns + 127) / 128, 128, 0, h->stream>>>(V, h->keys[h->cur].get(), ns, h->special_min, h->id_base, id_range, h->scan_b.get(), (uint32_t *)h->stage_buf.get());
  h->launches += 2;
  CUDA_TRY(h, cudaMemcpyAsync(records, h->stage_buf.get(), bytes, cudaMemcpyDeviceToHost, h->stream));
  if ((rc = mpmb_synchronize(h)) != MPMB_OK) return rc;
  CUDA_TRY(h, cudaGetLastError());
  *n_out = alive;
  return MPMB_OK;
}

// ------------------------------------------------------------------------------ CPIC host side
static int rigid_reserve_ids(MpmbEngine *h, int64_t n_ids) {
  if (h->p_states.get() && n_ids <= (int64_t)h->p_states.size()) return MPMB_OK;
  const int64_t cap = std::max<int64_t>(n_ids, 1024);
  DevBuf<uint32_t> st, nr;
  DevBuf<float4> cdf;
  CUDA_TRY(h, st.alloc(cap));
  CUDA_TRY(h, cdf.alloc(cap));
  CUDA_TRY(h, nr.alloc(cap));
  CUDA_TRY(h, cudaMemsetAsync(st.get(), 0, sizeof(uint32_t) * cap, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(cdf.get(), 0, sizeof(float4) * cap, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(nr.get(), 0, sizeof(uint32_t) * cap, h->stream));   // epoch 0 is never current
  if (h->p_states.size() > 0)
    CUDA_TRY(h, cudaMemcpyAsync(st.get(), h->p_states.get(), sizeof(uint32_t) * h->p_states.size(), cudaMemcpyDeviceToDevice, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->p_states = std::move(st); h->p_cdf = std::move(cdf); h->p_mark = std::move(nr);
  graph_reset(h);   // the captured rigid kernels hold the freed arrays and the old id_cap
  return MPMB_OK;
}

// per substep, after the ordering: pages + colour field of this pose, tile flags, particle colours
static int rigid_prepare(MpmbEngine *h, const View &V, int *nl) {
  if (!h->p_states.get() || (int64_t)h->p_states.size() < rigid_ids(h)) { int rc = rigid_reserve_ids(h, std::max<int64_t>(rigid_ids(h), h->cap)); if (rc != MPMB_OK) return rc; }
  const RigidView R = rigid_view(h);
  const int ns = R.n_samples, sb = (ns + 127) / 128;
  k_cdf_clear<<<sb, 128, 0, h->stream>>>(R, h->P);
  CUDA_TRY(h, cudaMemsetAsync(R.page, 0, h->page.size(), h->stream));
  k_cdf_raster<<<sb, 128, 0, h->stream>>>(R, h->P);
  k_rigid_tile_flags<<<(h->cap_tiles + 127) / 128, 128, 0, h->stream>>>(V, h->P, R);
  k_gather_cdf<<<(int)((h->cap + 127) / 128), 128, 0, h->stream>>>(V, h->P, R);
  *nl += 4;
  return MPMB_OK;
}

int mpmb_set_rigid_samples(MpmbHandle h, int32_t n_bodies, int64_t n_samples, const float *offset3, const float *tri9, const int32_t *rigid_id) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->rigid_pending) return fail(h, MPMB_ERR_STATE, "rigid samples change between substeps, not inside one");
  if (n_samples == 0) { h->rigid_on = false; h->motion_on = false; graph_reset(h); return MPMB_OK; }
  if (n_bodies < 2 || n_bodies > RIGID_MAX || n_samples < 0 || n_samples > (1 << 24) || !offset3 || !tri9 || !rigid_id)
    return fail(h, MPMB_ERR_INVALID, "need 2..%d bodies (entry 0 is the background body) and their boundary samples", RIGID_MAX);
  if (h->P.nnode[0] > 1023 || h->P.nnode[1] > 1023 || h->P.nnode[2] > 1023) return fail(h, MPMB_ERR_INVALID, "rigid coupling supports grids up to 1022 cells per axis");
  for (int64_t s = 0; s < n_samples; s++)
    if (rigid_id[s] < 1 || rigid_id[s] >= n_bodies) return fail(h, MPMB_ERR_INVALID, "sample %lld names body %d (valid: 1..%d)", (long long)s, rigid_id[s], n_bodies - 1);
  h->rs_offset.reset(); h->rs_tri.reset(); h->rs_rigid.reset(); h->s_base.reset();   // the old samples go before the new ones come
  CUDA_TRY(h, h->rs_offset.alloc(3 * n_samples));
  CUDA_TRY(h, h->rs_tri.alloc(9 * n_samples));
  CUDA_TRY(h, h->rs_rigid.alloc(n_samples));
  CUDA_TRY(h, h->s_base.alloc(n_samples));
  CUDA_TRY(h, cudaMemcpyAsync(h->rs_offset.get(), offset3, sizeof(float) * 3 * n_samples, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(h->rs_tri.get(), tri9, sizeof(float) * 9 * n_samples, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(h->rs_rigid.get(), rigid_id, sizeof(int) * n_samples, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->s_base.get(), 0xff, sizeof(int) * n_samples, h->stream));
  h->rigid_samples = (int)n_samples;
  h->rigid_bodies = n_bodies;
  if (!h->bodies.get()) {
    CUDA_TRY(h, h->bodies.alloc(RIGID_MAX));
    CUDA_TRY(h, cudaMemsetAsync(h->bodies.get(), 0, sizeof(RigidDev) * RIGID_MAX, h->stream));
    CUDA_TRY(h, h->epoch.alloc(1));
    CUDA_TRY(h, cudaMemsetAsync(h->epoch.get(), 0, sizeof(uint32_t), h->stream));
    CUDA_TRY(h, h->master.alloc(RIGID_MAX));
    CUDA_TRY(h, h->cursor.alloc(1));
    CUDA_TRY(h, cudaMemsetAsync(h->cursor.get(), 0, sizeof(int), h->stream));
  }
  {  // per-body sample lists for the level-set collision (samples need not be grouped by body)
    std::vector<int> order((size_t)n_samples);
    int cnt[RIGID_MAX + 1] = {};
    for (int64_t s = 0; s < n_samples; s++) cnt[rigid_id[s] + 1]++;
    for (int b = 0; b < RIGID_MAX; b++) cnt[b + 1] += cnt[b];
    for (int b = 0; b <= RIGID_MAX; b++) h->s_begin[b] = cnt[b];
    for (int64_t s = 0; s < n_samples; s++) order[(size_t)cnt[rigid_id[s]]++] = (int)s;
    h->contact.reset();   // contacts: allocated by mpmb_set_rigid_motion when the collision is asked for
    CUDA_TRY(h, h->s_order.alloc(n_samples));
    CUDA_TRY(h, cudaMemcpyAsync(h->s_order.get(), order.data(), sizeof(int) * n_samples, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));   // `order` lives on this stack frame
  }
  const size_t nn = (size_t)h->P.nnode[0] * h->P.nnode[1] * h->P.nnode[2];
  if (!h->node_key.get()) {
    CUDA_TRY(h, h->node_key.alloc(nn));
    CUDA_TRY(h, h->node_tags.alloc(nn));
    int *nb = h->rigid_nb;
    nb[0] = (h->P.nnode[0] + 3) / 4 + 1; nb[1] = (h->P.nnode[1] + 3) / 4 + 1; nb[2] = (h->P.nnode[2] + 7) / 8 + 1;
    CUDA_TRY(h, h->page.alloc((size_t)nb[0] * nb[1] * nb[2]));
    CUDA_TRY(h, h->tile_flag.alloc(std::max(h->cap_tiles, 1)));
    CUDA_TRY(h, cudaMemsetAsync(h->tile_flag.get(), 0, h->tile_flag.size(), h->stream));
  }
  CUDA_TRY(h, cudaMemsetAsync(h->node_key.get(), 0xff, sizeof(unsigned long long) * nn, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->node_tags.get(), 0, sizeof(uint32_t) * nn, h->stream));
  if (h->pushing_force == 0.f && h->penalty == 0.f) h->pushing_force = 20000.0f;   // src/mpm.cpp:35,40 defaults
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->rigid_on = true;
  h->motion_on = false;   // motion records describe a set of bodies: mpmb_set_rigid_motion follows the samples
  // poses change between substeps: unless the device advances the bodies (mpmb_set_rigid_motion) the host drives every substep,
  // and mpmb_substep does not replay graphs (use_graph itself keeps what the configuration asked for)
  graph_reset(h);
  return MPMB_OK;
}

int mpmb_set_rigid_coupling(MpmbHandle h, float penalty, float pushing_force) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  h->penalty = penalty;
  h->pushing_force = pushing_force;
  graph_reset(h);   // both are kernel arguments
  return MPMB_OK;
}

int mpmb_set_rigid_state(MpmbHandle h, int32_t n_bodies, const MpmbRigidBody *bodies) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!h->rigid_on) return fail(h, MPMB_ERR_STATE, "no rigid bodies: call mpmb_set_rigid_samples first");
  if (n_bodies != h->rigid_bodies || !bodies) return fail(h, MPMB_ERR_INVALID, "expected %d bodies", h->rigid_bodies);
  if (h->rigid_pending) return fail(h, MPMB_ERR_STATE, "z-slab rank: the bodies change after the impulse reduction, not before it");
  RigidDev dev[RIGID_MAX];
  memset(dev, 0, sizeof(dev));
  for (int b = 0; b < n_bodies; b++) {
    const MpmbRigidBody &s = bodies[b];
    RigidDev &d = dev[b];
    for (int k = 0; k < 3; k++) { d.pos[k] = s.position[k]; d.vel[k] = s.velocity[k]; d.ang[k] = s.angular_velocity[k]; }
    for (int k = 0; k < 9; k++) { d.rot[k] = s.rot[k]; d.inv_inertia[k] = s.inv_inertia[k]; }
    d.inv_mass = s.inv_mass;
    d.fric[0] = s.frictions[0]; d.fric[1] = s.frictions[1];
  }
  CUDA_TRY(h, cudaMemcpyAsync(h->bodies.get(), dev, sizeof(RigidDev) * RIGID_MAX, cudaMemcpyHostToDevice, h->stream));
  if (h->motion_on) {   // the master states restart from the given records
    for (int b = 0; b < n_bodies; b++) {
      RigidMaster &m = h->h_master[b];
      for (int k = 0; k < 3; k++) { m.pos[k] = dev[b].pos[k]; m.vel[k] = dev[b].vel[k]; m.ang[k] = dev[b].ang[k]; }
      for (int k = 0; k < 9; k++) m.rot[k] = dev[b].rot[k];
    }
    CUDA_TRY(h, cudaMemcpyAsync(h->master.get(), h->h_master, sizeof(RigidMaster) * RIGID_MAX, cudaMemcpyHostToDevice, h->stream));
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));   // `dev` lives on this stack frame
  return MPMB_OK;
}

int mpmb_get_rigid_state(MpmbHandle h, int32_t n_bodies, MpmbRigidBody *bodies) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!h->rigid_on) return fail(h, MPMB_ERR_STATE, "no rigid bodies");
  if (n_bodies != h->rigid_bodies || !bodies) return fail(h, MPMB_ERR_INVALID, "expected %d bodies", h->rigid_bodies);
  RigidDev dev[RIGID_MAX];
  CUDA_TRY(h, cudaMemcpyAsync(dev, h->bodies.get(), sizeof(RigidDev) * RIGID_MAX, cudaMemcpyDeviceToHost, h->stream));
  int rc = mpmb_synchronize(h);
  if (rc != MPMB_OK) return rc;
  for (int b = 0; b < n_bodies; b++) {
    MpmbRigidBody &s = bodies[b];
    const RigidDev &d = dev[b];
    for (int k = 0; k < 3; k++) { s.position[k] = d.pos[k]; s.velocity[k] = d.vel[k]; s.angular_velocity[k] = d.ang[k]; }
    for (int k = 0; k < 9; k++) { s.rot[k] = d.rot[k]; s.inv_inertia[k] = d.inv_inertia[k]; }
    s.inv_mass = d.inv_mass;
    s.frictions[0] = d.fric[0]; s.frictions[1] = d.fric[1];
  }
  return MPMB_OK;
}

int mpmb_set_rigid_motion(MpmbHandle h, int32_t n_bodies, const MpmbRigidMotion *motion, int32_t levelset_collision) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (n_bodies == 0) { h->motion_on = false; graph_reset(h); return MPMB_OK; }
  if (!h->rigid_on) return fail(h, MPMB_ERR_STATE, "no rigid bodies: call mpmb_set_rigid_samples first");
  if (h->stage != 0 || h->rigid_pending) return fail(h, MPMB_ERR_STATE, "rigid motion changes between substeps, not inside one");
  if (n_bodies != h->rigid_bodies || !motion) return fail(h, MPMB_ERR_INVALID, "expected %d motion records", h->rigid_bodies);
  bool scripted = false;
  for (int b = 1; b < n_bodies; b++) {
    const MpmbRigidMotion &m = motion[b];
    bool ok = std::isfinite(m.mass) && std::isfinite(m.linear_damping) && std::isfinite(m.angular_damping) && std::isfinite(m.restitution);
    for (int k = 0; k < 9; k++) ok = ok && std::isfinite(m.inv_inertia_body[k]);
    for (int k = 0; k < 3; k++) ok = ok && std::isfinite(m.rotation_axis[k]);
    if (!ok) return fail(h, MPMB_ERR_INVALID, "motion record of body %d is not finite", b);
    if (!m.scripted_position && !(m.mass > 0.f)) return fail(h, MPMB_ERR_INVALID, "body %d: a free body needs a positive mass", b);
    scripted = scripted || m.scripted_position || m.scripted_rotation;
  }
  RigidDev dev[RIGID_MAX];   // the master states start from the current records
  CUDA_TRY(h, cudaMemcpyAsync(dev, h->bodies.get(), sizeof(RigidDev) * RIGID_MAX, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  memset(h->h_master, 0, sizeof(h->h_master));
  for (int b = 1; b < n_bodies; b++) {
    const MpmbRigidMotion &s = motion[b];
    RigidMaster &m = h->h_master[b];
    for (int k = 0; k < 3; k++) { m.pos[k] = dev[b].pos[k]; m.vel[k] = dev[b].vel[k]; m.ang[k] = dev[b].ang[k]; m.axis[k] = s.rotation_axis[k]; }
    for (int k = 0; k < 9; k++) { m.rot[k] = dev[b].rot[k]; m.inv_inertia_body[k] = s.inv_inertia_body[k]; }
    m.mass = s.mass;
    m.inv_mass = s.scripted_position ? 0.0 : 1.0 / (double)s.mass;   // set_infinity_mass (src/mpm_rigid_body.cpp:198-200)
    m.lin_damp = s.linear_damping; m.ang_damp = s.angular_damping; m.restitution = s.restitution;
    m.scripted_pos = s.scripted_position != 0;
    m.scripted_rot = s.scripted_rotation != 0;
  }
  CUDA_TRY(h, cudaMemcpyAsync(h->master.get(), h->h_master, sizeof(RigidMaster) * RIGID_MAX, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->cursor.get(), 0, sizeof(int), h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (levelset_collision) CUDA_TRY(h, h->contact.reserve((size_t)CONTACT_STRIDE * h->rigid_samples));
  h->script_left = 0;
  h->motion_scripted = scripted;
  h->motion_collide = levelset_collision != 0;
  h->motion_on = true;
  graph_reset(h);
  return MPMB_OK;
}

int mpmb_set_rigid_script(MpmbHandle h, int32_t n_substeps, const double *poses) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!h->rigid_on || !h->motion_on) return fail(h, MPMB_ERR_STATE, "no device-advanced bodies: call mpmb_set_rigid_motion first");
  if (h->stage != 0 || h->rigid_pending) return fail(h, MPMB_ERR_STATE, "the script changes between substeps, not inside one");
  if (n_substeps < 0 || (n_substeps > 0 && !poses)) return fail(h, MPMB_ERR_INVALID, "need n_substeps >= 0 and a table");
  const int nb = h->rigid_bodies;
  const size_t n = (size_t)n_substeps * nb * SCRIPT_STRIDE;
  for (int64_t e = 0; e < n_substeps; e++)   // only the scripted parts are read
    for (int b = 1; b < nb; b++) {
      const double *p = poses + ((size_t)e * nb + b) * SCRIPT_STRIDE;
      bool ok = true;
      if (h->h_master[b].scripted_pos) for (int k : {0, 1, 2, 12, 13, 14}) ok = ok && std::isfinite(p[k]);
      if (h->h_master[b].scripted_rot) for (int k = 3; k < 12; k++) ok = ok && std::isfinite(p[k]);
      if (h->h_master[b].scripted_rot) for (int k = 15; k < 18; k++) ok = ok && std::isfinite(p[k]);
      if (!ok) return fail(h, MPMB_ERR_INVALID, "script entry %lld of body %d is not finite", (long long)e, b);
    }
  if (n > h->script.size()) {   // geometric growth: a fixed frame length allocates once (and keeps the captured graphs)
    CUDA_TRY(h, h->script.alloc(std::max(n, 2 * h->script.size())));
    graph_reset(h);
  }
  if (n) CUDA_TRY(h, cudaMemcpyAsync(h->script.get(), poses, sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->cursor.get(), 0, sizeof(int), h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));   // the caller owns `poses`
  h->script_left = n_substeps;
  return MPMB_OK;
}

// after the second apic_b-velocity transfer of a substep: level-set impulses, then the advance (one script entry)
static void launch_rigid_motion(MpmbEngine *h) {
  const RigidView R = rigid_view(h);
  const MotionView M = motion_view(h);
  if (M.collide) {
    k_rigid_contacts<<<(R.n_samples + 127) / 128, 128, 0, h->stream>>>(R, M, h->P, h->sdf4.get());
    h->launches++;
  }
  k_rigid_advance<<<1, 32, 0, h->stream>>>(R, M, h->P, make_float3(h->cfg.gravity[0], h->cfg.gravity[1], h->cfg.gravity[2]));
  h->launches++;
  if (h->motion_scripted) h->script_left--;
}

int mpmb_set_particle_states(MpmbHandle h, int64_t n, const uint32_t *states) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!h->rigid_on) return fail(h, MPMB_ERR_STATE, "no rigid bodies");
  if (n < 0 || (n > 0 && !states)) return fail(h, MPMB_ERR_INVALID, "bad argument");
  int rc = rigid_reserve_ids(h, std::max<int64_t>(n, h->cap));
  if (rc != MPMB_OK) return rc;
  CUDA_TRY(h, cudaMemcpyAsync(h->p_states.get(), states, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return MPMB_OK;
}

int mpmb_get_particle_cdf(MpmbHandle h, int64_t n, uint32_t *states, float *normal3, float *distance, uint8_t *near_boundary) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!h->rigid_on || !h->p_states.get()) return fail(h, MPMB_ERR_STATE, "no rigid bodies / no substep yet");
  if (n < 0 || n > (int64_t)h->p_states.size()) return fail(h, MPMB_ERR_INVALID, "n exceeds the %d particle ids tracked", (int)h->p_states.size());
  std::vector<float4> cdf((size_t)n);
  std::vector<uint32_t> mark((size_t)n);
  uint32_t epoch = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&epoch, h->epoch.get(), sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  if (states) CUDA_TRY(h, cudaMemcpyAsync(states, h->p_states.get(), sizeof(uint32_t) * n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(mark.data(), h->p_mark.get(), sizeof(uint32_t) * n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(cdf.data(), h->p_cdf.get(), sizeof(float4) * n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  for (int64_t i = 0; i < n; i++) {   // particles gather_cdf did not see in the last substep: distance 0, normal 0, not near (138-146)
    const bool fresh = (mark[i] >> 1) == epoch;
    if (normal3) { normal3[3 * i] = fresh ? cdf[i].x : 0.f; normal3[3 * i + 1] = fresh ? cdf[i].y : 0.f; normal3[3 * i + 2] = fresh ? cdf[i].z : 0.f; }
    if (distance) distance[i] = fresh ? cdf[i].w : 0.f;
    if (near_boundary) near_boundary[i] = (fresh && (mark[i] & 1u)) ? 1 : 0;
  }
  return MPMB_OK;
}

int mpmb_download_cdf(MpmbHandle h, uint32_t *node_states, float *node_distance) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (!h->rigid_on) return fail(h, MPMB_ERR_STATE, "no rigid bodies");
  const size_t nn = h->node_key.size();
  std::vector<unsigned long long> key(nn);
  std::vector<uint32_t> tags(nn);
  CUDA_TRY(h, cudaMemcpyAsync(key.data(), h->node_key.get(), sizeof(unsigned long long) * nn, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(tags.data(), h->node_tags.get(), sizeof(uint32_t) * nn, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  for (size_t i = 0; i < nn; i++) {
    const bool has = key[i] != CDF_NO_KEY;
    if (node_states) node_states[i] = (tags[i] & CDF_TAG_MASK) | (has ? ((uint32_t)key[i] & 0xffu) << 24 : 0u);
    if (node_distance) {
      uint32_t bits = (uint32_t)(key[i] >> 32);
      float d;
      memcpy(&d, &bits, 4);
      node_distance[i] = has ? d * h->P.dx : 0.f;
    }
  }
  return MPMB_OK;
}

// ------------------------------------------------------------------------------ stages
int mpmb_sort_particles_and_populate_grid(MpmbHandle h) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_order(h);
  if (h->stage != 0) return fail(h, MPMB_ERR_STATE, "sort must follow resample/upload");
  if (h->rigid_pending) return fail(h, MPMB_ERR_STATE, "z-slab rank: the G2P rigid impulses of the last substep have not been reduced");
  prof_begin(h, 0);
  int nl = 3;
  if (h->cap > 0) {
    View V = make_view(h);
    k_order_a<<<h->ord_blocks, ORD_B, 0, h->stream>>>(V, h->ntot);
    k_order_b<<<1, 1024, 0, h->stream>>>(V, h->ord_blocks);
    k_order_c<<<h->ord_blocks, ORD_B, 0, h->stream>>>(V, h->ntot, h->P.nt[1], h->P.nt[2], h->P.tz_off);
    if (!h->fresh) {
      k_mover_place<<<h->num_sms * 2, 256, 0, h->stream>>>(V, h->ntot);
      k_mover_rank<<<h->num_sms * 2, 256, 0, h->stream>>>(V, h->ntot);
      nl += 2;
    }
#ifdef MPMB_VALIDATE
    if (!h->fresh) k_validate_order<<<h->num_sms * 2, 256, 0, h->stream>>>(V, h->ntot);
#endif
    h->fresh = false;
    if (h->rigid_on) {
      int rc = rigid_prepare(h, V, &nl);
      if (rc != MPMB_OK) return rc;
    }
  }
  h->launches += nl;
  prof_end(h, nl);
  CUDA_TRY(h, cudaGetLastError());
  h->stage = 1;
  return MPMB_OK;
}

int mpmb_rasterize(MpmbHandle h) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_rasterize(h);
  if (h->stage != 1) return fail(h, MPMB_ERR_STATE, "rasterize must follow sort_particles_and_populate_grid");
  prof_begin(h, 1);
  View V = make_view(h);
  if (h->cap > 0) k_p2g<<<h->grid_p2g, P2G_T, P2G_DYN_BYTES, h->stream>>>(V, h->P, 0);
  h->launches += 1;
  if (h->cap > 0 && h->rigid_on) {  // block_op_rigid for the tiles of rigid pages, then apply_tmp_velocity (src/transfer.cpp:578-580)
    k_p2g_rigid<<<h->num_sms * 4, 128, 0, h->stream>>>(V, h->P, rigid_view(h), 0);
    h->launches += 1;
    if (h->cfg.world == 1) {
      k_rigid_apply<<<1, 32, 0, h->stream>>>(rigid_view(h));
      h->launches += 1;
    }
  }
  if (h->rigid_on && h->cfg.world > 1) h->rigid_pending = 1;   // z-slab rank: the impulses are summed over the ranks first
  prof_end(h, 1);
  CUDA_TRY(h, cudaGetLastError());
  h->stage = 2;
  return MPMB_OK;
}

// the k_g2p instantiation for this scene: apic_b stored or not, the three later material kinds compiled in or not
static void launch_g2p(MpmbEngine *h, const View &V, int part, int commit, bool store_b) {
  bool ext = false;
  for (int g = 0; g < MPMB_MAX_GROUPS; g++) ext |= h->P.mats[g].kind > MAT_SAND;
  if (ext) {
    if (store_b) k_g2p<128, true, true><<<h->grid_g2p, 128, 0, h->stream>>>(V, h->P, part, commit);
    else k_g2p<128, false, true><<<h->grid_g2p, 128, 0, h->stream>>>(V, h->P, part, commit);
  } else {
    if (store_b) k_g2p<128, true, false><<<h->grid_g2p, 128, 0, h->stream>>>(V, h->P, part, commit);
    else k_g2p<128, false, false><<<h->grid_g2p, 128, 0, h->stream>>>(V, h->P, part, commit);
  }
}

int mpmb_resample(MpmbHandle h) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_resample(h);
  if (h->stage != 2) return fail(h, MPMB_ERR_STATE, "resample must follow rasterize");
  if (h->rigid_pending) return fail(h, MPMB_ERR_STATE, "z-slab rank: reduce the P2G rigid impulses over the ranks before the resample");
  const bool motion = h->rigid_on && h->motion_on;
  if (motion && h->motion_scripted && h->script_left < 1) return fail(h, MPMB_ERR_STATE, "the rigid script has no entry left for this substep");
  const bool slab_rigid = h->rigid_on && h->cfg.world > 1;   // the G2P impulses, then the advance, follow the reduction
  View V = make_view(h);
  prof_begin(h, 2);
  if (h->cap > 0) {
    if (h->rigid_on) {
      k_g2p_rigid<<<h->num_sms * 4, 128, 0, h->stream>>>(V, h->P, rigid_view(h), 0);
      h->launches += 1;
    }
    launch_g2p(h, V, 0, 1, !h->skip_b || h->rigid_on);   // rigid tiles read apic_b back (the impulse needs dt * force)
    if (h->rigid_on && !slab_rigid) {
      k_rigid_apply<<<1, 32, 0, h->stream>>>(rigid_view(h));       // src/transfer.cpp:967-969
      h->launches += 1;
    }
  }
  if (motion && !slab_rigid) launch_rigid_motion(h);     // advect_rigid_bodies (src/mpm_rigid_body.cpp:273-287)
  if (slab_rigid) h->rigid_pending = 2;
  h->launches += 1;
  prof_end(h, 1);
  CUDA_TRY(h, cudaGetLastError());
  h->cur ^= 1;  // the buffer G2P wrote is the current storage ...
  h->ord ^= 1;  // ... its runs / stay counts are the current ones ...
  h->mov ^= 1;  // ... and its mover list feeds the next ordering
  h->xstep++;
  h->stage = 0;
  return MPMB_OK;
}

static bool peers_connected(MpmbEngine *h);
static bool rigid_connected(MpmbEngine *h);
static void rigid_mail_send(MpmbEngine *h);
static int rigid_mail_recv(MpmbEngine *h);
static int xchg_halo_fused(MpmbEngine *h);
static int xchg_migrate_fused(MpmbEngine *h);
int mpmb_halo_send(MpmbHandle h, int32_t face);
int mpmb_halo_recv(MpmbHandle h, int32_t face);
int mpmb_migrate_send(MpmbHandle h, int32_t face);
int mpmb_migrate_recv(MpmbHandle h, int32_t face);

// z-slab runs: the same two stages in two launches each, boundary-layer tiles (part 1) and the
// rest (part 2), so that the host can put the halo exchange between them (include/mpmb.h).
int mpmb_rasterize_part(MpmbHandle h, int32_t part) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (part != 1 && part != 2) return fail(h, MPMB_ERR_INVALID, "part must be 1 (boundary) or 2 (interior)");
  if (!((part == 1 && h->stage == 1) || (part == 2 && h->stage == 11))) return fail(h, MPMB_ERR_STATE, "rasterize_part: boundary first, then interior, after sort");
  prof_begin(h, 1);
  View V = make_view(h);
  if (h->cap > 0) k_p2g<<<h->grid_p2g, P2G_T, P2G_DYN_BYTES, h->stream>>>(V, h->P, part);
  h->launches += 1;
  const bool slab_rigid = h->rigid_on && h->cfg.world > 1;
  if (h->cap > 0 && slab_rigid) {   // the boundary layers' rigid arenas are final before halo_pack / halo_send
    k_p2g_rigid<<<h->num_sms * 4, 128, 0, h->stream>>>(V, h->P, rigid_view(h), part);
    h->launches += 1;
  }
  if (slab_rigid && part == 2) h->rigid_pending = 1;
  prof_end(h, 1);
  CUDA_TRY(h, cudaGetLastError());
  h->stage = part == 1 ? 11 : 2;
  return MPMB_OK;
}

int mpmb_resample_part(MpmbHandle h, int32_t part) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (part != 1 && part != 2) return fail(h, MPMB_ERR_INVALID, "part must be 1 (boundary) or 2 (interior)");
  if (!((part == 2 && h->stage == 2) || (part == 1 && h->stage == 22))) return fail(h, MPMB_ERR_STATE, "resample_part: interior first, then boundary, after rasterize");
  if (h->rigid_pending) return fail(h, MPMB_ERR_STATE, "z-slab rank: reduce the P2G rigid impulses over the ranks before the resample");
  const bool slab_rigid = h->rigid_on && h->cfg.world > 1;
  if (slab_rigid && h->motion_on && h->motion_scripted && h->script_left < 1)
    return fail(h, MPMB_ERR_STATE, "the rigid script has no entry left for this substep");
  prof_begin(h, 2);
  View V = make_view(h);
  int nl = 1;
  if (h->cap > 0) {
    if (slab_rigid) {
      k_g2p_rigid<<<h->num_sms * 4, 128, 0, h->stream>>>(V, h->P, rigid_view(h), part);
      nl++;
    }
    launch_g2p(h, V, part, part == 1 ? 1 : 0, true);
  }
  h->launches += nl;
  prof_end(h, nl);
  CUDA_TRY(h, cudaGetLastError());
  if (part == 2) { h->stage = 22; return MPMB_OK; }
  if (slab_rigid) h->rigid_pending = 2;
  h->cur ^= 1;
  h->ord ^= 1;
  h->mov ^= 1;
  h->xstep++;
  h->stage = 0;
  return MPMB_OK;
}

// one substep; skip_b: do not store apic_b (an intermediate substep of mpmb_substep)
static int substep_once(MpmbEngine *h, bool peers, bool skip_b) {
  int rc;
  if ((rc = mpmb_sort_particles_and_populate_grid(h)) != MPMB_OK) return rc;
  if ((rc = mpmb_rasterize(h)) != MPMB_OK) return rc;
  if (peers && h->rigid_pending) {   // rigid z-slab rank: the P2G impulses summed over the ranks through the mailboxes
    rigid_mail_send(h);
    if ((rc = rigid_mail_recv(h)) != MPMB_OK) return rc;
  }
  if (peers && (rc = xchg_halo_fused(h)) != MPMB_OK) return rc;  // boundary-layer arenas into the neighbours' memory, theirs in as ghosts
  h->skip_b = skip_b;
#ifdef MPMB_CHECKED
  { static const char *dbg = getenv("MPMB_DBG_SKIPB"); if (dbg) h->skip_b = dbg[0] == '1'; }   // debug: force one k_g2p instantiation
#endif
  rc = mpmb_resample(h);
  h->skip_b = false;
  if (rc != MPMB_OK) return rc;
  if (peers && h->rigid_pending) {   // ... and the G2P impulses, then the device advance
    rigid_mail_send(h);
    if ((rc = rigid_mail_recv(h)) != MPMB_OK) return rc;
  }
  if (peers && (rc = xchg_migrate_fused(h)) != MPMB_OK) return rc;
  return MPMB_OK;
}

// Captures two substeps (both buffer parities) into a graph for the parity the engine is in, and leaves the engine's
// host-side state as if they had run; the caller launches the graph.  Any failure turns graphs off for this handle.
static int graph_capture_pair(MpmbEngine *h, bool peers) {
  const int par = h->cur;
  if (!h->cap_stream && cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking) != cudaSuccess) { h->use_graph = false; cudaGetLastError(); return MPMB_OK; }
  cudaStream_t user = h->stream;
  const int64_t l0 = h->launches;
  const int cur0 = h->cur, ord0 = h->ord, mov0 = h->mov, x0 = h->xstep;
  const int64_t left0 = h->script_left;
  h->stream = h->cap_stream;
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal);
  int rc = MPMB_OK;
  if (e == cudaSuccess) {
    rc = substep_once(h, peers, true);
    if (rc == MPMB_OK) rc = substep_once(h, peers, true);
    e = cudaStreamEndCapture(h->cap_stream, &g);
  }
  h->stream = user;
  if (e == cudaSuccess && rc == MPMB_OK && g) e = cudaGraphInstantiate(&h->graph_exec[par], g, 0);
  if (g) cudaGraphDestroy(g);
  if (e != cudaSuccess || rc != MPMB_OK || !h->graph_exec[par]) {
    cudaGetLastError();
    h->graph_exec[par] = nullptr;
    h->use_graph = false;
    h->cur = cur0; h->ord = ord0; h->mov = mov0; h->xstep = x0; h->stage = 0; h->launches = l0; h->script_left = left0;   // nothing has run
    h->rigid_pending = 0; h->rigid_sent = false;
    h->sticky_cuda = false;
    return MPMB_OK;
  }
  h->graph_launches = (int)(h->launches - l0);
  h->cur = cur0; h->ord = ord0; h->mov = mov0; h->xstep = x0; h->launches = l0; h->script_left = left0;   // the caller's launch accounts for them
  return MPMB_OK;
}

int mpmb_substep(MpmbHandle h, int32_t nsub) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_substep(h, nsub);
  const bool peers = peers_connected(h);
  if (h->cfg.world > 1 && !peers) return fail(h, MPMB_ERR_STATE, "z-slab run: connect the peers (mpmb_xchg_connect) or drive the stages and move the buffers yourself");
  if (h->cfg.world > 1 && h->rigid_on && !rigid_connected(h))
    return fail(h, MPMB_ERR_STATE, "z-slab run with rigid bodies: connect every rank's rigid mailbox (mpmb_rigid_connect) or drive the stages yourself");
  int s = 0, rc;
  if (nsub > 0 && h->rigid_on && h->motion_on && h->motion_scripted && h->script_left < nsub)
    return fail(h, MPMB_ERR_STATE, "the rigid script has %lld entries left, %d substeps asked", (long long)h->script_left, nsub);
  // the by-id colour arrays cover every id before any capture: allocating them inside one would end graph replay for good
  if (nsub > 0 && h->rigid_on && h->cap > 0 && (!h->p_states.get() || (int64_t)h->p_states.size() < rigid_ids(h)) &&
      (rc = rigid_reserve_ids(h, std::max<int64_t>(rigid_ids(h), h->cap))) != MPMB_OK)
    return rc;
  // the first substep after an upload takes the radix-sorted arrival lists (a different ordering launch): never in a graph
  if (h->fresh && nsub > 0) {
    if ((rc = substep_once(h, peers, nsub > 1)) != MPMB_OK) return rc;
    s = 1;
  }
  // pairs of intermediate substeps through the captured graph; the last substep (it stores apic_b) always runs directly.
  // Rigid scenes replay too when the device advances the bodies (their per-substep state lives in device memory).
  while (h->use_graph && (!h->rigid_on || h->motion_on) && !h->profiling && h->cap > 0 && h->stage == 0 && nsub - s >= 3) {
    const int par = h->cur;
    if (!h->graph_exec[par]) {
      if ((rc = graph_capture_pair(h, peers)) != MPMB_OK) return rc;
      if (!h->graph_exec[par]) break;
    }
    CUDA_TRY(h, cudaGraphLaunch(h->graph_exec[par], h->stream));
    h->launches += h->graph_launches;
    if (h->rigid_on && h->motion_on && h->motion_scripted) h->script_left -= 2;
    h->xstep += 2;   // cur / ord / mov flip twice: unchanged
    s += 2;
  }
  for (; s < nsub; s++)
    if ((rc = substep_once(h, peers, s + 1 < nsub)) != MPMB_OK) return rc;
  return MPMB_OK;
}

int mpmb_download_grid(MpmbHandle h, int32_t which, float *dense4) {
  CHECK_HANDLE(h);
  if (h->m2) return m2_download_grid(h, which, dense4);
  if (h->stage != 2) return fail(h, MPMB_ERR_STATE, "the grid exists between rasterize and resample");
  if (!dense4 || which < 0 || which > 1) return fail(h, MPMB_ERR_INVALID, "bad argument");
  size_t n = (size_t)h->P.nnode[0] * h->P.nnode[1] * h->P.nnode[2];
  DevBuf<float4> d;
  CUDA_TRY(h, d.alloc(n));
  View V = make_view(h);
  k_dense_grid<<<h->num_sms * 8, 256, 0, h->stream>>>(V, h->P, which, d.get());
  h->launches++;
  CUDA_TRY(h, cudaMemcpyAsync(dense4, d.get(), sizeof(float4) * n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return MPMB_OK;
}

// ------------------------------------------------------------------------------ debug (not part of mpmb.h)
// Only in builds with -DMPMB_DEBUG_EXPORTS (python -m taichi_mpm_b200.build --define MPMB_DEBUG_EXPORTS --out ...):
// the product library exports exactly what include/mpmb.h declares.
#if defined(MPMB_CHECKED) || defined(MPMB_VALIDATE)
extern "C" int mpmb_debug_check(MpmbHandle h, int *out8) {
  CHECK_HANDLE(h);
  cudaStreamSynchronize(h->stream);
  Counters c;
  if (cudaMemcpy(&c, h->cnt.get(), sizeof(c), cudaMemcpyDeviceToHost) != cudaSuccess) return MPMB_ERR_CUDA;
  for (int k = 0; k < 8; k++) out8[k] = c.chk[k];
  out8[4] = c.n_store; out8[5] = c.n_alive; out8[6] = c.n_movers; out8[7] = c.n_tiles;
  return MPMB_OK;
}
#endif
#ifdef MPMB_DEBUG_EXPORTS
// which: 0 run_begin 1 run_len 2 stay 3 arr_len 4 out_begin 5 total 6 arr_off   (dense, ntot ints)
extern "C" int mpmb_debug_dense(MpmbHandle h, int which, int *out) {
  CHECK_HANDLE(h);
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  View V = make_view(h);
  const int *src[] = {V.run_begin, V.run_len, V.stay_cnt, V.arr_len, V.out_begin, V.total, V.arr_off};
  CUDA_TRY(h, cudaMemcpy(out, src[which], sizeof(int) * h->ntot, cudaMemcpyDeviceToHost));
  return h->ntot;
}
// keys and signed masses of the first n rows of the current storage; counters
extern "C" int mpmb_debug_rows(MpmbHandle h, int n, uint32_t *keys, float *mass4, int *counters8) {
  CHECK_HANDLE(h);
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (keys) CUDA_TRY(h, cudaMemcpy(keys, h->keys[h->cur].get(), sizeof(uint32_t) * n, cudaMemcpyDeviceToHost));
  if (mass4) CUDA_TRY(h, cudaMemcpy(mass4, h->q[h->cur][0].get(), sizeof(float4) * n, cudaMemcpyDeviceToHost));
  if (counters8) CUDA_TRY(h, cudaMemcpy(counters8, h->cnt.get(), sizeof(Counters), cudaMemcpyDeviceToHost));
  return MPMB_OK;
}
#endif  // MPMB_DEBUG_EXPORTS
#ifdef MPMB_TILE_TRACE
// the per-CTA records of the last launch of kernel `which` (TRACE_P2G / TRACE_G2P) as 32-byte
// {t0, t1, sm, tiles, rows, -}; returns the launch's CTA count (records copied: at most cap)
extern "C" int mpmb_debug_tile_trace(MpmbHandle h, int which, void *out, int cap) {
  CHECK_HANDLE(h);
  if (which < 0 || which > 1) return fail(h, MPMB_ERR_INVALID, "which must be 0 (k_p2g) or 1 (k_g2p)");
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  const int ctas = which == TRACE_P2G ? h->grid_p2g : h->grid_g2p;
  const int n = std::min(std::min(ctas, cap), (int)TRACE_CTAS);
  CUDA_TRY(h, cudaMemcpyFromSymbol(out, g_trace, sizeof(CtaTrace) * n, sizeof(CtaTrace) * TRACE_CTAS * which));
  return ctas;
}
#endif  // MPMB_TILE_TRACE

// ------------------------------------------------------------------------------ profiling
int mpmb_set_profiling(MpmbHandle h, int32_t enabled) {
  CHECK_HANDLE(h);
  if (!enabled && h->profiling) prof_collect(h);
  h->profiling = enabled != 0;
  return MPMB_OK;
}

int mpmb_get_profile(MpmbHandle h, double ms[MPMB_N_STAGES], int64_t launches[MPMB_N_STAGES], int32_t reset) {
  CHECK_HANDLE(h);
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  prof_collect(h);
  for (int s = 0; s < MPMB_N_STAGES; s++) {
    if (ms) ms[s] = h->prof_ms[s];
    if (launches) launches[s] = h->prof_launches[s];
    if (reset) { h->prof_ms[s] = 0; h->prof_launches[s] = 0; }
  }
  return MPMB_OK;
}

int mpmb_get_counters(MpmbHandle h, int64_t *active_tiles, int64_t *alive, int64_t *kernel_launches) {
  CHECK_HANDLE(h);
  int rc = mpmb_synchronize(h);
  if (rc != MPMB_OK) return rc;
  if (h->m2) {   // 2-D: the node tiles of the grid kernel, the live particles of the last ordering
    Counters2 c2;
    CUDA_TRY(h, cudaMemcpy(&c2, h->m2->cnt.get(), sizeof(c2), cudaMemcpyDeviceToHost));
    const Params2 &P2 = h->m2->P;
    if (active_tiles) *active_tiles = (int64_t)((P2.nnode[0] + M2_TILE - 1) / M2_TILE) * ((P2.nnode[1] + M2_TILE - 1) / M2_TILE);
    if (alive) *alive = c2.n_alive;
    if (kernel_launches) *kernel_launches = h->launches;
    return MPMB_OK;
  }
  Counters c;
  CUDA_TRY(h, cudaMemcpy(&c, h->cnt.get(), sizeof(c), cudaMemcpyDeviceToHost));
  if (active_tiles) *active_tiles = c.n_tiles;
  if (alive) *alive = c.n_alive;
  if (kernel_launches) *kernel_launches = h->launches;
  return MPMB_OK;
}

// rows of the current storage, movers waiting for the next ordering (= holes of their old runs), ghost tiles
int mpmb_get_ordering_stats(MpmbHandle h, int64_t *rows, int64_t *movers, int64_t *ghost_tiles) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = mpmb_synchronize(h);
  if (rc != MPMB_OK) return rc;
  Counters c;
  CUDA_TRY(h, cudaMemcpy(&c, h->cnt.get(), sizeof(c), cudaMemcpyDeviceToHost));
  if (rows) *rows = c.n_store;
  if (movers) *movers = c.n_movers;
  if (ghost_tiles) *ghost_tiles = c.n_ghost;
  return MPMB_OK;
}

// ------------------------------------------------------------------------------ multi-GPU (z slabs)
static int64_t halo_cap_xy(MpmbEngine *h) {
  int64_t full = (int64_t)h->P.nt[0] * h->P.nt[1];
  return (h->cfg.halo_capacity > 0 && h->cfg.halo_capacity < full) ? h->cfg.halo_capacity : full;
}
static int64_t halo_idx_bytes(MpmbEngine *h) { return (halo_cap_xy(h) * 4 + 15) / 16 * 16; }

int64_t mpmb_halo_bytes(MpmbHandle h) {
  if (h && h->m2) return fail(h, MPMB_ERR_STATE, "%s is not available on a 2-D handle (dim = 2)", __func__);
  if (!h || h->cfg.world <= 1) return 0;
  return 16 + halo_idx_bytes(h) + halo_cap_xy(h) * ARENA * (int64_t)sizeof(float4);
}

int mpmb_halo_pack(MpmbHandle h, int32_t face, void *dev_buf) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1) return fail(h, MPMB_ERR_STATE, "halo exchange needs world > 1");
  if (h->stage != 2 && h->stage != 11) return fail(h, MPMB_ERR_STATE, "halo_pack must follow rasterize (or its boundary part)");
  if (!dev_buf || face < 0 || face > 1) return fail(h, MPMB_ERR_INVALID, "bad argument");
  prof_begin(h, 3);
  char *b = (char *)dev_buf;
  CUDA_TRY(h, cudaMemsetAsync(b, 0, 16, h->stream));
  View V = make_view(h);
  const int layer = (face == 0 ? h->P.tile_z0 : h->P.tile_z1 - 1) - h->P.tz_off;
  k_halo_pack<<<h->num_sms * 4, 128, 0, h->stream>>>(V, h->P, layer, (int)halo_cap_xy(h), (int *)b, (int *)(b + 16),
                                                     (float4 *)(b + 16 + halo_idx_bytes(h)));
  h->launches++;
  prof_end(h, 1);
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

int mpmb_halo_unpack(MpmbHandle h, int32_t face, const void *dev_buf) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1) return fail(h, MPMB_ERR_STATE, "halo exchange needs world > 1");
  if (h->stage != 2 && h->stage != 22) return fail(h, MPMB_ERR_STATE, "halo_unpack must follow rasterize (and may follow the interior resample)");
  if (!dev_buf || face < 0 || face > 1) return fail(h, MPMB_ERR_INVALID, "bad argument");
  const int glayer = face == 0 ? h->P.tile_z0 - 1 : h->P.tile_z1;  // the neighbour's boundary layer
  if (glayer < 0 || glayer >= h->nt2_global) return fail(h, MPMB_ERR_INVALID, "no neighbour through face %d", face);
  const int layer = glayer - h->P.tz_off;
  prof_begin(h, 3);
  const char *b = (const char *)dev_buf;
  View V = make_view(h);
  k_halo_unpack<<<h->num_sms * 4, 128, 0, h->stream>>>(V, h->P, layer, (int)halo_cap_xy(h), (const int *)b, (const int *)(b + 16),
                                                       (const float4 *)(b + 16 + halo_idx_bytes(h)));
  h->launches++;
  prof_end(h, 1);
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

int64_t mpmb_migrate_bytes(MpmbHandle h) {
  if (h && h->m2) return fail(h, MPMB_ERR_STATE, "%s is not available on a 2-D handle (dim = 2)", __func__);
  if (!h || h->cfg.world <= 1) return 0;
  return 16 + h->mig_cap * N_Q * (int64_t)sizeof(float4);
}

int mpmb_migrate_pack(MpmbHandle h, int32_t face, void *dev_buf) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1) return fail(h, MPMB_ERR_STATE, "migration needs world > 1");
  if (h->stage != 0) return fail(h, MPMB_ERR_STATE, "migrate_pack must follow resample");
  if (!dev_buf || face < 0 || face > 1) return fail(h, MPMB_ERR_INVALID, "bad argument");
  prof_begin(h, 3);
  char *b = (char *)dev_buf;
  CUDA_TRY(h, cudaMemsetAsync(b, 0, 16, h->stream));
  View V = make_view(h);
  const uint32_t key_face = h->special_min + (face == 0 ? SPECIAL_MIG_DOWN : SPECIAL_MIG_UP);
  k_migrate_pack<<<h->num_sms * 2, 256, 0, h->stream>>>(V, key_face, h->key_dead, (int)h->mig_cap, (int *)b, (float4 *)(b + 16), state_words(h));
  h->launches++;
  prof_end(h, 1);
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

int mpmb_migrate_unpack(MpmbHandle h, int32_t face, const void *dev_buf) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1) return fail(h, MPMB_ERR_STATE, "migration needs world > 1");
  if (h->stage != 0) return fail(h, MPMB_ERR_STATE, "migrate_unpack must follow resample");
  if (!dev_buf || face < 0 || face > 1) return fail(h, MPMB_ERR_INVALID, "bad argument");
  prof_begin(h, 3);
  const char *b = (const char *)dev_buf;
  View V = make_view(h);
  k_migrate_unpack<<<64, 256, 0, h->stream>>>(V, h->P, (int)h->mig_cap, (const int *)b, (const float4 *)(b + 16), state_words(h));
  k_migrate_commit<<<1, 1, 0, h->stream>>>(h->cnt.get(), (const int *)b, (int)h->mig_cap, (int)h->cap);
  h->launches += 2;
  prof_end(h, 2);
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}


// ------------------------------------------------------------------------------ peer-memory exchange
int mpmb_xchg_buffer(MpmbHandle h, int32_t kind, int32_t face, void **dev_ptr) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || kind < 0 || kind > 1 || face < 0 || face > 1 || !dev_ptr) return fail(h, MPMB_ERR_INVALID, "bad argument");
  *dev_ptr = h->rx[kind][face].get();
  return MPMB_OK;
}

int mpmb_xchg_ipc_handle(MpmbHandle h, int32_t kind, int32_t face, void *out64) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || kind < 0 || kind > 1 || face < 0 || face > 1 || !out64) return fail(h, MPMB_ERR_INVALID, "bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t hd;
  CUDA_TRY(h, cudaIpcGetMemHandle(&hd, h->rx[kind][face].get()));
  memcpy(out64, &hd, 64);
  return MPMB_OK;
}

// Through face f this rank writes into the neighbour's receive buffer of the OPPOSITE face.  Give
// either that buffer's IPC handle (another process) or its device pointer (same process).
int mpmb_xchg_connect(MpmbHandle h, int32_t kind, int32_t face, const void *handle64, void *same_process_ptr) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || kind < 0 || kind > 1 || face < 0 || face > 1) return fail(h, MPMB_ERR_INVALID, "bad argument");
  if (same_process_ptr) {
    h->tx[kind][face] = (char *)same_process_ptr;
    h->tx_ipc[kind][face] = false;
  } else {
    if (!handle64) return fail(h, MPMB_ERR_INVALID, "handle or pointer required");
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handle64, 64);
    void *p = nullptr;
    CUDA_TRY(h, cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
    h->tx[kind][face] = (char *)p;
    h->tx_ipc[kind][face] = true;
  }
  // a (re)connection restarts the sequence: my own receive headers of this kind must not hold an old, larger seq
  for (int f = 0; f < 2; f++)
    if (h->rx[kind][f].get()) CUDA_TRY(h, cudaMemset(h->rx[kind][f].get(), 0, 16));
  CUDA_TRY(h, cudaMemset(&h->cnt.get()->xstep, 0, sizeof(int)));
  CUDA_TRY(h, cudaMemset(h->rmail.get(), 0, h->rmail.size()));   // the rigid mailbox's seq words restart with the sequence too
  h->xstep = 0;
  graph_reset(h);
  return MPMB_OK;
}

static bool peers_connected(MpmbEngine *h) {
  if (h->cfg.world <= 1) return false;
  const bool lo = h->P.tile_z0 > 0 && h->cfg.rank > 0, hi = h->cfg.rank + 1 < h->cfg.world;
  for (int k = 0; k < 2; k++) {
    if (lo && !h->tx[k][0]) return false;
    if (hi && !h->tx[k][1]) return false;
  }
  return lo || hi;
}

// both faces of one message kind as the fused kernels take them
static void xfaces(MpmbEngine *h, int kind, XFace f[2], int *mask) {
  *mask = 0;
  for (int k = 0; k < 2; k++) {
    f[k].tx = h->tx[kind][k];
    f[k].rx = h->rx[kind][k].get();
    f[k].layer = 0;
    f[k].key = h->special_min + (k == 0 ? SPECIAL_MIG_DOWN : SPECIAL_MIG_UP);
    if (h->tx[kind][k]) *mask |= 1 << k;
  }
}

static int xchg_halo_launch(MpmbEngine *h, int mask_send, int mask_recv) {
  XFace s[2], r[2];
  int mask;
  xfaces(h, 0, s, &mask);
  xfaces(h, 0, r, &mask);
  s[0].layer = h->P.tile_z0 - h->P.tz_off;      s[1].layer = h->P.tile_z1 - 1 - h->P.tz_off;  // my boundary layers
  r[0].layer = h->P.tile_z0 - 1 - h->P.tz_off;  r[1].layer = h->P.tile_z1 - h->P.tz_off;      // the neighbours'
  prof_begin(h, 3);
  View V = make_view(h);
  int nl = 0;
  if (mask_send & mask) {
    k_halo_send2<<<h->num_sms * 4, 128, 0, h->stream>>>(V, h->P, (int)halo_cap_xy(h), (int)halo_idx_bytes(h), s[0], s[1], mask_send & mask, h->xcount.get(),
                                                         h->xcount.get() + 16);
    nl++;
  }
  if (mask_recv & mask) {
    k_halo_recv2<<<h->num_sms * 4, 128, 0, h->stream>>>(V, h->P, (int)halo_cap_xy(h), (int)halo_idx_bytes(h), r[0], r[1], mask_recv & mask);
    nl++;
  }
  h->launches += nl;
  prof_end(h, nl);
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

static int xchg_migrate_launch(MpmbEngine *h, int mask_send, int mask_recv) {
  XFace f[2];
  int mask;
  xfaces(h, 1, f, &mask);
  prof_begin(h, 3);
  View V = make_view(h);
  int nl = 0;
  if (mask_send & mask) {
    k_migrate_send2<<<h->num_sms * 2, 256, 0, h->stream>>>(V, h->key_dead, (int)h->mig_cap, f[0], f[1], mask_send & mask, h->xcount.get() + 8, h->xcount.get() + 20,
                                                          state_words(h));
    nl++;
  }
  if (mask_recv & mask) {
    k_migrate_recv2<<<1, 1024, 0, h->stream>>>(V, h->P, (int)h->mig_cap, f[0], f[1], mask_recv & mask, state_words(h));
    nl++;
  }
  h->launches += nl;
  prof_end(h, nl);
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

// what mpmb_substep runs on a z-slab rank: both faces per launch
static int xchg_halo_fused(MpmbEngine *h) {
  if (h->stage != 2) return fail(h, MPMB_ERR_STATE, "halo exchange must follow rasterize");
  return xchg_halo_launch(h, 3, 3);
}
static int xchg_migrate_fused(MpmbEngine *h) {
  if (h->stage != 0) return fail(h, MPMB_ERR_STATE, "migration must follow resample");
  return xchg_migrate_launch(h, 3, 3);
}

// the same steps one face at a time, for hosts that drive the stages themselves (same kernels, one-face masks)
int mpmb_halo_send(MpmbHandle h, int32_t face) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || face < 0 || face > 1 || !h->tx[0][face]) return fail(h, MPMB_ERR_STATE, "no connected peer through face %d", face);
  if (h->stage != 2) return fail(h, MPMB_ERR_STATE, "halo_send must follow rasterize");
  return xchg_halo_launch(h, 1 << face, 0);
}

int mpmb_halo_recv(MpmbHandle h, int32_t face) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || face < 0 || face > 1 || !h->tx[0][face]) return fail(h, MPMB_ERR_STATE, "no connected peer through face %d", face);
  if (h->stage != 2) return fail(h, MPMB_ERR_STATE, "halo_recv must follow rasterize");
  return xchg_halo_launch(h, 0, 1 << face);
}

int mpmb_migrate_send(MpmbHandle h, int32_t face) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || face < 0 || face > 1 || !h->tx[1][face]) return fail(h, MPMB_ERR_STATE, "no connected peer through face %d", face);
  if (h->stage != 0) return fail(h, MPMB_ERR_STATE, "migrate_send must follow resample");
  return xchg_migrate_launch(h, 1 << face, 0);
}

int mpmb_migrate_recv(MpmbHandle h, int32_t face) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || face < 0 || face > 1 || !h->tx[1][face]) return fail(h, MPMB_ERR_STATE, "no connected peer through face %d", face);
  if (h->stage != 0) return fail(h, MPMB_ERR_STATE, "migrate_recv must follow resample");
  return xchg_migrate_launch(h, 0, 1 << face);
}

// ------------------------------------------------------------------------------ rigid impulses of z-slab ranks
static int rigid_reduce_allowed(MpmbEngine *h, const char *what) {
  if (h->cfg.world <= 1 || !h->rigid_on) return fail(h, MPMB_ERR_STATE, "%s: z-slab ranks with rigid coupling only", what);
  if (!h->rigid_pending) return fail(h, MPMB_ERR_STATE, "%s follows a whole transfer (rasterize or resample, both parts)", what);
  return MPMB_OK;
}
// the sum is applied: after the G2P transfer the device-advanced bodies take their step (as mpmb_resample does on one engine)
static int rigid_reduced(MpmbEngine *h) {
  if (h->rigid_pending == 2 && h->motion_on) launch_rigid_motion(h);
  h->rigid_pending = 0;
  h->rigid_sent = false;
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}
static bool rigid_connected(MpmbEngine *h) {
  for (char *p : h->rmail_tx)
    if (!p) return false;
  return !h->rmail_tx.empty();
}
static void rigid_mail_send(MpmbEngine *h) {
  k_rigid_mail_send<<<1, 128, 0, h->stream>>>(rigid_view(h), h->rmail_dev.get(), h->cfg.world, h->cfg.rank, h->rigid_pending - 1, h->rigid_pending == 1 ? 1 : 0, h->cnt.get());
  h->launches++;
  h->rigid_sent = true;
}
static int rigid_mail_recv(MpmbEngine *h) {
  k_rigid_mail_recv<<<1, 128, 0, h->stream>>>(rigid_view(h), h->rmail.get(), h->cfg.world, h->rigid_pending - 1, h->rigid_pending == 1 ? 1 : 0, h->cnt.get());
  h->launches++;
  return rigid_reduced(h);
}

int64_t mpmb_rigid_impulse_bytes(MpmbHandle h) {
  if (h && h->m2) return fail(h, MPMB_ERR_STATE, "%s is not available on a 2-D handle (dim = 2)", __func__);
  if (!h || h->cfg.world <= 1) return 0;
  return (int64_t)sizeof(float) * RIGID_IMPULSE_FLOATS;
}

int mpmb_rigid_impulse_pack(MpmbHandle h, void *dev_buf) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = rigid_reduce_allowed(h, "rigid_impulse_pack");
  if (rc != MPMB_OK) return rc;
  if (!dev_buf) return fail(h, MPMB_ERR_INVALID, "null buffer");
  k_rigid_impulse_pack<<<1, 128, 0, h->stream>>>(rigid_view(h), (float *)dev_buf);
  h->launches++;
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

int mpmb_rigid_impulse_apply(MpmbHandle h, const void *dev_all) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = rigid_reduce_allowed(h, "rigid_impulse_apply");
  if (rc != MPMB_OK) return rc;
  if (!dev_all) return fail(h, MPMB_ERR_INVALID, "null buffer");
  k_rigid_impulse_apply<<<1, 32, 0, h->stream>>>(rigid_view(h), (const float *)dev_all, h->cfg.world);
  h->launches++;
  return rigid_reduced(h);
}

int mpmb_rigid_mailbox(MpmbHandle h, void **dev_ptr) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || !dev_ptr) return fail(h, MPMB_ERR_INVALID, "bad argument");
  *dev_ptr = h->rmail.get();
  return MPMB_OK;
}

int mpmb_rigid_mailbox_ipc_handle(MpmbHandle h, void *out64) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || !out64) return fail(h, MPMB_ERR_INVALID, "bad argument");
  cudaIpcMemHandle_t hd;
  CUDA_TRY(h, cudaIpcGetMemHandle(&hd, h->rmail.get()));
  memcpy(out64, &hd, 64);
  return MPMB_OK;
}

int mpmb_rigid_connect(MpmbHandle h, int32_t rank, const void *handle64, void *same_process_ptr) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  if (h->cfg.world <= 1 || rank < 0 || rank >= h->cfg.world || rank == h->cfg.rank) return fail(h, MPMB_ERR_INVALID, "bad rank %d", rank);
  if (h->rigid_pending) return fail(h, MPMB_ERR_STATE, "rigid mailboxes connect between substeps");
  if (h->rmail_ipc[rank] && h->rmail_tx[rank]) cudaIpcCloseMemHandle(h->rmail_tx[rank]);
  h->rmail_tx[rank] = nullptr;
  h->rmail_ipc[rank] = false;
  if (same_process_ptr) {
    h->rmail_tx[rank] = (char *)same_process_ptr;
  } else {
    if (!handle64) return fail(h, MPMB_ERR_INVALID, "handle or pointer required");
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handle64, 64);
    void *p = nullptr;
    CUDA_TRY(h, cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
    h->rmail_tx[rank] = (char *)p;
    h->rmail_ipc[rank] = true;
  }
  CUDA_TRY(h, cudaMemcpy(h->rmail_dev.get(), h->rmail_tx.data(), sizeof(char *) * h->cfg.world, cudaMemcpyHostToDevice));
  graph_reset(h);
  return MPMB_OK;
}

int mpmb_rigid_send(MpmbHandle h) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = rigid_reduce_allowed(h, "rigid_send");
  if (rc != MPMB_OK) return rc;
  if (!rigid_connected(h)) return fail(h, MPMB_ERR_STATE, "rigid_send: connect every rank's mailbox first (mpmb_rigid_connect)");
  if (h->rigid_sent) return fail(h, MPMB_ERR_STATE, "rigid_send: this transfer's impulses were sent already");
  rigid_mail_send(h);
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

int mpmb_rigid_recv(MpmbHandle h) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = rigid_reduce_allowed(h, "rigid_recv");
  if (rc != MPMB_OK) return rc;
  if (!h->rigid_sent) return fail(h, MPMB_ERR_STATE, "rigid_recv follows rigid_send");
  return rigid_mail_recv(h);
}

// ------------------------------------------------------------------------------ re-cut of the z slabs
static int recut_allowed(MpmbEngine *h, const char *what) {
  if (h->cfg.world <= 1) return fail(h, MPMB_ERR_STATE, "%s re-cuts z-slab runs (world > 1)", what);
  if (h->stage != 0 || h->rigid_pending) return fail(h, MPMB_ERR_STATE, "%s runs between substeps, not inside one", what);
  return MPMB_OK;
}

// the scratch of the re-cut kernels: the layer histogram, then {bad arrivals, largest id}
static int recut_reserve(MpmbEngine *h) {
  CUDA_TRY(h, h->recut_buf.reserve(h->nt2_global + 1));   // allocated once: nt2_global does not change
  return MPMB_OK;
}
static int *recut_ints(MpmbEngine *h) { return (int *)(h->recut_buf.get() + h->nt2_global); }

// live rows per global tile layer into counts[nt2_global] (synchronises; nt2_global counters cross the bus)
static int layer_hist(MpmbEngine *h, int64_t *counts) {
  int rc = recut_reserve(h);
  if (rc != MPMB_OK) return rc;
  const int nl = h->nt2_global;
  CUDA_TRY(h, cudaMemsetAsync(h->recut_buf.get(), 0, sizeof(unsigned long long) * nl, h->stream));
  if (h->cap > 0) {
    k_layer_hist<<<h->num_sms * 4, 256, 0, h->stream>>>(h->keys[h->cur].get(), h->q[h->cur][0].get(), h->special_min, h->P.inv_dx, nl, h->cnt.get(), h->recut_buf.get());
    h->launches++;
  }
  static_assert(sizeof(int64_t) == sizeof(unsigned long long), "64-bit counters");
  CUDA_TRY(h, cudaMemcpyAsync(counts, h->recut_buf.get(), sizeof(int64_t) * nl, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

int mpmb_layer_counts(MpmbHandle h, int32_t n_layers, int64_t *counts) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = recut_allowed(h, "layer_counts");
  if (rc != MPMB_OK) return rc;
  if (!counts) return fail(h, MPMB_ERR_INVALID, "null argument");
  if (n_layers != h->nt2_global) return fail(h, MPMB_ERR_INVALID, "n_layers %d: the domain has %d tile layers", n_layers, h->nt2_global);
  return layer_hist(h, counts);
}

int mpmb_recut_pack(MpmbHandle h, const int32_t *cuts, void *dev_buf, int64_t cap_rows, int64_t *counts) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = recut_allowed(h, "recut_pack");
  if (rc != MPMB_OK) return rc;
  const int world = h->cfg.world, nl = h->nt2_global;
  if (!cuts || !counts || cap_rows < 0) return fail(h, MPMB_ERR_INVALID, "bad argument");
  if (cuts[0] != 0 || cuts[world] != nl) return fail(h, MPMB_ERR_INVALID, "cuts must run from 0 to %d tile layers", nl);
  for (int r = 0; r < world; r++)
    if (cuts[r + 1] <= cuts[r]) return fail(h, MPMB_ERR_INVALID, "cuts must increase strictly (rank %d: [%d, %d))", r, cuts[r], cuts[r + 1]);
  std::vector<int64_t> hist(nl);
  if ((rc = layer_hist(h, hist.data())) != MPMB_OK) return rc;
  int64_t total = 0;
  for (int d = 0; d < world; d++) {
    counts[d] = 0;
    if (d != h->cfg.rank)
      for (int l = cuts[d]; l < cuts[d + 1]; l++) counts[d] += hist[l];
    total += counts[d];
  }
  if (!dev_buf || total == 0) return MPMB_OK;
  if (total > cap_rows) return fail(h, MPMB_ERR_CAPACITY, "%lld departing rows do not fit in the %lld records provided", (long long)total, (long long)cap_rows);
  int ns = 0;
  if ((rc = read_n_store(h, &ns)) != MPMB_OK) return rc;
  if ((rc = scan_reserve(h, (size_t)ns)) != MPMB_OK) return rc;
  View V = make_view(h);
  int64_t off = 0;
  for (int d = 0; d < world; d++) {   // grouped by destination in ascending rank order, storage order within a destination
    if (counts[d] == 0) continue;
    k_layer_flags<<<(ns + 255) / 256, 256, 0, h->stream>>>(h->keys[h->cur].get(), h->q[h->cur][0].get(), ns, h->special_min, h->P.inv_dx, cuts[d], cuts[d + 1], h->scan_a.get());
    int got = 0;
    if ((rc = scan_flags(h, (size_t)ns, &got)) != MPMB_OK) return rc;
    if (got != counts[d]) return fail(h, MPMB_ERR_STATE, "rank %d: %d rows flagged, %lld counted", d, got, (long long)counts[d]);
    k_recut_pack<<<(ns + 127) / 128, 128, 0, h->stream>>>(V, ns, h->scan_b.get(), (float4 *)dev_buf + (size_t)off * N_Q, state_words(h));
    h->launches += 2;
    off += counts[d];
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

int mpmb_recut_apply(MpmbHandle h, int32_t tile_z0, int32_t tile_z1, int64_t n_in, const void *dev_records) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = recut_allowed(h, "recut_apply");
  if (rc != MPMB_OK) return rc;
  if (tile_z0 < 0 || tile_z1 > h->nt2_global || tile_z0 >= tile_z1)
    return fail(h, MPMB_ERR_INVALID, "bad slab [%d,%d) for %d tile layers", tile_z0, tile_z1, h->nt2_global);
  if (n_in < 0 || (n_in > 0 && !dev_records)) return fail(h, MPMB_ERR_INVALID, "n_in >= 0 records are required");
  if (n_in >= (1ll << 30)) return fail(h, MPMB_ERR_CAPACITY, "%lld arriving records exceed 2^30 particle rows per GPU", (long long)n_in);
  Slicing sl;
  if (!slab_slicing(h->P, h->nt2_global, h->cfg.world, tile_z0, tile_z1, &sl)) return fail(h, MPMB_ERR_INVALID, "tile grid too large for 32-bit keys");
  Params Pn = h->P;
  Pn.tz_off = sl.tz_off; Pn.nt[2] = sl.nt2; Pn.tile_z0 = sl.tile_z0; Pn.tile_z1 = sl.tile_z1; Pn.ntiles_total = sl.ntot;
  if ((rc = recut_reserve(h)) != MPMB_OK) return rc;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  int ns = 0, kept = 0;
  if (h->cap > 0 && (rc = read_n_store(h, &ns)) != MPMB_OK) return rc;
  // checks first: what stays, whether every arrival belongs here, whether a configured capacity holds both
  if (ns > 0) {
    if ((rc = scan_reserve(h, (size_t)ns)) != MPMB_OK) return rc;
    k_layer_flags<<<(ns + 255) / 256, 256, 0, h->stream>>>(h->keys[h->cur].get(), h->q[h->cur][0].get(), ns, h->special_min, h->P.inv_dx, tile_z0, tile_z1, h->scan_a.get());
    h->launches++;
    if ((rc = scan_flags(h, (size_t)ns, &kept)) != MPMB_OK) return rc;
  }
  int *ints = recut_ints(h);   // {bad arrivals, largest id held}
  CUDA_TRY(h, cudaMemsetAsync(ints, 0, sizeof(int), h->stream));
  CUDA_TRY(h, cudaMemsetAsync(ints + 1, 0xFF, sizeof(int), h->stream));
  if (n_in > 0) {
    k_recut_check<<<std::min<int64_t>((n_in + 255) / 256, h->num_sms * 8), 256, 0, h->stream>>>(Pn, (int)n_in, (const float4 *)dev_records, ints, ints + 1);
    h->launches++;
    int bad = 0;
    CUDA_TRY(h, cudaMemcpyAsync(&bad, ints, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    CUDA_TRY(h, cudaGetLastError());
    if (bad) return fail(h, MPMB_ERR_INVALID, "%d of %lld arriving records lie outside tile layers [%d, %d)", bad, (long long)n_in, tile_z0, tile_z1);
  }
  const int64_t need = (int64_t)kept + n_in;
  if (need >= (1ll << 30)) return fail(h, MPMB_ERR_CAPACITY, "%lld particle rows exceed 2^30 per GPU", (long long)need);
  if (h->cfg.capacity > 0 && need > h->cap)
    return fail(h, MPMB_ERR_CAPACITY, "%lld particle rows exceed the configured capacity %lld", (long long)need, (long long)h->cap);
  // the engine changes from here on: a thicker slab grows the tile arrays, the rows grow if they must
  if (sl.ntot > h->cap_tiles && (rc = alloc_tile_arrays(h, sl.ntot)) != MPMB_OK) return rc;
  if (h->rigid_on && h->tile_flag.size() < (size_t)h->cap_tiles) CUDA_TRY(h, h->tile_flag.alloc(h->cap_tiles));   // rewritten by every ordering
  if (need > 0 && (rc = grow_keeping_rows(h, need, ns)) != MPMB_OK) return rc;
  set_slicing(h, sl);
  h->cfg.tile_z0 = tile_z0;
  h->cfg.tile_z1 = tile_z1;
  if (h->cap > 0) {
    if (kept > 0) {   // the staying rows, compacted in storage order into the other buffer, re-keyed; departing rows are left behind
      k_recut_keep<<<std::min((ns + 255) / 256, h->num_sms * 8), 256, 0, h->stream>>>(make_view(h), h->P, ns, h->scan_b.get(), ints + 1);
      h->launches++;
    }
    h->cur ^= 1;
    if (n_in > 0) {
      k_recut_unpack<<<(unsigned)((n_in + 127) / 128), 128, 0, h->stream>>>(make_view(h), h->P, (int)n_in, kept, (const float4 *)dev_records, state_words(h));
      h->launches++;
    }
  }
  int max_id = -1;
  CUDA_TRY(h, cudaMemcpyAsync(&max_id, ints + 1, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  h->id_end = std::max<int64_t>(h->id_end, (int64_t)max_id + 1);
  h->aos_host_pool = nullptr;
  graph_reset(h);
  return reorder_from_scratch(h, need);
}

}  // extern "C"

// =====================================================================================
// AsyncMPM pools (mpmb_async_*, SURVEY §8f row 3): the particle records live on the device; the block scheduler's state and
// decisions too with mpmb_async_schedule / mpmb_async_advance_level, the step loop on the host
// =====================================================================================
static int async_check(MpmbEngine *h, bool need_init) {
  if (need_init && !h->async_on) return fail(h, MPMB_ERR_STATE, "mpmb_async_init has not been called");
  if (h->cfg.world > 1) return fail(h, MPMB_ERR_STATE, "AsyncMPM pools are implemented for single-GPU engines (world == 1)");
  if (h->rigid_on) return fail(h, MPMB_ERR_STATE, "AsyncMPM pools do not support rigid bodies");
  if (h->stage != 0) return fail(h, MPMB_ERR_STATE, "AsyncMPM pools are edited between substeps, not inside one");
  return MPMB_OK;
}

// room for `need` records in both buffers of a pool, keeping the current records (grows by at least half, as
// grow_keeping_rows does for the resident set)
static int apool_reserve(MpmbEngine *h, MpmbEngine::APool &p, int64_t need) {
  const int64_t cap = arec_cap(p.buf[0]);
  if (need <= cap) return MPMB_OK;
  const int64_t want = std::max<int64_t>(need, cap + cap / 2);
  DevBuf<float> nb[2];
  for (auto &b : nb) CUDA_TRY(h, b.alloc((size_t)AREC_WORDS * want));
  const ARec n0 = arec_of(nb[0]), o = p.rec(p.cur);
  const size_t n = (size_t)p.n;
  if (n > 0) {
    const struct { void *d; const void *s; size_t w; } cp[] = {{n0.x, o.x, 3}, {n0.v, o.v, 3}, {n0.F, o.F, 9}, {n0.b, o.b, 9}, {n0.mass, o.mass, 1},
                                                              {n0.vol, o.vol, 1}, {n0.scalar, o.scalar, 1}, {n0.group, o.group, 1}, {n0.id, o.id, 1},
                                                              {n0.block, o.block, 1}};
    for (const auto &c : cp) CUDA_TRY(h, cudaMemcpyAsync(c.d, c.s, 4 * c.w * n, cudaMemcpyDeviceToDevice, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  for (int b = 0; b < 2; b++) p.buf[b] = std::move(nb[b]);
  p.cur = 0;
  return MPMB_OK;
}

static unsigned nblocks(int64_t n) { return (unsigned)((n + 255) / 256); }

// pool <- pool[records of blocks without `bit`]; with `to` the others are appended to that pool, in order.  Stable.
static int apool_split(MpmbEngine *h, MpmbEngine::APool &p, int bit, MpmbEngine::APool *to) {
  const int n = (int)p.n;
  if (n == 0) return MPMB_OK;
  int rc, moved = 0;
  if ((rc = scan_reserve(h, (size_t)n)) != MPMB_OK) return rc;
  k_async_rec_flags<<<nblocks(n), 256, 0, h->stream>>>(p.rec(p.cur).block, n, h->a_bfl.get(), bit, h->scan_a.get());
  h->launches++;
  if ((rc = scan_flags(h, (size_t)n, &moved)) != MPMB_OK) return rc;
  if (moved == 0) return MPMB_OK;
  if (to && (rc = apool_reserve(h, *to, to->n + moved)) != MPMB_OK) return rc;
  k_async_split<<<nblocks(n), 256, 0, h->stream>>>(p.rec(p.cur), n, h->scan_a.get(), h->scan_b.get(), to ? to->rec(to->cur) : ARec{}, to ? (int)to->n : 0,
                                                    to ? 1 : 0, p.rec(p.cur ^ 1), 0, 1);
  h->launches++;
  CUDA_TRY(h, cudaGetLastError());
  p.cur ^= 1;
  p.n = n - moved;
  if (to) to->n += moved;
  return MPMB_OK;
}

extern "C" {

int mpmb_async_init(MpmbHandle h, const int32_t nb[3], float inv_dx) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = async_check(h, false);
  if (rc != MPMB_OK) return rc;
  if (!nb) return fail(h, MPMB_ERR_INVALID, "null argument");
  for (int d = 0; d < 3; d++)
    if (nb[d] < 1 || nb[d] > 4096) return fail(h, MPMB_ERR_INVALID, "nb[%d] = %d outside [1, 4096]", d, nb[d]);
  if (!(inv_dx > 0.f) || !std::isfinite(inv_dx)) return fail(h, MPMB_ERR_INVALID, "inv_dx must be positive and finite");
  const int64_t nblk = (int64_t)nb[0] * nb[1] * nb[2];
  if (nblk >= (1ll << 30)) return fail(h, MPMB_ERR_INVALID, "too many scheduler blocks");
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  // empty pools and no gather scratch: every capacity starts again from nothing
  for (auto &p : h->apool) p = MpmbEngine::APool{};
  h->a_gbuf.reset(); h->a_sbuf.reset(); h->a_rowk.reset(); h->a_cub.reset();
  for (auto &k : h->a_key) k.reset();
  for (auto &u : h->a_u) u.reset();
  h->async_on = false;
  for (int d = 0; d < 3; d++) h->anb[d] = nb[d];
  h->nblk = (int)nblk;
  h->a_inv_dx = inv_dx;
  CUDA_TRY(h, h->a_bfl.alloc(nblk));
  CUDA_TRY(h, h->a_bflag.alloc(nblk));
  CUDA_TRY(h, h->a_bmin.alloc(nblk));
  CUDA_TRY(h, h->a_bmax.alloc(nblk));
  CUDA_TRY(h, h->a_blk.alloc(nblk));
  CUDA_TRY(h, h->a_lim.alloc(2 * nblk));
  CUDA_TRY(h, h->a_bad.alloc(1));
  CUDA_TRY(h, h->a_level.alloc(nblk));
  CUDA_TRY(h, h->a_lvnew.alloc(nblk));
  CUDA_TRY(h, h->a_local_min.alloc(nblk));
  CUDA_TRY(h, h->a_particle_t.alloc(nblk));
  CUDA_TRY(h, h->a_backup_t.alloc(nblk));
  CUDA_TRY(h, h->a_sched.alloc(1));
  k_async_state_init<<<nblocks(nblk), 256, 0, h->stream>>>((int)nblk, h->a_level.get(), h->a_local_min.get(), h->a_particle_t.get(), h->a_backup_t.get());
  h->launches++;
  CUDA_TRY(h, cudaGetLastError());
  for (auto &p : h->apool)
    if ((rc = apool_reserve(h, p, 1024)) != MPMB_OK) return rc;
  h->async_on = true;
  return MPMB_OK;
}

int mpmb_async_add(MpmbHandle h, int32_t which, int64_t n, const float *x, const float *v, const float *F, const float *b, const float *mass,
                   const float *vol, const float *scalar, const int32_t *group, const uint32_t *id) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = async_check(h, true);
  if (rc != MPMB_OK) return rc;
  if (which < 0 || which > 1) return fail(h, MPMB_ERR_INVALID, "which = %d: 0 (particle pool) or 1 (backup pool)", which);
  if (n < 0 || (n > 0 && (!x || !v || !F || !b || !mass || !vol || !scalar || !group || !id))) return fail(h, MPMB_ERR_INVALID, "every field is required");
  if (n == 0) return MPMB_OK;
  MpmbEngine::APool &p = h->apool[which];
  if (p.n + n >= (1ll << 30)) return fail(h, MPMB_ERR_CAPACITY, "an AsyncMPM pool holds fewer than 2^30 records");
  if ((rc = apool_reserve(h, p, p.n + n)) != MPMB_OK) return rc;
  const ARec r = p.rec(p.cur);
  const size_t o = (size_t)p.n;
  const struct { void *d; const void *s; size_t w; } cp[] = {{r.x + 3 * o, x, 3}, {r.v + 3 * o, v, 3}, {r.F + 9 * o, F, 9}, {r.b + 9 * o, b, 9},
                                                            {r.mass + o, mass, 1}, {r.vol + o, vol, 1}, {r.scalar + o, scalar, 1}, {r.group + o, group, 1},
                                                            {r.id + o, id, 1}};
  for (const auto &c : cp) CUDA_TRY(h, cudaMemcpyAsync(c.d, c.s, 4 * c.w * (size_t)n, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->a_bad.get(), 0, sizeof(int), h->stream));
  k_async_blocks<<<nblocks(n), 256, 0, h->stream>>>(r.x + 3 * o, (int)n, h->a_inv_dx, h->anb[0], h->anb[1], h->anb[2], r.block + o, h->a_bad.get());
  h->launches++;
  int bad = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&bad, h->a_bad.get(), sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  if (bad) return fail(h, MPMB_ERR_INVALID, "%d records lie outside the %d x %d x %d scheduler blocks", bad, h->anb[0], h->anb[1], h->anb[2]);
  p.n += n;
  return MPMB_OK;
}

int mpmb_async_block_limits(MpmbHandle h, int32_t with_limits, int64_t cap, int64_t *n_blocks, int32_t *block, float *min_dt, float *max_v2) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = async_check(h, true);
  if (rc != MPMB_OK) return rc;
  if (!n_blocks || (cap > 0 && !block) || (with_limits && cap > 0 && (!min_dt || !max_v2))) return fail(h, MPMB_ERR_INVALID, "null argument");
  *n_blocks = 0;
  const int nblk = h->nblk;
  const MpmbEngine::APool &p = h->apool[0];
  CUDA_TRY(h, cudaMemsetAsync(h->a_bflag.get(), 0, sizeof(uint32_t) * nblk, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->a_bad.get(), 0, sizeof(int), h->stream));
  if (with_limits) {
    k_fill_u32<<<nblocks(nblk), 256, 0, h->stream>>>((uint32_t *)h->a_bmin.get(), nblk, 0x3dcccccdu);   // 0.1f
    k_fill_u32<<<nblocks(nblk), 256, 0, h->stream>>>((uint32_t *)h->a_bmax.get(), nblk, 0x2539705fu);   // 1e-16f
    h->launches += 2;
  }
  if (p.n > 0) {
    k_async_limits<<<nblocks(p.n), 256, 0, h->stream>>>(p.rec(p.cur), (int)p.n, h->P, with_limits ? 1 : 0, h->a_bflag.get(), h->a_bmin.get(), h->a_bmax.get(), h->a_bad.get());
    h->launches++;
  }
  int bad = 0, total = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&bad, h->a_bad.get(), sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if ((rc = scan_reserve(h, (size_t)nblk)) != MPMB_OK) return rc;
  k_async_occupied<<<nblocks(nblk), 256, 0, h->stream>>>(h->a_bflag.get(), nblk, h->scan_a.get());
  h->launches++;
  if ((rc = scan_flags(h, (size_t)nblk, &total)) != MPMB_OK) return rc;
  if (bad) return fail(h, MPMB_ERR_INVALID, "%d pool particles are of a type without a time-step limit (linear / jelly)", bad);
  *n_blocks = total;
  if (total > cap) return fail(h, MPMB_ERR_CAPACITY, "%d occupied blocks do not fit in the %lld entries provided", total, (long long)cap);
  if (total == 0) return MPMB_OK;
  float *dmin = h->a_lim.get(), *dmax = h->a_lim.get() + nblk;
  k_async_block_out<<<nblocks(nblk), 256, 0, h->stream>>>(h->a_bflag.get(), h->a_bmin.get(), h->a_bmax.get(), nblk, h->scan_b.get(), h->a_blk.get(), dmin, dmax);
  h->launches++;
  CUDA_TRY(h, cudaMemcpyAsync(block, h->a_blk.get(), sizeof(int) * total, cudaMemcpyDeviceToHost, h->stream));
  if (with_limits) {
    CUDA_TRY(h, cudaMemcpyAsync(min_dt, dmin, sizeof(float) * total, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(max_v2, dmax, sizeof(float) * total, cudaMemcpyDeviceToHost, h->stream));
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

}  // extern "C"

// The pool work of one advance on the block flags in a_bfl (mpmb_async_advance: steps 1-5).  sc holds the MPMB_ASYNC_SWAP /
// MPMB_ASYNC_CLEAR bits present in some block, or is -1: flags built on the device, whose bits a_sched->sc holds; they are
// read with the candidate count (no candidates: both pools are empty and their edits do nothing).
static int async_advance_body(MpmbEngine *h, float dt, int sc, int64_t *n_gathered) {
  int rc;
  *n_gathered = 0;
  MpmbEngine::APool &P0 = h->apool[0], &B0 = h->apool[1];

  // 1. gather: flagged candidates -> sort by (part, page index) -> first copy of every id -> the set, in that order
  const int np = (int)P0.n, nbk = (int)B0.n;
  const int64_t nc_all = 2 * (int64_t)np + nbk;
  int nc = 0, ng = 0;
  ARec G{}, S{};   // the gathered set and its survivors
  if (nc_all > 0) {
    if ((rc = scan_reserve(h, (size_t)nc_all + (sc < 0 ? 1 : 0))) != MPMB_OK) return rc;
    k_async_cand_flags<<<nblocks(nc_all), 256, 0, h->stream>>>(P0.rec(P0.cur).block, np, B0.rec(B0.cur).block, nbk, h->a_bfl.get(), h->scan_a.get());
    h->launches++;
    if ((rc = scan_flags(h, (size_t)nc_all, &nc, sc < 0 ? &h->a_sched.get()->sc : nullptr, &sc)) != MPMB_OK) return rc;
  }
  const bool any_swap = sc > 0 && (sc & MPMB_ASYNC_SWAP), any_clear = sc > 0 && (sc & MPMB_ASYNC_CLEAR);
  if (nc > 0) {
    const int64_t ccap = (int64_t)h->a_rowk.size();   // the candidate capacity
    if (nc > ccap) {
      const int64_t want = std::max<int64_t>(nc, ccap + ccap / 2);
      for (auto &k : h->a_key) k.reset();   // the old candidate scratch goes before the new comes
      for (auto &u : h->a_u) u.reset();
      h->a_rowk.reset(); h->a_cub.reset();
      for (auto &k : h->a_key) CUDA_TRY(h, k.alloc(want));
      for (auto &u : h->a_u) CUDA_TRY(h, u.alloc(want));
      CUDA_TRY(h, h->a_rowk.alloc(want));
      size_t b1 = 0, b2 = 0;
      cub::DeviceRadixSort::SortPairs(nullptr, b1, h->a_key[0].get(), h->a_key[1].get(), h->a_u[0].get(), h->a_u[1].get(), (int)want, 0, 38, h->stream);
      cub::DeviceRadixSort::SortPairs(nullptr, b2, h->a_u[2].get(), h->a_u[3].get(), h->a_u[0].get(), h->a_u[0].get(), (int)want, 0, 32, h->stream);
      CUDA_TRY(h, h->a_cub.alloc(std::max(b1, b2)));
    }
    // keys and candidate indices; once sorted, the unsorted candidate list holds the positions sorted by id, and a_rowk
    // (rewritten by the routing) the unsorted positions
    unsigned long long *key = h->a_key[0].get(), *key_s = h->a_key[1].get();
    uint32_t *cand = h->a_u[0].get(), *cand_s = h->a_u[1].get(), *ids = h->a_u[2].get(), *ids_s = h->a_u[3].get();
    uint32_t *pos = (uint32_t *)h->a_rowk.get(), *pos_s = h->a_u[0].get();
    k_async_cand_keys<<<nblocks(nc_all), 256, 0, h->stream>>>(P0.rec(P0.cur).block, np, B0.rec(B0.cur).block, nbk, h->scan_a.get(), h->scan_b.get(), h->anb[1], h->anb[2], key, cand);
    size_t bytes = h->a_cub.size();
    cub::DeviceRadixSort::SortPairs(h->a_cub.get(), bytes, key, key_s, cand, cand_s, nc, 0, 38, h->stream);
    k_async_cand_ids<<<nblocks(nc), 256, 0, h->stream>>>(cand_s, nc, P0.rec(P0.cur).id, np, B0.rec(B0.cur).id, ids, pos);
    bytes = h->a_cub.size();
    cub::DeviceRadixSort::SortPairs(h->a_cub.get(), bytes, ids, ids_s, pos, pos_s, nc, 0, 32, h->stream);
    k_async_first<<<nblocks(nc), 256, 0, h->stream>>>(ids_s, pos_s, nc, h->scan_a.get());
    h->launches += 5;
    if ((rc = scan_flags(h, (size_t)nc, &ng)) != MPMB_OK) return rc;
    if (ng > arec_cap(h->a_gbuf)) CUDA_TRY(h, h->a_gbuf.alloc((size_t)AREC_WORDS * std::max<int64_t>(ng, 3 * (int64_t)ng / 2)));
    G = arec_of(h->a_gbuf);
    k_async_gather<<<nblocks(nc), 256, 0, h->stream>>>(cand_s, nc, h->scan_a.get(), h->scan_b.get(), P0.rec(P0.cur), np, B0.rec(B0.cur), G);
    h->launches++;
    CUDA_TRY(h, cudaGetLastError());
  }
  // the engine must hold the set: a configured capacity that is too small changes nothing
  if (ng > 0 && (rc = ensure_capacity(h, ng)) != MPMB_OK) return rc;

  // 2. the level's pools become their blocks' backups
  if (any_swap) {
    if ((rc = apool_split(h, B0, MPMB_ASYNC_SWAP, nullptr)) != MPMB_OK) return rc;
    if ((rc = apool_split(h, P0, MPMB_ASYNC_SWAP, &B0)) != MPMB_OK) return rc;
  }

  // 3. one ordinary substep on the set; survivors (storage order) with their new blocks
  int64_t alive = 0;
  if (ng > 0) {
    apply_delta_t(h, dt);
    h->aos_host_pool = nullptr;
    if ((rc = pack_rows(h, ng, G.x, G.v, G.F, G.b, G.mass, G.vol, G.scalar, G.group, 0, 0)) != MPMB_OK) return rc;
    if ((rc = finish_upload(h, ng)) != MPMB_OK) return rc;
    if ((rc = mpmb_substep(h, 1)) != MPMB_OK) return rc;
    if ((rc = mpmb_synchronize(h)) != MPMB_OK) return rc;
    int ns = 0;
    if ((rc = read_n_store(h, &ns)) != MPMB_OK) return rc;
    if (ns > 0 && (rc = live_prefix(h, ns, &alive)) != MPMB_OK) return rc;
    if (alive > arec_cap(h->a_sbuf)) CUDA_TRY(h, h->a_sbuf.alloc((size_t)AREC_WORDS * std::max<int64_t>(alive, arec_cap(h->a_gbuf))));
    S = arec_of(h->a_sbuf);
    if (alive > 0) {
      unpack_live(h, ns, S.id, S.x, S.v, S.F, S.b, S.mass, S.vol, S.scalar, S.group);
      k_async_blocks<<<nblocks(alive), 256, 0, h->stream>>>(S.x, (int)alive, h->a_inv_dx, h->anb[0], h->anb[1], h->anb[2], S.block, h->a_bad.get());
      h->launches++;
    }
  }

  // 4. blocks whose backups were consumed drop them
  if (any_clear && (rc = apool_split(h, B0, MPMB_ASYNC_CLEAR, nullptr)) != MPMB_OK) return rc;

  // 5. survivors, in gather order, to the pool of their new block (EQUAL) or to the backup (CLEAR, not EQUAL)
  if (alive > 0) {
    k_fill_u32<<<nblocks(ng), 256, 0, h->stream>>>((uint32_t *)h->a_rowk.get(), ng, 0xffffffffu);
    k_async_rank<<<nblocks(alive), 256, 0, h->stream>>>(S.id, (int)alive, h->a_rowk.get());
    h->launches += 2;
    if ((rc = scan_reserve(h, (size_t)ng)) != MPMB_OK) return rc;
    for (int to_backup = 0; to_backup < 2; to_backup++) {
      MpmbEngine::APool &D = to_backup ? B0 : P0;
      int cnt = 0;
      k_async_route_flags<<<nblocks(ng), 256, 0, h->stream>>>(h->a_rowk.get(), ng, S.block, h->a_bfl.get(), to_backup, h->scan_a.get());
      h->launches++;
      if ((rc = scan_flags(h, (size_t)ng, &cnt)) != MPMB_OK) return rc;
      if (cnt == 0) continue;
      if ((rc = apool_reserve(h, D, D.n + cnt)) != MPMB_OK) return rc;
      k_async_route<<<nblocks(ng), 256, 0, h->stream>>>(h->a_rowk.get(), ng, h->scan_a.get(), h->scan_b.get(), S, G.id, D.rec(D.cur), (int)D.n);
      h->launches++;
      D.n += cnt;
    }
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  *n_gathered = ng;
  return MPMB_OK;
}

extern "C" {

int mpmb_async_advance(MpmbHandle h, const uint8_t *flags, float dt, int64_t *n_gathered) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = async_check(h, true);
  if (rc != MPMB_OK) return rc;
  if (!flags || !n_gathered) return fail(h, MPMB_ERR_INVALID, "null argument");
  if (!(dt > 0.f) || !std::isfinite(dt)) return fail(h, MPMB_ERR_INVALID, "dt must be positive and finite");
  *n_gathered = 0;
  int sc = 0;
  for (int i = 0; i < h->nblk; i++) sc |= flags[i] & (MPMB_ASYNC_SWAP | MPMB_ASYNC_CLEAR);
  CUDA_TRY(h, cudaMemcpyAsync(h->a_bfl.get(), flags, (size_t)h->nblk, cudaMemcpyHostToDevice, h->stream));
  return async_advance_body(h, dt, sc, n_gathered);
}

int mpmb_async_schedule(MpmbHandle h, int64_t t, float strength_mul, float cfl_mul, float dx, float inv_unit, int64_t max_units, int32_t *min_level,
                        int32_t *max_level) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = async_check(h, true);
  if (rc != MPMB_OK) return rc;
  if (!min_level || !max_level) return fail(h, MPMB_ERR_INVALID, "null argument");
  if (t < 0) return fail(h, MPMB_ERR_INVALID, "t = %lld is negative", (long long)t);
  if (max_units < 1 || max_units > (1ll << 30)) return fail(h, MPMB_ERR_INVALID, "max_units = %lld outside [1, 2^30]", (long long)max_units);
  const int nblk = h->nblk;
  const MpmbEngine::APool &p = h->apool[0];
  ASched *S = h->a_sched.get();
  k_async_sched_reset<<<nblocks(nblk), 256, 0, h->stream>>>(nblk, h->a_bflag.get(), h->a_bmin.get(), h->a_bmax.get(), S);
  h->launches++;
  if (p.n > 0) {
    k_async_limits<<<nblocks(p.n), 256, 0, h->stream>>>(p.rec(p.cur), (int)p.n, h->P, 1, h->a_bflag.get(), h->a_bmin.get(), h->a_bmax.get(), &S->bad);
    h->launches++;
  }
  k_async_sched_due<<<nblocks(nblk), 256, 0, h->stream>>>(h->a_bflag.get(), h->a_bmin.get(), h->a_bmax.get(), h->a_level.get(), h->a_lvnew.get(), nblk, (long long)t,
                                                          strength_mul, cfl_mul, dx, inv_unit, (long long)max_units, S);
  k_async_sched_commit<<<nblocks(nblk), 256, 0, h->stream>>>(h->a_bflag.get(), h->a_lvnew.get(), h->a_level.get(), nblk, (long long)t, S);
  k_async_local_min<<<nblocks(nblk), 256, 0, h->stream>>>(h->a_level.get(), h->a_particle_t.get(), h->a_local_min.get(), h->anb[0], h->anb[1], h->anb[2], S);
  h->launches += 3;
  ASched s;
  CUDA_TRY(h, cudaMemcpyAsync(&s, S, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, cudaGetLastError());
  if (s.bad && s.due) return fail(h, MPMB_ERR_INVALID, "%d pool particles are of a type without a time-step limit (linear / jelly)", s.bad);
  if (s.low) return fail(h, MPMB_ERR_LIMIT, "a due block's time-step limit is below unit_delta_t");
  *min_level = s.lv_min;
  *max_level = s.lv_max;
  return MPMB_OK;
}

int mpmb_async_advance_level(MpmbHandle h, int64_t t, int32_t limit, float dt, int64_t *n_gathered) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = async_check(h, true);
  if (rc != MPMB_OK) return rc;
  if (!n_gathered) return fail(h, MPMB_ERR_INVALID, "null argument");
  *n_gathered = 0;
  if (t < 0) return fail(h, MPMB_ERR_INVALID, "t = %lld is negative", (long long)t);
  if (limit < 1 || (limit & (limit - 1))) return fail(h, MPMB_ERR_INVALID, "limit = %d is not a positive power of two", limit);
  if (!(dt > 0.f) || !std::isfinite(dt)) return fail(h, MPMB_ERR_INVALID, "dt must be positive and finite");
  const int nblk = h->nblk;
  CUDA_TRY(h, cudaMemsetAsync(&h->a_sched.get()->sc, 0, sizeof(int), h->stream));
  k_async_level_flags<<<nblocks(nblk), 256, 0, h->stream>>>(h->a_level.get(), h->a_particle_t.get(), h->a_local_min.get(), h->anb[0], h->anb[1], h->anb[2],
                                                            (long long)t, limit, h->a_bfl.get(), h->a_sched.get());
  h->launches++;
  if ((rc = async_advance_body(h, dt, -1, n_gathered)) != MPMB_OK) return rc;
  // the clocks move only once the advance has succeeded
  k_async_level_clocks<<<nblocks(nblk), 256, 0, h->stream>>>(h->a_bfl.get(), nblk, (long long)t, limit, h->a_particle_t.get(), h->a_backup_t.get());
  h->launches++;
  CUDA_TRY(h, cudaGetLastError());
  return MPMB_OK;
}

int mpmb_async_block_state(MpmbHandle h, int32_t *level, int64_t *local_min, int64_t *particle_t, int64_t *backup_t) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = async_check(h, true);
  if (rc != MPMB_OK) return rc;
  const size_t n = (size_t)h->nblk;
  const struct { void *d; const void *s; size_t w; } cp[] = {{level, h->a_level.get(), sizeof(int32_t)}, {local_min, h->a_local_min.get(), sizeof(int64_t)},
                                                            {particle_t, h->a_particle_t.get(), sizeof(int64_t)}, {backup_t, h->a_backup_t.get(), sizeof(int64_t)}};
  for (const auto &c : cp)
    if (c.d) CUDA_TRY(h, cudaMemcpyAsync(c.d, c.s, c.w * n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return MPMB_OK;
}

int mpmb_async_size(MpmbHandle h, int64_t *n_pool, int64_t *n_backup) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = async_check(h, true);
  if (rc != MPMB_OK) return rc;
  if (n_pool) *n_pool = h->apool[0].n;
  if (n_backup) *n_backup = h->apool[1].n;
  return MPMB_OK;
}

int mpmb_async_download(MpmbHandle h, int32_t which, int64_t cap, int64_t *n_out, uint32_t *id, int32_t *block, float *x, float *v, float *F,
                        float *b, float *mass, float *vol, float *scalar, int32_t *group) {
  CHECK_HANDLE(h);
  NOT_2D(h);
  int rc = async_check(h, true);
  if (rc != MPMB_OK) return rc;
  if (which < 0 || which > 1) return fail(h, MPMB_ERR_INVALID, "which = %d: 0 (particle pool) or 1 (backup pool)", which);
  if (!n_out) return fail(h, MPMB_ERR_INVALID, "n_out is required");
  const MpmbEngine::APool &p = h->apool[which];
  *n_out = p.n;
  if (p.n > cap) return fail(h, MPMB_ERR_CAPACITY, "%lld records do not fit in the %lld rows provided", (long long)p.n, (long long)cap);
  const ARec r = p.rec(p.cur);
  const size_t n = (size_t)p.n;
  const struct { void *d; const void *s; size_t w; } cp[] = {{id, r.id, 1}, {block, r.block, 1}, {x, r.x, 3}, {v, r.v, 3}, {F, r.F, 9}, {b, r.b, 9},
                                                            {mass, r.mass, 1}, {vol, r.vol, 1}, {scalar, r.scalar, 1}, {group, r.group, 1}};
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  for (const auto &c : cp)
    if (c.d && n > 0) CUDA_TRY(h, cudaMemcpyAsync(c.d, c.s, 4 * c.w * n, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return MPMB_OK;
}

}  // extern "C"
