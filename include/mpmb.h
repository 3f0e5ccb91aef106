/*
 * mpmb.h — C-ABI of the H100-native MLS-MPM substep engine (libmpmb.so).
 *
 * This is the drop-in boundary for ONE hot path of yuanming-hu/taichi_mpm: the calls made by
 * MPM<3>::substep() (reference src/mpm.cpp:452-575) between particle ordering and particle
 * deletion.  Every entry point names the reference interface it replaces (path:line under the
 * reference tree).  Plain C types only: opaque handle, pointers and sizes; no exceptions cross the
 * boundary; every call returns 0 on success or a negative MpmbStatus, and the text of the last
 * failure is available from mpmb_last_error().
 *
 * Ownership: the library owns all device memory; the caller owns every host buffer it passes and
 * no host pointer is retained after a call returns.  Entry points are not re-entrant per handle;
 * distinct handles are independent.  One handle drives one GPU (one process per GPU; multi-GPU
 * z-slab runs exchange the buffers exposed by the mpmb_halo_* / mpmb_migrate_* calls with
 * whatever transport the host owns — torch.distributed/NCCL in this repository).
 *
 * Numeric contract: fp32 state (reference `real = float`, README.md:316-317), 3x3 matrices stored
 * column-major as 9 floats (m[c*3+r]; reference `M[i]` is column i, README.md:314), `b` is the
 * reference's `apic_b` (src/particles.h:24-45): C = -4/dx * b in the 88-line notation.
 */
#ifndef MPMB_H_
#define MPMB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPMB_VERSION 1
#define MPMB_MAX_GROUPS 16  /* material groups per handle */
#define MPMB_MAT_PARAMS 8

typedef struct MpmbEngine *MpmbHandle;

typedef enum MpmbStatus {
  MPMB_OK = 0,
  MPMB_ERR_INVALID = -1,   /* bad argument */
  MPMB_ERR_CUDA = -2,      /* a CUDA call failed (sticky per handle) */
  MPMB_ERR_CAPACITY = -3,  /* particle / tile / exchange-buffer capacity exceeded */
  MPMB_ERR_STATE = -4,     /* call not valid in the current state */
  MPMB_ERR_LIMIT = -5      /* AsyncMPM: a block's time-step limit is below one unit (mpmb_async_schedule) */
} MpmbStatus;

/* Material kinds = the registered particle type names of the reference
 * (TC_REGISTER_MPM_PARTICLE, src/particles.cpp:845-856; all eight deformable types).  Parameter vectors (unused entries 0):
 *   LINEAR  "linear" (src/particles.cpp:297-363): [0]=mu [1]=lambda
 *   JELLY   "jelly"  (src/particles.cpp:365-438): [0]=mu [1]=lambda
 *   SNOW    "snow"   (src/particles.cpp:165-295): [0]=mu_0 [1]=lambda_0 [2]=hardening [3]=theta_c
 *                                                  [4]=theta_s [5]=min_Jp [6]=max_Jp ; scalar = Jp
 *   WATER   "water"  (src/particles.cpp:440-499): [0]=k [1]=gamma ; scalar = j
 *   SAND    "sand"   (src/particles.cpp:563-676): [0]=mu_0 [1]=lambda_0 [2]=alpha [3]=cohesion
 *                                                  [4]=beta ; scalar = logJp
 *   ELASTIC "elastic" (src/particles.cpp:764-841): [0]=mu_0 [1]=lambda_0   (Hencky, no return map)
 *   VON_MISES "von_mises" (src/particles.cpp:679-761): [0]=mu_0 [1]=lambda_0 [2]=yield_stress
 *   VISCO   "visco"  (src/particles.cpp:40-163): [0]=mu_0 [1]=lambda_0 [2]=visco_nu [3]=visco_kappa
 *                                                  [4]=dt (the particle's own `base_delta_t` key, default 1e-4,
 *                                                  src/particles.cpp:66) ; scalar = visco_tau              */
typedef enum MpmbMaterial {
  MPMB_MAT_LINEAR = 0,
  MPMB_MAT_JELLY = 1,
  MPMB_MAT_SNOW = 2,
  MPMB_MAT_WATER = 3,
  MPMB_MAT_SAND = 4,
  MPMB_MAT_ELASTIC = 5,
  MPMB_MAT_VON_MISES = 6,
  MPMB_MAT_VISCO = 7
} MpmbMaterial;

/* Mirrors the keys MPM<dim>::initialize reads from its Config (src/mpm.cpp:27-75). */
typedef struct MpmbConfig {
  int32_t res[3];            /* cells per axis (`res`); nodes = res+1 (src/mpm.cpp:66)            */
  float dx;                  /* `delta_x`                                                         */
  float dt;                  /* `base_delta_t` (already multiplied by dt_multiplier)              */
  float gravity[3];          /* `gravity` (src/mpm.cpp:38)                                        */
  int32_t particle_gravity;  /* src/mpm.cpp:47 (default 1): kick particles in P2G, not the grid   */
  int32_t clean_boundary;    /* src/mpm.cpp:563 (default 1): delete particles in the 7-cell band  */
                             /* 0: particles in the band are kept and simulated.  Whatever the flag, a particle
                              * whose 27-node stencil [base, base+2] (base = int(x/dx - 0.5) per axis) leaves the
                              * (res+1)^3 node grid, or whose position is not finite, is deleted: at upload and
                              * after every G2P.  It is gone from the downloads and from mpmb_num_particles, and
                              * no error is reported.  (The reference would write past res into its SPGrid.)   */
  int32_t device;            /* CUDA device ordinal                                               */
  int64_t capacity;          /* max resident particles; 0 = sized at the first upload             */
  /* z-slab decomposition (SURVEY §8e).  world==1: whole domain.  A rank owns the particles whose
   * base node lies in tile layers [tile_z0, tile_z1) (tiles are 4x4x4 nodes).                    */
  int32_t rank, world;
  int32_t tile_z0, tile_z1;
  int64_t migrate_capacity;  /* max particles leaving through one face per substep (world>1)      */
  int32_t halo_capacity;     /* max active tiles in one boundary layer; 0 = the whole cross-section */
  int32_t no_graph;          /* 1: launch every kernel from the host; 0 (default): mpmb_substep replays pairs of
                              * substeps as a CUDA graph (same kernels, same order, same results)              */
  /* 0 or 3: MPM<3> (everything above and below).  2: MPM<2> (src/mpm.cpp:983-988): res[2] == 0, gravity[2] == 0,
   * world == 1; particle arrays are dim-packed (x[n][2], v[n][2], F[n][4] and b[n][4] column-major), a dense node
   * array is [res0+1][res1+1][4] with the z component 0, and only these entry points work on the handle:
   *   mpmb_create, mpmb_destroy, mpmb_last_error, mpmb_set_stream, mpmb_synchronize, mpmb_set_material,
   *   mpmb_set_delta_t, mpmb_set_planes / mpmb_set_levelset_shapes (planes, circles as MPMB_SHAPE_SPHERE, rectangles as
   *   MPMB_SHAPE_CUBOID; every z part must be 0), mpmb_set_sdf, mpmb_upload_particles, mpmb_set_id_base,
   *   mpmb_num_particles, mpmb_get_update_count, mpmb_download_particles, mpmb_download_bgeo_points (z = 0, as
   *   MPM<2>::write_partio writes), mpmb_substep and its three stages, mpmb_download_grid, mpmb_set_profiling,
   *   mpmb_get_profile, mpmb_get_counters, mpmb_upload_aos and mpmb_download_aos (MPM<2>'s own pool; the 2-D meaning of
   *   MpmbAosLayout is given there).
   * Every other entry point returns MPMB_ERR_STATE (the *_bytes calls included) with a message: lattice seeding,
   * appends and deletions, rigid bodies, AsyncMPM, z-slabs and re-cuts are MPM<3> only.
   * The deletion rule is the same as in 3-D with the 9-node stencil; in addition G2P clamps the position to
   * [0, res - 1e-6] cells as MPM<2>::resample does, and a particle whose velocity is not finite is deleted too.      */
  int32_t dim;
  /* `apic_damping` / `rpic_damping` (src/mpm.cpp:33-34, src/mpm.h:465-469): apic_b = (1 - rpic) sym(b) + (1 - apic)
   * skew(b).  dim == 2 only (0 otherwise: MPM<3>'s optimized resample passes them a block index).                  */
  float apic_damping, rpic_damping;
  int32_t reserved[3];       /* must be 0                                                         */
} MpmbConfig;

/* Byte offsets of the fields of one reference particle slot (ParticleContainer<3>, 320 B,
 * src/mpm_fwd.h:59-67; fields src/particles.h:24-45).  Obtained with offsetof() on the reference
 * side (INTEGRATION.md); never hard-coded here.  Offset < 0 = field absent.
 *
 * On a 2-D handle (MpmbConfig.dim = 2) the same struct describes a ParticleContainer<2> slot of MPM<2>
 * (192 B in the reference's build): pos is float[2], v_and_m float[3] = (vx, vy, mass) (v_and_m[dim]
 * is the mass, src/particles.h:66-72), dg_e and apic_b are 2 columns of 2 floats col_pitch apart
 * (column-major, as MatrixND<2> stores them), and vol and the scalar modes are as in 3-D.  Every field
 * must lie inside `stride` at a 4-aligned offset, stride must be a multiple of 4 and col_pitch a multiple
 * of 4 that is at least 8; otherwise both AoS calls return MPMB_ERR_INVALID and change nothing.
 *
 * The plastic scalar has two modes.
 *  - Single offset (off_scalar_by_kind all 0, the zero-initialised struct): every row's scalar is at
 *    off_scalar.  With off_scalar = -1 the upload packs 0 for every row, snow and water included (not
 *    the Jp = 1 / j = 1 of mpmb_upload_particles; kept as it always was), and the download writes none.
 *  - Per kind (any off_scalar_by_kind entry != 0): the pool mixes particle types, each of which keeps
 *    its scalar at its own offset.  off_scalar must be -1, and each entry is -1 (no scalar in the slot)
 *    or a 4-aligned offset in (0, stride - 4]; otherwise both AoS calls return MPMB_ERR_INVALID and
 *    change nothing.  A row's offset follows the material KIND of its group (mpmb_set_material), not
 *    the group number: snow reads Jp, water j, sand logJp, visco visco_tau.  Rows of a kind without an
 *    offset (linear, jelly, elastic, von Mises, or an entry of -1) get mpmb_upload_particles' defaults
 *    (Jp = 1, j = 1, otherwise 0) and have no scalar written back.                                    */
typedef struct MpmbAosLayout {
  int32_t stride;      /* bytes per slot (320)                                       */
  int32_t off_pos;     /* float[3]   `pos`                         (2-D: float[2])     */
  int32_t off_v_and_m; /* float[4]   `v_and_m` = (vx,vy,vz,mass)   (2-D: (vx,vy,mass)) */
  int32_t off_dg_e;    /* 3 x float[4] padded columns of `dg_e` (column pitch below)
                        *                                          (2-D: 2 x float[2]) */
  int32_t off_apic_b;  /* 3 x float[4] padded columns of `apic_b`  (2-D: 2 x float[2]) */
  int32_t col_pitch;   /* bytes between matrix columns (16)          (2-D: >= 8)         */
  int32_t off_vol;     /* float      `vol`                                           */
  int32_t off_scalar;  /* float      Jp / j / logJp of the subclass, or -1           */
  /* float  per-kind scalar: [0] SnowParticle::Jp, [1] WaterParticle::j, [2] SandParticle::logJp,
   * [3] ViscoParticle::visco_tau; -1 = not in the slot; all 0 = single-offset mode (above)          */
  int32_t off_scalar_by_kind[4];
} MpmbAosLayout;

/* ------------------------------------------------------------------------------ lifetime */
/* Replaces MPM<3>::initialize (src/mpm.cpp:27-75): sizes the tile grid, allocates device state. */
int mpmb_create(const MpmbConfig *cfg, MpmbHandle *out);
int mpmb_destroy(MpmbHandle h);
/* Text of the last error on this handle ("" if none).  h may be NULL for create-time errors.    */
const char *mpmb_last_error(MpmbHandle h);
int mpmb_version(void);
/* All work is enqueued on `cuda_stream` (a cudaStream_t cast to void*; NULL = default stream).   */
int mpmb_set_stream(MpmbHandle h, void *cuda_stream);
int mpmb_synchronize(MpmbHandle h);

/* ------------------------------------------------------------------------------ scene     */
/* Replaces Particle::initialize(config) of the registered type (e.g. SandParticle::initialize,
 * src/particles.cpp:587-597) for every particle of `group`.                                      */
int mpmb_set_material(MpmbHandle h, int32_t group, int32_t kind, const float *params, int32_t n_params);
/* (Called with particles of `group` already resident — between substeps — it also rebuilds their cached
 * affine matrices, so the next rasterize uses the new material's stress; apic_b must be current, i.e. the
 * call follows an upload or a completed mpmb_substep / mpmb_resample.)                              */
/* `base_delta_t` of the following substeps.  MPM<3> keeps it fixed, but AsyncMPM sets it before every MPM<dim>::substep() it
 * schedules (src/async/async_mpm.cpp:407-409: base_delta_t = unit_delta_t * delta_t_int), and a host that adapts its step does
 * the same.  With particles resident their cached affine matrices are rebuilt for the new step (apic_b must be current, as for
 * mpmb_set_material); an upload after the call needs nothing.  Between substeps only.                                      */
int mpmb_set_delta_t(MpmbHandle h, float dt);
/* Replaces Simulation::set_levelset + DynamicLevelSet::sample/get_spatial_gradient as used by
 * apply_grid_boundary_conditions (src/mpm.cpp:296-372) for a static level set.  `sdf4` is a host
 * array [res0+1][res1+1][res2+1][4] = (n_x,n_y,n_z,phi), phi in grid units at the node, n the
 * unit spatial gradient.  NULL removes the boundary.  `friction` = levelset0->friction
 * (-1 sticky, <=-2 slip, >=0 separate with Coulomb friction; src/mpm_fwd.h:25-57).               */
int mpmb_set_sdf(MpmbHandle h, const float *sdf4, float friction);
/* Same boundary built on the device from half-spaces phi_i(X) = n_i . X + d_i (grid units, n unit):
 * phi = min_i phi_i, n = n of the minimiser (levelset.add_plane in scripts/mls-cpic/sand_sweep.py:13-19). */
int mpmb_set_planes(MpmbHandle h, int32_t n_planes, const float *planes4, float friction);

/* The level set rasterised on the device from analytic solids (what the reference's scripts build with
 * levelset.add_plane / add_sphere / add_cuboid, e.g. scripts/mls-cpic/sand_sweep.py:13-19, scripts/async/sand.py:35,
 * scripts/mls-cpic/sand_stir.py:9): phi = min over the shapes of their signed distance in GRID units (negative inside
 * the obstacle), n = unit gradient of the minimiser; inside_out makes a container of a solid.  Parameters (grid units):
 *   PLANE  p = {n_x, n_y, n_z, d}       phi = n.X + d  (n unit)
 *   SPHERE p = {c_x, c_y, c_z, r}       phi = |X - c| - r
 *   CUBOID p = {lo_x, lo_y, lo_z, hi_x, hi_y, hi_z}   exact box distance
 * The shape formulas of the reference live in its un-vendored core (LevelSet3D): planes are pinned by the in-place build
 * (DESIGN.md §2), sphere and cuboid follow the published signed-distance definitions — parity unpinned for those two. */
typedef enum MpmbShapeKind { MPMB_SHAPE_PLANE = 0, MPMB_SHAPE_SPHERE = 1, MPMB_SHAPE_CUBOID = 2 } MpmbShapeKind;
typedef struct MpmbShape {
  int32_t kind;        /* MpmbShapeKind */
  int32_t inside_out;  /* 0: the solid is the obstacle; 1: its complement is (a container) */
  float p[6];
} MpmbShape;
int mpmb_set_levelset_shapes(MpmbHandle h, int32_t n_shapes, const MpmbShape *shapes, float friction);

/* ------------------------------------------------------------------------------ particles */
/* Replaces MPM<3>::add_particles' writes into the particle pool (src/mpm.cpp:93-148) for n
 * particles given field-wise: x[n][3], v[n][3], F[n][9], b[n][9] (apic_b), mass[n], vol[n],
 * scalar[n] (Jp/j/logJp), group[n].  F, b, scalar, group may be NULL (identity, 0, material
 * default, group 0).  Replaces the resident set.  Particle k gets id k.                           */
int mpmb_upload_particles(MpmbHandle h, int64_t n, const float *x, const float *v, const float *F, const float *b,
                          const float *mass, const float *vol, const float *scalar, const int32_t *group);
/* Particle k of the next upload gets id `base + k` (default 0); z-slab ranks use disjoint ranges so
 * that ids stay unique after migration.  Ids must stay below 2^28.                                 */
int mpmb_set_id_base(MpmbHandle h, int64_t base);
/* Same, reading the reference's own AoS pool: slot indices[k] of `pool` (ParticleAllocator::pool,
 * src/particle_allocator.h:39; MPM::particles index vector, src/mpm.h:116).  group[k] may be NULL.
 * With per-kind scalar offsets (MpmbAosLayout) the call takes a snapshot of the 16 groups' kinds: set
 * every group's material BEFORE the upload.  The snapshot picks each row's scalar offset here and in the
 * next mpmb_download_aos, whatever mpmb_set_material does in between.                              */
/* On a 2-D handle the rows are those mpmb_upload_particles makes of the same particles.  A slot index
 * outside the pool returns MPMB_ERR_INVALID and leaves the resident set as it was.                  */
int mpmb_upload_aos(MpmbHandle h, int64_t n, const void *pool, int64_t pool_slots, const uint32_t *indices,
                    const MpmbAosLayout *layout, const int32_t *group);
/* Replaces the `benchmark` branch of MPM<3>::add_particles (src/mpm.cpp:149-186: 8 particles per cell of the
 * block [lo_cell, hi_cell) at the cell centre +- 0.25 dx, F = I, apic_b = 0, velocity v0) ON THE DEVICE — no host
 * array, which is what makes 10^7..10^8-particle scenes start in milliseconds.  `vol` / `mass` are the per-particle
 * values the caller derives as add_particles does (vol = dx^3 / maximum, mass = vol * density, src/mpm.cpp:134-135).
 * `jitter` (grid units, < 0.25; 0 = the reference's lattice) displaces every particle by a hash of its lattice index
 * and `seed`, so positions do not depend on the z-slab partition.  Particle ids are id_base + lattice index
 * (((ix*ny + iy)*nz + iz)*8 + corner, cells relative to lo_cell); a z-slab rank keeps the particles it owns;
 * particles within 7 cells of a face are not created (src/mpm.cpp:129-132).  Replaces the resident set.           */
int mpmb_seed_lattice(MpmbHandle h, const int32_t lo_cell[3], const int32_t hi_cell[3], float vol, float mass, float jitter,
                      uint32_t seed, int32_t group, const float v0[3], int64_t *n_seeded);
/* Appends n particles to the resident set (MPM<3>::add_particles' push onto `particles`, src/mpm.cpp:147; ids from
 * ParticleAllocator::particle_counter, src/particle_allocator.h:72).  Fields as mpmb_upload_particles (F, b, scalar,
 * group may be NULL).  Resident particles keep their rows' state, ids and CPIC colours; the new ones get ids
 * id_base + id_span .. + n - 1, where id_span is the end of the ids handed out so far (n of an upload, the lattice range
 * of mpmb_seed_lattice, plus every earlier append); *first_id (may be NULL) receives the first, also for n == 0, which
 * changes nothing.  The same rule as an upload drops particles that are not finite or whose stencil leaves the node grid
 * (they still consume their ids).  The storage needs the resident rows plus n: with capacity == 0 it grows (by at least
 * half) keeping the resident rows; a configured capacity that is too small returns MPMB_ERR_CAPACITY and changes
 * nothing.  Ids past 2^28 return MPMB_ERR_CAPACITY.  The whole set is ordered again, as after an upload, so the next
 * substep is not replayed from a graph.  After an append the index vector of an earlier mpmb_upload_aos does not cover
 * the new ids: mpmb_download_aos then reports MPMB_ERR_INVALID (the new particles are not written anywhere) and the
 * AoS caller must upload again.  Between substeps; world == 1 (else MPMB_ERR_STATE).                                    */
int mpmb_append_particles(MpmbHandle h, int64_t n, const float *x, const float *v, const float *F, const float *b,
                          const float *mass, const float *vol, const float *scalar, const int32_t *group, int64_t *first_id);
/* delete_particles_inside_level_set (src/mpm.cpp:959-973): removes every live particle whose level set value, trilinear
 * in the node phi of the current level set at x / dx (clamped to the node grid, node values capped at 1e20), is < 0.
 * Survivors keep their ids and state; *n_deleted receives the number removed.  No level set: deletes none.  Between
 * substeps; world == 1 (else MPMB_ERR_STATE).                                                                           */
int mpmb_delete_inside_levelset(MpmbHandle h, int64_t *n_deleted);
/* The same two edits for z-slab ranks (world > 1), valid on world == 1 too, with one particle-id sequence across ranks.
 * Every rank receives the SAME batch and the same first_id; particle k gets id first_id + k on the rank that owns it, the
 * rank whose tile layers [tile_z0, tile_z1) hold its base node's tile layer (decided on the device with the key that packs
 * it, as mpmb_seed_lattice decides it).  An in-domain, finite particle is therefore kept by exactly one rank; *n_kept
 * receives this rank's count.  Dropped particles consume their ids as well: every rank, also one that keeps none, raises
 * its id end to max(id_end, first_id + n).  first_id must not lie below mpmb_id_end (MPMB_ERR_INVALID, nothing changed);
 * the next free id of a run is the maximum of mpmb_id_end over its ranks.  On world == 1 the append keeps every particle
 * mpmb_append_particles keeps and, with first_id = the id that call would hand out, gives the same state bit for bit.
 * Growth and capacity as mpmb_append_particles; growth on a z-slab rank keeps its migration headroom, and the exchange
 * buffers the neighbours have mapped (mpmb_xchg_connect) stay where they are.  Ids past 2^28 return MPMB_ERR_CAPACITY.
 * Contract on z-slab runs: every rank makes the same edit at the same substep boundary (between two mpmb_substep calls, or
 * after the migration of the last substep when the host drives the stages).  Peer-connected ranks then go on with
 * mpmb_substep(h, n): the first substep after an edit runs outside the graph, the exchange sequence numbers are untouched.
 * Appends can unbalance the slabs; mpmb_recut_apply moves the cuts.  Between substeps (else MPMB_ERR_STATE); x, v, mass,
 * vol and n_kept are required (MPMB_ERR_INVALID).                                                                       */
int mpmb_append_owned_particles(MpmbHandle h, int64_t n, const float *x, const float *v, const float *F, const float *b,
                                const float *mass, const float *vol, const float *scalar, const int32_t *group,
                                int64_t first_id, int64_t *n_kept);
/* mpmb_delete_inside_levelset on this rank's particles; the level set covers the whole node grid on every rank, so a
 * particle is deleted exactly when one engine holding it would delete it.  Sum *n_deleted over the ranks for the total. */
int mpmb_delete_owned_inside_levelset(MpmbHandle h, int64_t *n_deleted);
/* End of the ids handed out so far (absolute, never below id_base): id_base + n after an upload, id_base + 8 * cells of the
 * whole lattice after mpmb_seed_lattice (on every rank), raised by every append.                                          */
int mpmb_id_end(MpmbHandle h, int64_t *id_end);
/* Number of live particles, counted on the device (4 bytes cross the bus; synchronises).
 * Reference: particles.size().                                                                    */
int mpmb_num_particles(MpmbHandle h, int64_t *n);
/* Sum over all substeps so far of the particles each one updated — the reference's `update_counter +=
 * particles.size()` per substep (src/mpm.cpp:436,449), counted on the device (exact when particles are
 * deleted in the middle of a frame).                                                               */
int mpmb_get_update_count(MpmbHandle h, int64_t *updates);
/* Copies the live particles out, any pointer may be NULL.  Row k of every array belongs to the
 * particle whose id (upload index) is id[k]; rows are in the engine's storage order.  `cap` rows
 * are available in each array; *n_out receives the number written.                                */
int mpmb_download_particles(MpmbHandle h, int64_t cap, int64_t *n_out, uint32_t *id, float *x, float *v, float *F,
                            float *b, float *mass, float *vol, float *scalar, int32_t *group);
/* Writes the live particles back into the reference's AoS pool (slot = indices[id]); returns the
 * number of survivors and compacts `indices` to the survivors (in id order), which is what
 * clear_boundary_particles (src/mpm.cpp:583-633) leaves in MPM::particles.  The scatter runs on the
 * device into the image of the pool kept since mpmb_upload_aos; both directions move only the window of
 * every slot that holds the layout's fields (a 2-D copy with the slot stride as pitch: 204 of the
 * reference's 320 bytes), so bytes outside it (vptr, flags, ...) are never touched on the host.  Fields
 * inside the window that the engine does not own (e.g. boundary_normal) return as uploaded: do not
 * modify the pool between the two calls (the device owns the particles during step(), SURVEY §8b).
 * Without a preceding mpmb_upload_aos of the same pool the image is read first.  With per-kind scalar
 * offsets each row's scalar goes to the offset of its group's kind as of the last mpmb_upload_aos (its
 * snapshot), and only for kinds that have one; no other byte of any slot is written.  That mode needs an
 * mpmb_upload_aos on the handle since the last mpmb_upload_particles / mpmb_seed_lattice (else
 * MPMB_ERR_STATE).                                                                                  */
/* On a 2-D handle a particle id or slot index outside the vectors returns MPMB_ERR_INVALID before any
 * byte of the host pool or of `indices` is written.                                                   */
int mpmb_download_aos(MpmbHandle h, void *pool, int64_t pool_slots, uint32_t *indices, int64_t n_indices,
                      const MpmbAosLayout *layout, int64_t *n_alive);

/* Frame dump without a host pass over the particles: the per-point records of MPM<3>::write_partio through Partio's
 * BGEO writer (src/visualize.cpp:16-100, external/partio/src/io/BGEO.cpp:131-150) — big-endian words position xyz,
 * w = 1, type = 0, index = id, limit = (1,1,1), v xyz: 48 bytes per particle, non-verbose dump — packed on the device in
 * id order and copied into `records` (cap_records x 48 bytes).  `id_range`: ids are below id_base + id_range.  The caller
 * writes the file header and trailer around the block (taichi_mpm_b200/bgeo.py does).                              */
int mpmb_download_bgeo_points(MpmbHandle h, int64_t id_range, void *records, int64_t cap_records, int64_t *n_out);

/* ------------------------------------------------------------------------------ hot path  */
/* The whole of MPM<3>::substep() on the fast path, `nsub` times (src/mpm.cpp:452-575):
 * sort_particles_and_populate_grid (464-465) -> rasterize_optimized (510-512) ->
 * normalize_grid_and_apply_external_force (526-533) -> apply_grid_boundary_conditions (539-540) ->
 * resample_optimized (548-549) -> clear_boundary_particles (563-565).  Asynchronous.              */
int mpmb_substep(MpmbHandle h, int32_t nsub);
/* The same stages one at a time (for parity tests and for a host that interleaves its own work,
 * e.g. rigid bodies).  Must be called in this order; mpmb_substep == these three.                  */
int mpmb_sort_particles_and_populate_grid(MpmbHandle h); /* src/mpm.cpp:770-918                   */
int mpmb_rasterize(MpmbHandle h);                        /* src/transfer.cpp:361-581 (P2G)        */
int mpmb_resample(MpmbHandle h);                         /* src/mpm.cpp:277-372 + src/transfer.cpp:702-970 + src/mpm.cpp:583-633 */

/* z-slab runs (world>1): the same two stages, each in two launches — part 1 = the tiles of the
 * slab's two boundary layers (they produce and consume halo data), part 2 = all other tiles — so
 * that the host can overlap the halo exchange with the interior work:
 *   sort; rasterize_part(1); halo_pack; [send/recv starts]; rasterize_part(2); resample_part(2);
 *   [send/recv done]; halo_unpack; resample_part(1); migrate_*.                                     */
int mpmb_rasterize_part(MpmbHandle h, int32_t part);
int mpmb_resample_part(MpmbHandle h, int32_t part);

/* Parity/debug: dense node grid [res0+1][res1+1][res2+1][4] on the host.
 * which=0: (p_x,p_y,p_z,m) after P2G; which=1: (v_x,v_y,v_z,m) after normalise + boundary.
 * Valid between mpmb_rasterize and the next mpmb_sort_particles_and_populate_grid.                 */
int mpmb_download_grid(MpmbHandle h, int32_t which, float *dense4);

/* ------------------------------------------------------------------------------ rigid bodies (CPIC) */
/* Two-way coupling with rigid bodies as the reference's optimized path does it (SURVEY §8f row 2).  On the device:
 * update_rigid_page_map (src/mpm.cpp:1026-1076), rasterize_rigid_boundary and gather_cdf (src/rigid_transfer.cpp:18-113,
 * 120-274) and the block_op_rigid branches of rasterize_optimized / resample_optimized (src/transfer.cpp:367-463, 706-835),
 * selected per 4x4x8-node page exactly as block_op_switch does.  The bodies themselves (RigidBody: integration, scripted
 * motion, rigid-rigid collisions, articulation — src/mpm_rigid_body.cpp:252-330 call into the reference's un-vendored core for
 * these) are advanced in one of two ways:
 *   - by the host (the default): per substep the host hands over poses and velocities and reads the velocities back,
 *         mpmb_set_rigid_state -> mpmb_substep(h, 1) -> mpmb_get_rigid_state -> host: advect_rigid_bodies
 *     (mpmb_substep(h, n > 1) keeps the pose fixed over the n substeps; no CUDA-graph replay);
 *   - on the device, after mpmb_set_rigid_motion: every substep ends with advect_rigid_bodies (and, if asked for,
 *     rigid_body_levelset_collision) on an fp64 master state per body, scripted parts taken from a table the host uploads
 *     with mpmb_set_rigid_script.  mpmb_substep(h, n) then runs n whole coupled substeps and replays CUDA graphs.
 * Rigid-rigid collisions (rigidify) and articulation are not implemented.  z-slab runs (world > 1): every rank holds every
 * body and every boundary sample and rasterises the colour field over the whole node grid; each transfer's impulses are summed
 * over the ranks in rank order (mpmb_rigid_* below), so the bodies are bit-identical on every rank.
 * What the device assumes of the core's RigidBody (it cannot be read here; SURVEY appendix C):
 *   get_velocity_at(p) = velocity + angular_velocity x (p - position);
 *   apply_tmp_impulse(j, p): tmp_velocity += inv_mass j, tmp_angular_velocity += inv_inertia ((p - position) x j);
 *   apply_tmp_velocity(): velocity += tmp_velocity, angular_velocity += tmp_angular_velocity (after each transfer);
 *   get_mesh_to_world() = get_centroid_to_world() = x -> position + rot x;
 *   world_to_element(e) = [v1 - v0, v2 - v0, n]^-1 with n the unit normal (v1 - v0) x (v2 - v0).                      */
typedef struct MpmbRigidBody {
  float position[3];          /* centre of mass, world units                                  */
  float rot[9];               /* mesh -> world linear part, column-major                      */
  float velocity[3];
  float angular_velocity[3];
  float inv_mass;             /* 0: scripted / infinite mass (set_infinity_mass)               */
  float inv_inertia[9];       /* world-space inverse inertia, column-major; 0: scripted rotation */
  float frictions[2];         /* RigidBody::frictions: [side of the particle's colour bit]     */
} MpmbRigidBody;
/* Replaces the RigidBoundaryParticles of MPM<3>::add_rigid_particle (src/mpm_rigid_body.cpp:137-250,
 * src/boundary_particle.h): sample s belongs to body rigid_id[s] (the index into MPM::rigids: 1..n_bodies-1; 0 is the
 * background body, src/mpm.cpp:72-74), sits at `offset` in the body's centroid frame and carries its triangle
 * `untransformed_element` (v0, v1, v2; 9 floats).  n_samples = 0 switches the coupling off.  n_bodies <= 12
 * (GridState::max_num_rigid_bodies, src/mpm_fwd.h:79).                                                                 */
int mpmb_set_rigid_samples(MpmbHandle h, int32_t n_bodies, int64_t n_samples, const float *offset3, const float *tri9,
                           const int32_t *rigid_id);
/* `penalty` (src/mpm.cpp:35, default 0) and `pushing_force` (src/mpm.cpp:40, default 20000).                          */
/* (mpmb_set_rigid_samples switches device advection off: the motion records describe one set of bodies.)               */
int mpmb_set_rigid_coupling(MpmbHandle h, float penalty, float pushing_force);
/* Poses and velocities of all n_bodies bodies (entry 0 ignored) for the next substep(s).  With device advection on it also
 * restarts the fp64 master states from these (fp32) values.                                                           */
int mpmb_set_rigid_state(MpmbHandle h, int32_t n_bodies, const MpmbRigidBody *bodies);
/* The same records (synchronises).  Host-advanced bodies: velocity / angular_velocity as the two transfers of the last
 * substep left them, the pose as set.  Device-advanced bodies: the advanced pose and velocities (fp32 copies of the master
 * state) and the world-space inverse inertia of that pose.                                                            */
int mpmb_get_rigid_state(MpmbHandle h, int32_t n_bodies, MpmbRigidBody *bodies);
/* Device advection (advect_rigid_bodies, src/mpm_rigid_body.cpp:273-287), one record per body (entry 0 ignored: the
 * background body is never advanced).  After the second transfer of every substep, per body in fp64:
 *   [levelset_collision != 0 and a level set is set: rigid_body_levelset_collision (src/mpm_rigid_body.cpp:347-384) — phi
 *    trilinear in the node phi at every boundary sample, its central-difference gradient (eps 0.25 grid units) normalised,
 *    normal + Coulomb friction impulses (frictions[0]) with restitution applied sample after sample in sample order;
 *    bodies with zero inverse mass and inertia are skipped]
 *   enforce the rotation axis; free position: v *= exp(-linear_damping dt), x += v dt; scripted position: x, v of the script
 *   entry; free rotation: w *= exp(-angular_damping dt), R = exp([w dt]x) R; scripted rotation: R, w of the entry; gravity
 *   impulse v += g mass dt inv_mass (inv_mass = 0 for a scripted position, else 1 / mass); enforce the axis again;
 *   inverse inertia = R inv_inertia_body R^T.
 * The master states start from the current records (mpmb_set_rigid_state, before or after this call).  Velocities entering a
 * substep's advance are the fp32 values the transfers produced, as a host reading them back sees them.  Requires
 * mpmb_set_rigid_samples first (else MPMB_ERR_STATE); n_bodies must match (else MPMB_ERR_INVALID), fields finite and a free
 * body's mass positive (else MPMB_ERR_INVALID).  n_bodies == 0 switches device advection off (host-advanced contract).
 * Resets the script (no entries left).  The level-set collision runs after the transfers of a substep, not between the grid
 * normalisation and the grid boundary condition as in the reference (src/mpm.cpp:535-538).                            */
typedef struct MpmbRigidMotion {
  float mass;
  float inv_inertia_body[9];   /* body frame, column-major; all 0 = scripted / infinite inertia                      */
  float rotation_axis[3];      /* enforce_angular_velocity_parallel_to when max |axis| > 0.1                        */
  float linear_damping, angular_damping, restitution;
  int32_t scripted_position, scripted_rotation;
  int32_t reserved[4];
} MpmbRigidMotion;
int mpmb_set_rigid_motion(MpmbHandle h, int32_t n_bodies, const MpmbRigidMotion *motion, int32_t levelset_collision);
/* Script table of the scripted parts: poses[n_substeps][n_bodies][18] = position (3), rotation (9, column-major), velocity
 * (3), angular velocity (3) at the END of substep k; only the scripted parts of an entry are read.  Resets the cursor;
 * every device advance consumes one entry.  When a scripted body is present and fewer than nsub entries are left,
 * mpmb_substep(h, nsub) returns MPMB_ERR_STATE and enqueues nothing (mpmb_resample likewise with none left).  Needs
 * mpmb_set_rigid_motion first (else MPMB_ERR_STATE); n_substeps < 0, a NULL table or non-finite scripted parts:
 * MPMB_ERR_INVALID.  The table is copied (synchronises).                                                               */
int mpmb_set_rigid_script(MpmbHandle h, int32_t n_substeps, const double *poses);
/* MPMParticle::states (src/particles.h) by particle id - id_base: set (default 0 for uploaded particles) / read together
 * with boundary_normal, boundary_distance and near_boundary_ of the last substep.  Any pointer may be NULL.
 * z-slab ranks index both by the ABSOLUTE particle id (entry k = id k); only the entries of the particles the rank owns
 * are meaningful.                                                                                                     */
int mpmb_set_particle_states(MpmbHandle h, int64_t n, const uint32_t *states);
int mpmb_get_particle_cdf(MpmbHandle h, int64_t n, uint32_t *states, float *normal3, float *distance, uint8_t *near_boundary);
/* Parity/debug: the node colour field of the last substep, dense [res0+1][res1+1][res2+1]: GridState::states
 * (tags | (rigid id + 1) << 24) and GridState::distance (world units).                                                 */
int mpmb_download_cdf(MpmbHandle h, uint32_t *node_states, float *node_distance);

/* ------------------------------------------------------------------------------ AsyncMPM pools */
/* The particle_pool and backup_pool of the reference's AsyncMPM<3> (src/async/async_mpm.h:85-117), kept on the device so that
 * the block scheduler (levels, neighbour masks: on the host or with mpmb_async_schedule / mpmb_async_advance_level on the
 * device; the step loop on the host) moves no particle record across the bus.  A record
 * is x, v, F, b, mass, vol, scalar, group, id and the linear index of its 4x4x8-node scheduler block,
 *   base = int(x * inv_dx - 0.5) (fp32, the HOST's inv_dx), block (base_x >> 2, base_y >> 2, base_z >> 3),
 *   linear (bx * nb1 + by) * nb2 + bz.
 * Each advance gathers a particle set from the pools and runs one ordinary substep on it (src/async/async_mpm.cpp:256-373):
 * the engine's resident set is replaced by every advance.  Single-GPU engines without rigid samples, between substeps (else
 * MPMB_ERR_STATE); every call but mpmb_async_init needs a preceding mpmb_async_init (else MPMB_ERR_STATE).                */
enum { MPMB_ASYNC_SMALLER = 1, MPMB_ASYNC_EQUAL = 2, MPMB_ASYNC_LARGER = 4, MPMB_ASYNC_SWAP = 8, MPMB_ASYNC_CLEAR = 16 };
/* nb = scheduler blocks per axis (each in [1, 4096]); inv_dx = the host's float32(1 / dx).  Empties both pools.           */
int mpmb_async_init(MpmbHandle h, const int32_t nb[3], float inv_dx);
/* Appends n records to pool `which` (0 particle_pool, 1 backup_pool) in order; their blocks are computed from x.  Every
 * array is required.  A record whose block lies outside the nb grid: MPMB_ERR_INVALID and the pool is unchanged.         */
int mpmb_async_add(MpmbHandle h, int32_t which, int64_t n, const float *x, const float *v, const float *F, const float *b, const float *mass,
                   const float *vol, const float *scalar, const int32_t *group, const uint32_t *id);
/* One pass over the particle pool (the backup pool is not read): the occupied blocks in ascending linear index into block[],
 * *n_blocks their number (MPMB_ERR_CAPACITY if more than cap).  With with_limits also, per block, min(0.1, allowed_dt) over
 * its particles starting from 0.1 and max |v|^2 starting from 1e-16 (update_dt_limits, src/async/async_mpm.cpp:100-112);
 * |v|^2 = (vx vx + vy vy) + vz vz rounded per operation, allowed_dt = MPMParticle::get_allowed_dt of snow, water, sand,
 * elastic, von_mises and visco; a NaN makes the block's value NaN.  A pool particle of a type without a limit (linear,
 * jelly) returns MPMB_ERR_INVALID (the reference stops, :112-124).  min_dt / max_v2 may be NULL without limits.          */
int mpmb_async_block_limits(MpmbHandle h, int32_t with_limits, int64_t cap, int64_t *n_blocks, int32_t *block, float *min_dt, float *max_v2);
/* AsyncMPM::advance for one time level: flags[nb0 * nb1 * nb2] are the MPMB_ASYNC_* bits of every block, dt the level's step.
 *  1. gather: pool entries of SMALLER blocks, then pool entries of EQUAL blocks, then backup entries of LARGER blocks, each
 *     part stably ordered by the block's SPGrid page index; the first copy of every id is kept; gather index k is engine id k;
 *  2. backup <- backup[not SWAP] ++ pool[SWAP], pool <- pool[not SWAP];
 *  3. if the set is not empty: the step becomes dt (as mpmb_set_delta_t), the set replaces the resident particles and one
 *     substep runs; the survivors' blocks are computed from their new x;
 *  4. backup <- backup[not CLEAR];
 *  5. in gather order, survivors whose new block is EQUAL are appended to the pool, those whose new block is CLEAR and not
 *     EQUAL to the backup; the others are dropped.
 * *n_gathered receives the size of the set (the reference's update_counter increment).  All pool edits are stable.  A
 * configured capacity below the set: MPMB_ERR_CAPACITY, both pools unchanged.  NULL flags: MPMB_ERR_INVALID.             */
int mpmb_async_advance(MpmbHandle h, const uint8_t *flags, float dt, int64_t *n_gathered);
/* Records in the pools (either pointer may be NULL).                                                                      */
int mpmb_async_size(MpmbHandle h, int64_t *n_pool, int64_t *n_backup);
/* Copies pool `which` out in pool order, any array may be NULL; *n_out receives its size (MPMB_ERR_CAPACITY and nothing
 * written if it exceeds cap).  Synchronises.                                                                              */
int mpmb_async_download(MpmbHandle h, int32_t which, int64_t cap, int64_t *n_out, uint32_t *id, int32_t *block, float *x, float *v, float *F,
                        float *b, float *mass, float *vol, float *scalar, int32_t *group);
/* The block scheduler on the device.  mpmb_async_init sets every block's state: level 1 (a power of two, in units),
 * local_min 1, particle_t 0 and backup_t 0 (clocks in units).  The two calls below make the decisions of
 * AsyncMPM::update_dt_limits and AsyncMPM::advance (src/async/async_mpm.cpp:90-373) from that state, so that a scheduler
 * iteration needs no host work per block.
 *
 * update_dt_limits at clock t >= 0.  One pass over the particle pool as mpmb_async_block_limits; then every occupied block
 * whose level divides t (due) takes
 *   sdl = int64((strength_mul min_dt) inv_unit),  cdl = int64(((cfl_mul dx) inv_unit) (1 / sqrt(max_v2))),
 *   tmp = min(cdl, sdl, max_units)
 * (fp32, every operation rounded on its own; int64() truncates, a NaN or |x| >= 2^63 gives INT64_MIN as on x86) and halves
 * its level while tmp < level, doubles it while tmp >= 2 level and 2 level divides t.  Aligned empty blocks move the same
 * way toward the occupied blocks' max level (1 if none is occupied).  *min_level / *max_level receive the min / max level
 * over all blocks; blocks whose level is not that min set local_min to the least particle_t + level of their in-range
 * 26 neighbours (2^31 if none).  Fails, with no block state changed:
 *   MPMB_ERR_INVALID  the pool holds a particle of a type without a limit (linear, jelly) while some occupied block is due;
 *   MPMB_ERR_LIMIT    some due block has tmp < 1 (a NaN limit included).
 * max_units outside [1, 2^30], t < 0 or a NULL output: MPMB_ERR_INVALID.                                                  */
int mpmb_async_schedule(MpmbHandle h, int64_t t, float strength_mul, float cfl_mul, float dx, float inv_unit, int64_t max_units, int32_t *min_level,
                        int32_t *max_level);
/* advance(limit) at clock t: every block's flags are built from the block state, then mpmb_async_advance's steps 1-5 run
 * with dt.  EQUAL: level == limit; SWAP: EQUAL and particle_t == t; SMALLER / LARGER: level < / > limit and an in-range
 * neighbour has level == limit; CLEAR: LARGER and local_min == t + limit.  After the advance, per block: backup_t = t on
 * SWAP, particle_t = t + limit on EQUAL, backup_t = t + limit on CLEAR.  *n_gathered as mpmb_async_advance.  limit not a
 * positive power of two, t < 0, dt not positive and finite or NULL n_gathered: MPMB_ERR_INVALID.  A failed advance leaves
 * the block clocks as they were.                                                                                            */
int mpmb_async_advance_level(MpmbHandle h, int64_t t, int32_t limit, float dt, int64_t *n_gathered);
/* Copies the block state out, nb0 * nb1 * nb2 entries each in linear block order; any pointer may be NULL.  Synchronises. */
int mpmb_async_block_state(MpmbHandle h, int32_t *level, int64_t *local_min, int64_t *particle_t, int64_t *backup_t);

/* ------------------------------------------------------------------------------ profiling */
#define MPMB_N_STAGES 5 /* 0 sort+tiles, 1 P2G, 2 G2P (with the grid update), 3 exchange pack/unpack, 4 unused: 0 */
/* When enabled, CUDA events bracket every stage on the engine's stream.                          */
int mpmb_set_profiling(MpmbHandle h, int32_t enabled);
/* Accumulated milliseconds and launch counts per stage since the last reset (synchronises).      */
int mpmb_get_profile(MpmbHandle h, double ms[MPMB_N_STAGES], int64_t launches[MPMB_N_STAGES], int32_t reset);
/* Device counters: active tiles of the last substep, live particles, kernels launched so far.    */
int mpmb_get_counters(MpmbHandle h, int64_t *active_tiles, int64_t *alive, int64_t *kernel_launches);

/* State of the incremental ordering: rows of the current storage, particles that changed tile in the last substep
 * (they are holes of their old runs until the next ordering re-bins them), ghost tiles received from the neighbours. */
int mpmb_get_ordering_stats(MpmbHandle h, int64_t *rows, int64_t *movers, int64_t *ghost_tiles);

/* ------------------------------------------------------------------------------ multi-GPU */
/* z-slab runs (world>1).  The host moves the bytes; the engine packs and unpacks on the device.
 * Halo: after mpmb_rasterize, face 0 (-z) / 1 (+z) tile-layer partial sums of (p,m) are packed
 * into a device buffer of mpmb_halo_bytes() bytes; the neighbour unpacks them as ghost tiles
 * before mpmb_resample.  Migration: after mpmb_resample, particles that left the slab through a
 * face are packed (mpmb_migrate_bytes() bytes per face) and appended by the neighbour before its
 * next sort.  All pointers are DEVICE pointers owned by the caller.                               */
int64_t mpmb_halo_bytes(MpmbHandle h);
int mpmb_halo_pack(MpmbHandle h, int32_t face, void *dev_buf);
int mpmb_halo_unpack(MpmbHandle h, int32_t face, const void *dev_buf);
int64_t mpmb_migrate_bytes(MpmbHandle h);
int mpmb_migrate_pack(MpmbHandle h, int32_t face, void *dev_buf);
int mpmb_migrate_unpack(MpmbHandle h, int32_t face, const void *dev_buf);

/* Peer-memory exchange: with the neighbours' receive buffers mapped (CUDA IPC between processes, or
 * plain pointers inside one process) the engine needs no host transport at all — the pack kernels
 * store straight into the neighbour GPU over NVLink, a {count, seq} header is released system-wide
 * and the neighbour's unpack waits on it.  mpmb_substep(h, n) then runs whole z-slab substeps,
 * exchanges included, without returning to the host.
 *   kind 0 = halo arenas, kind 1 = migrating particles.  Through face f a rank writes into the
 *   neighbour's buffer of the OPPOSITE face.                                                        */
int mpmb_xchg_buffer(MpmbHandle h, int32_t kind, int32_t face, void **dev_ptr);      /* my receive buffer   */
int mpmb_xchg_ipc_handle(MpmbHandle h, int32_t kind, int32_t face, void *out64);     /* its 64-byte IPC handle */
int mpmb_xchg_connect(MpmbHandle h, int32_t kind, int32_t face, const void *handle64, void *same_process_ptr);
/* the four exchange steps of one substep, for hosts that drive the stages themselves */
int mpmb_halo_send(MpmbHandle h, int32_t face);     /* after mpmb_rasterize                      */
int mpmb_halo_recv(MpmbHandle h, int32_t face);     /* before mpmb_resample                      */
int mpmb_migrate_send(MpmbHandle h, int32_t face);  /* after mpmb_resample                       */
int mpmb_migrate_recv(MpmbHandle h, int32_t face);  /* before the next ordering                  */

/* Re-cut of a z-slab run (world > 1): the cuts move between substeps, the particles move to their new owner ranks on the
 * device and keep their ids and state bit for bit.  Contract as for the slab edits: every rank makes the three calls at
 * the same substep boundary (between two mpmb_substep calls, or after the migration of the last substep when the host
 * drives the stages); the host moves the packed records between the ranks (any rank may send to any other, so not through
 * the ring-only peer buffers; taichi_mpm_b200/slab.py uses NCCL all-to-all).  On world == 1 and inside a substep every
 * call returns MPMB_ERR_STATE.  The live rows are the rows of the current storage, immigrants of the last migration
 * included; a row's layer is the global tile layer of its base node, int(z / dx - 0.5) >> 2 in the arithmetic that decides
 * ownership.
 *
 * This rank's live rows per global tile layer: counts[n_layers], n_layers = the domain's tile layers ((res[2] + 4) / 4 + 1;
 * otherwise MPMB_ERR_INVALID).  One histogram pass on the device; n_layers counters cross the bus.  Sum over the ranks
 * for the histogram of the run.                                                                                       */
int mpmb_layer_counts(MpmbHandle h, int32_t n_layers, int64_t *counts);
/* Departing rows of the new cuts cuts[world + 1] (rank r is to own [cuts[r], cuts[r + 1]); cuts[0] = 0, cuts[world] =
 * n_layers, strictly increasing, else MPMB_ERR_INVALID): counts[world] receives, per destination rank, the live rows whose
 * layer lies in that rank's new range (0 for this rank).  With dev_buf (a DEVICE buffer of cap_rows records) they are
 * packed there, grouped by destination in ascending rank order, in storage order within a destination: deterministic.
 * A record is the migration record, the particle's N_Q = 10 raw float4 rows (160 B) as stored (the sign of a mover's mass
 * included), so ids, groups, the plastic scalar, apic_b and the cached affine matrix travel bit for bit.  More rows than
 * cap_rows: MPMB_ERR_CAPACITY, nothing written.  Read-only: the engine is unchanged until mpmb_recut_apply.            */
int mpmb_recut_pack(MpmbHandle h, const int32_t *cuts, void *dev_buf, int64_t cap_rows, int64_t *counts);
/* Re-slices this rank to own tile layers [tile_z0, tile_z1) and appends the n_in records (DEVICE memory, the layout of
 * mpmb_recut_pack) that the other ranks packed for it.  Checked first, nothing changed on failure: the range (else
 * MPMB_ERR_INVALID), every record owned under the new range (else MPMB_ERR_INVALID), a configured capacity holding the
 * kept rows plus n_in (else MPMB_ERR_CAPACITY; with capacity 0 the rows grow, keeping the migration headroom).  Then:
 * the tile grid is sized for the new slab as mpmb_create sizes it (its tile arrays grow when the slab gets thicker and
 * keep their size otherwise); the rows whose layer stays in range are kept in storage order, the others are dropped (the
 * departing rows: another rank received them); the records follow in the order given; id end = max(id end, 1 + the
 * largest id held), so the next free id of the run is unchanged; the whole set is ordered again from scratch.  Exchange
 * sequence numbers, the exchange buffers and the peers mapped into them (mpmb_xchg_connect) are untouched (their size
 * does not depend on the slab thickness): peer-connected ranks go on with mpmb_substep(h, n), whose first substep after
 * the re-cut runs outside the graph.  A rank may end with no particles.  With rigid coupling the records carry each
 * particle's colour state (see below).  AsyncMPM pools do not exist on z-slab ranks.                                    */
int mpmb_recut_apply(MpmbHandle h, int32_t tile_z0, int32_t tile_z1, int64_t n_in, const void *dev_records);

/* Rigid bodies on z-slab ranks (world > 1, after mpmb_set_rigid_samples with the same samples, bodies and states on every
 * rank).  A rank's transfers rewrite only its own tiles (those of the part being run) and sum only its own particles'
 * impulses.  After each of the two transfers of a substep (mpmb_rasterize, or both of its parts; mpmb_resample, or both of
 * its parts) every rank gathers all ranks' partial sums, adds them in rank order 0..world-1 and applies the sum; after the
 * second one device-advanced bodies take their step.  Until then the next stage returns MPMB_ERR_STATE (mpmb_resample /
 * mpmb_resample_part after the P2G transfer, mpmb_sort_particles_and_populate_grid, the slab edits, the re-cut and the
 * rigid set-up calls after either).
 * A particle's colour state (MPMParticle::states) travels with it: the migration and re-cut records carry it in row 9 .y
 * (that row holds only apic_b[8] in .x), so record sizes are unchanged, and runs without rigid coupling move the same bytes
 * as before.  The by-id colour arrays of a slab rank are indexed by ABSOLUTE id up to its id end (24 B per id per rank: state, normal + distance, mark):
 * after per-rank uploads, raise every rank's id end to the run's (the maximum of mpmb_id_end over the ranks) with
 * mpmb_append_owned_particles(n = 0, first_id = that maximum; taichi_mpm_b200/slab.py share_id_end does it, and
 * connect_peers and SlabRunner call it); an immigrant past it raises the device error flag.
 *
 * Host transport: mpmb_rigid_impulse_pack writes this rank's partial sums (mpmb_rigid_impulse_bytes bytes) into a DEVICE
 * buffer; the host all-gathers them into world consecutive blocks in rank order and every rank calls
 * mpmb_rigid_impulse_apply on that gathered buffer.                                                                    */
int64_t mpmb_rigid_impulse_bytes(MpmbHandle h);
int mpmb_rigid_impulse_pack(MpmbHandle h, void *dev_buf);
int mpmb_rigid_impulse_apply(MpmbHandle h, const void *dev_all);
/* Peer transport: every rank owns a small mailbox that every other rank maps (CUDA IPC handle between processes, the
 * pointer inside one process; mpmb_rigid_connect once per other rank).  mpmb_rigid_send stores this rank's partial sums
 * into every mailbox and releases a sequence number system-wide; mpmb_rigid_recv waits for all ranks (a bounded spin: a
 * missing peer raises the device error flag instead of hanging) and applies the sum.  With the halo peers and every
 * mailbox connected, mpmb_substep(h, n) does both reductions itself and, with device-advanced bodies, replays graphs;
 * with a mailbox unconnected it returns MPMB_ERR_STATE and enqueues nothing.  Hosts that drive the stages on one stream
 * issue every rank's mpmb_rigid_send before any rank's mpmb_rigid_recv.                                               */
int mpmb_rigid_mailbox(MpmbHandle h, void **dev_ptr);
int mpmb_rigid_mailbox_ipc_handle(MpmbHandle h, void *out64);
int mpmb_rigid_connect(MpmbHandle h, int32_t rank, const void *handle64, void *same_process_ptr);
int mpmb_rigid_send(MpmbHandle h);
int mpmb_rigid_recv(MpmbHandle h);

#ifdef __cplusplus
}
#endif
#endif /* MPMB_H_ */
