"""ctypes binding of the C-ABI in include/mpmb.h (libmpmb.so).

This is the only way Python reaches the engine: plain pointers and sizes, no torch types.
The library must exist (build.py builds it in-tree); there is NO CPU fallback — if the CUDA
library cannot be loaded, import of this module's `lib()` raises.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build

MPMB_MAX_GROUPS = 16
MPMB_MAT_PARAMS = 8
MPMB_N_STAGES = 5
MAT_LINEAR, MAT_JELLY, MAT_SNOW, MAT_WATER, MAT_SAND, MAT_ELASTIC, MAT_VON_MISES, MAT_VISCO = range(8)
MATERIAL_BY_NAME = {"linear": MAT_LINEAR, "jelly": MAT_JELLY, "snow": MAT_SNOW, "water": MAT_WATER, "sand": MAT_SAND,
                    "elastic": MAT_ELASTIC, "von_mises": MAT_VON_MISES, "visco": MAT_VISCO}

# every symbol include/mpmb.h declares
EXPORTS = [
    "mpmb_create", "mpmb_destroy", "mpmb_last_error", "mpmb_version", "mpmb_set_stream", "mpmb_synchronize",
    "mpmb_set_material", "mpmb_set_delta_t", "mpmb_set_sdf", "mpmb_set_planes", "mpmb_set_levelset_shapes", "mpmb_set_id_base",
    "mpmb_upload_particles", "mpmb_upload_aos", "mpmb_seed_lattice", "mpmb_append_particles", "mpmb_delete_inside_levelset",
    "mpmb_append_owned_particles", "mpmb_delete_owned_inside_levelset", "mpmb_id_end", "mpmb_num_particles", "mpmb_get_update_count", "mpmb_download_bgeo_points", "mpmb_download_particles", "mpmb_download_aos",
    "mpmb_substep", "mpmb_sort_particles_and_populate_grid", "mpmb_rasterize", "mpmb_resample", "mpmb_rasterize_part",
    "mpmb_resample_part", "mpmb_download_grid",
    "mpmb_set_profiling", "mpmb_get_profile", "mpmb_get_counters", "mpmb_get_ordering_stats",
    "mpmb_halo_bytes", "mpmb_halo_pack", "mpmb_halo_unpack", "mpmb_migrate_bytes", "mpmb_migrate_pack", "mpmb_migrate_unpack",
    "mpmb_set_rigid_samples", "mpmb_set_rigid_coupling", "mpmb_set_rigid_state", "mpmb_get_rigid_state", "mpmb_set_rigid_motion",
    "mpmb_set_rigid_script", "mpmb_set_particle_states",
    "mpmb_get_particle_cdf", "mpmb_download_cdf",
    "mpmb_xchg_buffer", "mpmb_xchg_ipc_handle", "mpmb_xchg_connect", "mpmb_halo_send", "mpmb_halo_recv", "mpmb_migrate_send", "mpmb_migrate_recv",
    "mpmb_async_init", "mpmb_async_add", "mpmb_async_block_limits", "mpmb_async_advance", "mpmb_async_size", "mpmb_async_download",
    "mpmb_async_schedule", "mpmb_async_advance_level", "mpmb_async_block_state",
    "mpmb_layer_counts", "mpmb_recut_pack", "mpmb_recut_apply",
    "mpmb_rigid_impulse_bytes", "mpmb_rigid_impulse_pack", "mpmb_rigid_impulse_apply", "mpmb_rigid_mailbox", "mpmb_rigid_mailbox_ipc_handle",
    "mpmb_rigid_connect", "mpmb_rigid_send", "mpmb_rigid_recv",
]
ASYNC_SMALLER, ASYNC_EQUAL, ASYNC_LARGER, ASYNC_SWAP, ASYNC_CLEAR = 1, 2, 4, 8, 16   # per-block flags of mpmb_async_advance
ERR_INVALID, ERR_LIMIT = -1, -5   # MPMB_ERR_INVALID; MPMB_ERR_LIMIT: a due block's time-step limit is below one unit
RECORD_BYTES = 160   # one particle record of mpmb_recut_pack / mpmb_recut_apply (and of the migration messages)


class MpmbConfig(C.Structure):
    _fields_ = [
        ("res", C.c_int32 * 3),
        ("dx", C.c_float),
        ("dt", C.c_float),
        ("gravity", C.c_float * 3),
        ("particle_gravity", C.c_int32),
        ("clean_boundary", C.c_int32),
        ("device", C.c_int32),
        ("capacity", C.c_int64),
        ("rank", C.c_int32),
        ("world", C.c_int32),
        ("tile_z0", C.c_int32),
        ("tile_z1", C.c_int32),
        ("migrate_capacity", C.c_int64),
        ("halo_capacity", C.c_int32),
        ("no_graph", C.c_int32),
        ("dim", C.c_int32),
        ("apic_damping", C.c_float),
        ("rpic_damping", C.c_float),
        ("reserved", C.c_int32 * 3),
    ]


class MpmbAosLayout(C.Structure):
    _fields_ = [
        ("stride", C.c_int32), ("off_pos", C.c_int32), ("off_v_and_m", C.c_int32), ("off_dg_e", C.c_int32),
        ("off_apic_b", C.c_int32), ("col_pitch", C.c_int32), ("off_vol", C.c_int32), ("off_scalar", C.c_int32),
        ("off_scalar_by_kind", C.c_int32 * 4),
    ]

    # the material kinds that keep a plastic scalar, in the order of off_scalar_by_kind (snow Jp, water j, sand logJp, visco_tau)
    SCALAR_KINDS = (2, 3, 4, 7)

    def set_scalar_offsets(self, by_kind):
        """Per-kind plastic-scalar offsets for a pool that mixes particle types: `by_kind` maps a material kind (scenes.MAT_*) to
        the byte offset of its scalar in the slot.  Kinds left out get -1 (no scalar in the slot: the upload's default);
        off_scalar becomes -1.  A kind without a plastic scalar is an error."""
        bad = set(by_kind) - set(self.SCALAR_KINDS)
        if bad:
            raise ValueError("kinds without a plastic scalar: %s" % sorted(bad))
        self.off_scalar = -1
        self.off_scalar_by_kind[:] = [int(by_kind.get(k, -1)) for k in self.SCALAR_KINDS]
        return self


class MpmbShape(C.Structure):
    _fields_ = [("kind", C.c_int32), ("inside_out", C.c_int32), ("p", C.c_float * 6)]


class MpmbRigidBody(C.Structure):
    _fields_ = [("position", C.c_float * 3), ("rot", C.c_float * 9), ("velocity", C.c_float * 3), ("angular_velocity", C.c_float * 3),
                ("inv_mass", C.c_float), ("inv_inertia", C.c_float * 9), ("frictions", C.c_float * 2)]


class MpmbRigidMotion(C.Structure):
    _fields_ = [("mass", C.c_float), ("inv_inertia_body", C.c_float * 9), ("rotation_axis", C.c_float * 3), ("linear_damping", C.c_float),
                ("angular_damping", C.c_float), ("restitution", C.c_float), ("scripted_position", C.c_int32), ("scripted_rotation", C.c_int32),
                ("reserved", C.c_int32 * 4)]


RIGID_SCRIPT_STRIDE = 18   # position, rotation (column-major), velocity, angular velocity per body and substep


SHAPE_PLANE, SHAPE_SPHERE, SHAPE_CUBOID = range(3)
_LIB = None


def lib_path():
    """The product library, or the A/B variant named by MPMB_LIB (a build of the same source with
    experiment defines, `python -m taichi_mpm_b200.build --define ...`; kernel tuning only)."""
    return os.environ.get("MPMB_LIB") or _build.LIB


def lib():
    """Loads libmpmb.so (building it in-tree if the source is newer).  Raises if unavailable."""
    global _LIB
    if _LIB is None:
        path = _build.build()
        if os.environ.get("MPMB_LIB"):
            path = os.environ["MPMB_LIB"]
        if not os.path.exists(path):
            raise RuntimeError("libmpmb.so is missing: the CUDA engine has not been built (python -m taichi_mpm_b200.build)")
        L = C.CDLL(path)
        L.mpmb_last_error.restype = C.c_char_p
        L.mpmb_last_error.argtypes = [C.c_void_p]
        L.mpmb_halo_bytes.restype = C.c_int64
        L.mpmb_migrate_bytes.restype = C.c_int64
        L.mpmb_halo_bytes.argtypes = [C.c_void_p]
        L.mpmb_migrate_bytes.argtypes = [C.c_void_p]
        L.mpmb_rigid_impulse_bytes.restype = C.c_int64
        L.mpmb_rigid_impulse_bytes.argtypes = [C.c_void_p]
        L.mpmb_create.argtypes = [C.POINTER(MpmbConfig), C.POINTER(C.c_void_p)]
        for name in EXPORTS:
            getattr(L, name)  # AttributeError if a declared symbol is not exported
        _LIB = L
    return _LIB


class MpmbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("mpmb error %d: %s" % (code, msg))
        self.code = code


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(a, shape=None):
    if a is None:
        return None
    a = np.ascontiguousarray(a, np.float32)
    if shape is not None:
        a = a.reshape(shape)
    return a


class Engine:
    """Thin object wrapper over one MpmbHandle."""

    def __init__(self, res, dx, dt, gravity=(0.0, -10.0, 0.0), particle_gravity=True, clean_boundary=True, device=0,
                 capacity=0, rank=0, world=1, tile_z0=0, tile_z1=0, migrate_capacity=0, halo_capacity=0, no_graph=False, dim=0,
                 apic_damping=0.0, rpic_damping=0.0):
        self.L = lib()
        cfg = MpmbConfig()
        if np.isscalar(res):
            res = (res, res, res)
        cfg.res[:] = [int(r) for r in res] + [0] * (3 - len(res))
        cfg.dim = int(dim)
        cfg.apic_damping, cfg.rpic_damping = float(apic_damping), float(rpic_damping)
        cfg.dx, cfg.dt = float(dx), float(dt)
        cfg.gravity[:] = [float(g) for g in gravity] + [0.0] * (3 - len(gravity))
        cfg.particle_gravity = int(bool(particle_gravity))
        cfg.clean_boundary = int(bool(clean_boundary))
        cfg.device = int(device)
        cfg.capacity = int(capacity)
        cfg.rank, cfg.world, cfg.tile_z0, cfg.tile_z1 = int(rank), int(world), int(tile_z0), int(tile_z1)
        cfg.migrate_capacity = int(migrate_capacity)
        cfg.halo_capacity = int(halo_capacity)
        cfg.no_graph = int(bool(no_graph))
        self.res = tuple(int(r) for r in res)
        self.cfg = cfg
        self.h = C.c_void_p()
        rc = self.L.mpmb_create(C.byref(cfg), C.byref(self.h))
        if rc != 0:
            raise MpmbError(rc, self.L.mpmb_last_error(None).decode())

    def _check(self, rc):
        if rc != 0:
            raise MpmbError(rc, self.L.mpmb_last_error(self.h).decode())

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            self.L.mpmb_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- scene
    def set_stream(self, cuda_stream):
        self._check(self.L.mpmb_set_stream(self.h, C.c_void_p(int(cuda_stream))))

    def synchronize(self):
        self._check(self.L.mpmb_synchronize(self.h))

    def set_material(self, group, kind, params):
        p = np.zeros(MPMB_MAT_PARAMS, np.float32)
        p[: len(params)] = params
        self._check(self.L.mpmb_set_material(self.h, C.c_int32(group), C.c_int32(kind), _ptr(p), C.c_int32(len(params))))

    def set_delta_t(self, dt):
        self._check(self.L.mpmb_set_delta_t(self.h, C.c_float(float(dt))))

    def set_sdf(self, sdf4, friction):
        if sdf4 is not None:
            sdf4 = _f32(sdf4)
            assert sdf4.shape == tuple(r + 1 for r in self.res) + (4,)
        self._check(self.L.mpmb_set_sdf(self.h, _ptr(sdf4), C.c_float(friction)))

    def set_planes(self, planes4, friction):
        planes4 = _f32(planes4).reshape(-1, 4)
        self._check(self.L.mpmb_set_planes(self.h, C.c_int32(len(planes4)), _ptr(planes4), C.c_float(friction)))

    def set_levelset_shapes(self, shapes, friction):
        """shapes: [(kind, inside_out, params[<=6])] in GRID units (mpmb.h)."""
        arr = (MpmbShape * len(shapes))()
        for k, (kind, io, prm) in enumerate(shapes):
            arr[k].kind, arr[k].inside_out = int(kind), int(bool(io))
            for j, v in enumerate(prm):
                arr[k].p[j] = float(v)
        self._check(self.L.mpmb_set_levelset_shapes(self.h, C.c_int32(len(shapes)), arr, C.c_float(friction)))

    def set_id_base(self, base):
        self._check(self.L.mpmb_set_id_base(self.h, C.c_int64(int(base))))

    # --- particles
    def upload(self, x, v, mass, vol, F=None, b=None, scalar=None, group=None):
        x = _f32(x).reshape(-1, 3)
        n = len(x)
        v, F, b = _f32(v, (n, 3)), _f32(F, (n, 9)), _f32(b, (n, 9))
        mass, vol, scalar = _f32(mass, (n,)), _f32(vol, (n,)), _f32(scalar, (n,))
        group = None if group is None else np.ascontiguousarray(group, np.int32).reshape(n)
        self._check(self.L.mpmb_upload_particles(self.h, C.c_int64(n), _ptr(x), _ptr(v), _ptr(F), _ptr(b), _ptr(mass), _ptr(vol),
                                                 _ptr(scalar), _ptr(group)))

    def append(self, x, v, mass, vol, F=None, b=None, scalar=None, group=None):
        """Adds particles to the resident set; resident particles keep their ids and state.  Returns the first new id
        (the new ones are numbered consecutively after every id handed out so far)."""
        x = _f32(x).reshape(-1, 3)
        n = len(x)
        v, F, b = _f32(v, (n, 3)), _f32(F, (n, 9)), _f32(b, (n, 9))
        mass, vol, scalar = _f32(mass, (n,)), _f32(vol, (n,)), _f32(scalar, (n,))
        group = None if group is None else np.ascontiguousarray(group, np.int32).reshape(n)
        first = C.c_int64(0)
        self._check(self.L.mpmb_append_particles(self.h, C.c_int64(n), _ptr(x), _ptr(v), _ptr(F), _ptr(b), _ptr(mass), _ptr(vol),
                                                 _ptr(scalar), _ptr(group), C.byref(first)))
        return first.value

    def delete_inside_levelset(self):
        """Removes the particles where the level set is negative (delete_particles_inside_level_set); returns how many."""
        n = C.c_int64(0)
        self._check(self.L.mpmb_delete_inside_levelset(self.h, C.byref(n)))
        return n.value

    def append_owned(self, x, v, mass, vol, F=None, b=None, scalar=None, group=None, *, first_id):
        """Appends the particles of a batch that this engine owns (z-slab ranks: base node in its tile layers; world == 1:
        every in-domain one), particle k with id first_id + k.  Every rank of a run gets the same batch and first_id, at
        least the maximum of id_end() over the ranks (slab.global_id_end).  Returns how many this engine kept."""
        x = _f32(x).reshape(-1, 3)
        n = len(x)
        v, F, b = _f32(v, (n, 3)), _f32(F, (n, 9)), _f32(b, (n, 9))
        mass, vol, scalar = _f32(mass, (n,)), _f32(vol, (n,)), _f32(scalar, (n,))
        group = None if group is None else np.ascontiguousarray(group, np.int32).reshape(n)
        kept = C.c_int64(0)
        self._check(self.L.mpmb_append_owned_particles(self.h, C.c_int64(n), _ptr(x), _ptr(v), _ptr(F), _ptr(b), _ptr(mass), _ptr(vol),
                                                       _ptr(scalar), _ptr(group), C.c_int64(int(first_id)), C.byref(kept)))
        return kept.value

    def delete_owned_inside_levelset(self):
        """Removes this engine's particles where the level set is negative (any world); returns how many."""
        n = C.c_int64(0)
        self._check(self.L.mpmb_delete_owned_inside_levelset(self.h, C.byref(n)))
        return n.value

    def id_end(self):
        """End of the ids handed out so far (absolute); the next free id of a z-slab run is the maximum over its ranks."""
        n = C.c_int64(0)
        self._check(self.L.mpmb_id_end(self.h, C.byref(n)))
        return n.value

    def upload_ptrs(self, n, x, v, F, b, mass, vol, scalar, group):
        """Raw-pointer variant (ints), e.g. pinned host buffers owned by the caller."""
        vp = lambda p: C.c_void_p(p) if p else None
        self._check(self.L.mpmb_upload_particles(self.h, C.c_int64(n), vp(x), vp(v), vp(F), vp(b), vp(mass), vp(vol), vp(scalar), vp(group)))

    def download_ptrs(self, cap, id_, x, v, F, b, mass, vol, scalar, group):
        vp = lambda p: C.c_void_p(p) if p else None
        n = C.c_int64(0)
        self._check(self.L.mpmb_download_particles(self.h, C.c_int64(cap), C.byref(n), vp(id_), vp(x), vp(v), vp(F), vp(b), vp(mass),
                                                   vp(vol), vp(scalar), vp(group)))
        return n.value

    def seed_lattice(self, lo_cell, hi_cell, vol, mass, jitter=0.0, seed=0, group=0, v0=(0.0, 0.0, 0.0)):
        """Device-side `benchmark` lattice (src/mpm.cpp:149-186); returns the number of particles this engine created."""
        lo = (C.c_int32 * 3)(*[int(v) for v in lo_cell])
        hi = (C.c_int32 * 3)(*[int(v) for v in hi_cell])
        vv = (C.c_float * 3)(*[float(v) for v in v0])
        n = C.c_int64(0)
        self._check(self.L.mpmb_seed_lattice(self.h, lo, hi, C.c_float(vol), C.c_float(mass), C.c_float(jitter), C.c_uint32(int(seed)),
                                             C.c_int32(group), vv, C.byref(n)))
        return n.value

    def upload_aos(self, pool, indices, layout, group=None):
        pool = np.ascontiguousarray(pool, np.uint8)
        indices = np.ascontiguousarray(indices, np.uint32)
        slots = pool.size // layout.stride
        group = None if group is None else np.ascontiguousarray(group, np.int32)
        self._check(self.L.mpmb_upload_aos(self.h, C.c_int64(len(indices)), _ptr(pool), C.c_int64(slots), _ptr(indices), C.byref(layout),
                                           _ptr(group)))

    def download_aos(self, pool, indices, layout):
        assert pool.dtype == np.uint8 and pool.flags.c_contiguous and indices.dtype == np.uint32
        n = C.c_int64(0)
        self._check(self.L.mpmb_download_aos(self.h, _ptr(pool), C.c_int64(pool.size // layout.stride), _ptr(indices), C.c_int64(len(indices)),
                                             C.byref(layout), C.byref(n)))
        return n.value

    def num_particles(self):
        n = C.c_int64(0)
        self._check(self.L.mpmb_num_particles(self.h, C.byref(n)))
        return n.value

    def download_bgeo_points(self, id_range, cap=None):
        """Device-packed BGEO point block (48 big-endian bytes per particle, id order): (n, bytes ndarray)."""
        if cap is None:
            cap = max(self.num_particles(), 1)
        buf = np.empty(cap * 48, np.uint8)
        n = C.c_int64(0)
        self._check(self.L.mpmb_download_bgeo_points(self.h, C.c_int64(int(id_range)), _ptr(buf), C.c_int64(cap), C.byref(n)))
        return n.value, buf[: n.value * 48]

    def update_count(self):
        """Particle updates so far, as the reference's update_counter counts them (src/mpm.cpp:436)."""
        n = C.c_int64(0)
        self._check(self.L.mpmb_get_update_count(self.h, C.byref(n)))
        return n.value

    def download(self, cap=None, sort_by_id=True):
        """Returns dict(id,x,v,F,b,mass,vol,ps,group) of the live particles."""
        if cap is None:
            cap = max(self.num_particles(), 1)
        out = dict(id=np.zeros(cap, np.uint32), x=np.zeros((cap, 3), np.float32), v=np.zeros((cap, 3), np.float32),
                   F=np.zeros((cap, 9), np.float32), b=np.zeros((cap, 9), np.float32), mass=np.zeros(cap, np.float32),
                   vol=np.zeros(cap, np.float32), ps=np.zeros(cap, np.float32), group=np.zeros(cap, np.int32))
        n = C.c_int64(0)
        self._check(self.L.mpmb_download_particles(self.h, C.c_int64(cap), C.byref(n), _ptr(out["id"]), _ptr(out["x"]), _ptr(out["v"]),
                                                   _ptr(out["F"]), _ptr(out["b"]), _ptr(out["mass"]), _ptr(out["vol"]), _ptr(out["ps"]),
                                                   _ptr(out["group"])))
        out = {k: a[: n.value] for k, a in out.items()}
        if sort_by_id:
            o = np.argsort(out["id"], kind="stable")
            out = {k: a[o] for k, a in out.items()}
        return out

    # --- AsyncMPM pools (mpmb_async_*): which = 0 particle pool, 1 backup pool
    def async_init(self, nb, inv_dx):
        """Empties both pools; nb = scheduler blocks per axis, inv_dx = the host's float32(1 / dx)."""
        self._async_nb = tuple(int(n) for n in nb)
        self._check(self.L.mpmb_async_init(self.h, (C.c_int32 * 3)(*self._async_nb), C.c_float(float(inv_dx))))

    def async_add(self, which, rec):
        """Appends records dict(x, v, F, b, mass, vol, ps, group, id) to a pool; their blocks come from x."""
        x = _f32(rec["x"]).reshape(-1, 3)
        n = len(x)
        v, F, b = _f32(rec["v"], (n, 3)), _f32(rec["F"], (n, 9)), _f32(rec["b"], (n, 9))
        mass, vol, ps = _f32(rec["mass"], (n,)), _f32(rec["vol"], (n,)), _f32(rec["ps"], (n,))
        group = np.ascontiguousarray(rec["group"], np.int32).reshape(n)
        ids = np.ascontiguousarray(rec["id"], np.uint32).reshape(n)
        self._check(self.L.mpmb_async_add(self.h, C.c_int32(which), C.c_int64(n), _ptr(x), _ptr(v), _ptr(F), _ptr(b), _ptr(mass), _ptr(vol),
                                          _ptr(ps), _ptr(group), _ptr(ids)))

    def async_block_limits(self, with_limits):
        """Occupied blocks of the particle pool (linear indices, ascending) and, with limits, their min(0.1, allowed_dt) and
        max |v|^2 (else None): (block, min_dt, max_v2)."""
        cap = int(np.prod(self._async_nb))
        blk = np.empty(cap, np.int32)
        mn = np.empty(cap, np.float32) if with_limits else None
        mx = np.empty(cap, np.float32) if with_limits else None
        n = C.c_int64(0)
        self._check(self.L.mpmb_async_block_limits(self.h, C.c_int32(int(bool(with_limits))), C.c_int64(cap), C.byref(n), _ptr(blk), _ptr(mn), _ptr(mx)))
        k = n.value
        return blk[:k], None if mn is None else mn[:k], None if mx is None else mx[:k]

    def async_advance(self, flags, dt):
        """One AsyncMPM advance; flags = uint8 ASYNC_* bits per block (C order of the block grid).  Returns the gathered count."""
        fl = np.ascontiguousarray(flags, np.uint8).reshape(-1)
        assert fl.size == int(np.prod(self._async_nb))
        n = C.c_int64(0)
        self._check(self.L.mpmb_async_advance(self.h, _ptr(fl), C.c_float(float(dt)), C.byref(n)))
        return n.value

    def async_size(self):
        a, b = C.c_int64(0), C.c_int64(0)
        self._check(self.L.mpmb_async_size(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def async_download(self, which, fields=("id", "block", "x", "v", "F", "b", "mass", "vol", "ps", "group")):
        """A pool in pool order: dict of the asked fields (id uint32, block = linear block index int32)."""
        n = self.async_size()[which]
        shape = dict(id=((), np.uint32), block=((), np.int32), x=((3,), np.float32), v=((3,), np.float32), F=((9,), np.float32),
                     b=((9,), np.float32), mass=((), np.float32), vol=((), np.float32), ps=((), np.float32), group=((), np.int32))
        out = {k: np.empty((n,) + shape[k][0], shape[k][1]) for k in fields}
        got = C.c_int64(0)
        self._check(self.L.mpmb_async_download(self.h, C.c_int32(which), C.c_int64(n), C.byref(got), *[_ptr(out.get(k)) for k in (
            "id", "block", "x", "v", "F", "b", "mass", "vol", "ps", "group")]))
        return out

    # --- AsyncMPM's block scheduler on the device: block state level / local_min / particle_t / backup_t
    def async_schedule(self, t, strength_mul, cfl_mul, dx, inv_unit, max_units):
        """update_dt_limits at clock t (the float32 scalars as the host scheduler rounds them).  Returns (min level, max level)."""
        lo, hi = C.c_int32(0), C.c_int32(0)
        self._check(self.L.mpmb_async_schedule(self.h, C.c_int64(int(t)), C.c_float(float(strength_mul)), C.c_float(float(cfl_mul)),
                                               C.c_float(float(dx)), C.c_float(float(inv_unit)), C.c_int64(int(max_units)), C.byref(lo), C.byref(hi)))
        return lo.value, hi.value

    def async_advance_level(self, t, limit, dt):
        """advance(limit) at clock t with the flags built on the device.  Returns the gathered count."""
        n = C.c_int64(0)
        self._check(self.L.mpmb_async_advance_level(self.h, C.c_int64(int(t)), C.c_int32(int(limit)), C.c_float(float(dt)), C.byref(n)))
        return n.value

    def async_block_state(self, fields=("level", "local_min", "particle_t", "backup_t")):
        """The asked block state arrays, int64 of shape nb."""
        nb = self._async_nb
        out = {k: np.empty(nb, np.int32 if k == "level" else np.int64) for k in fields}
        self._check(self.L.mpmb_async_block_state(self.h, *[_ptr(out.get(k)) for k in ("level", "local_min", "particle_t", "backup_t")]))
        return {k: v.astype(np.int64) for k, v in out.items()}

    # --- hot path
    def substep(self, nsub=1):
        self._check(self.L.mpmb_substep(self.h, C.c_int32(nsub)))

    # ---- rigid bodies (CPIC): `rigid` is the dict scenes.make_rigid builds (row 0 = the background body)
    def _rigid_records(self, rigid):
        nb = len(rigid["inv_mass"])
        arr = (MpmbRigidBody * nb)()
        for b in range(nb):
            arr[b].position[:] = [float(v) for v in rigid["position"][b]]
            arr[b].rot[:] = [float(v) for v in np.asarray(rigid["rot"][b]).reshape(9)]
            arr[b].velocity[:] = [float(v) for v in rigid["velocity"][b]]
            arr[b].angular_velocity[:] = [float(v) for v in rigid["angular_velocity"][b]]
            arr[b].inv_mass = float(rigid["inv_mass"][b])
            arr[b].inv_inertia[:] = [float(v) for v in np.asarray(rigid["inv_inertia"][b]).reshape(9)]
            arr[b].frictions[:] = [float(v) for v in rigid["frictions"][b]]
        return nb, arr

    def set_rigid(self, rigid):
        """Boundary samples + coupling constants + the current state of every body."""
        off, tri = _f32(rigid["sample_offset"], (-1, 3)), _f32(rigid["sample_tri"], (-1, 9))
        rid = np.ascontiguousarray(rigid["sample_rigid"], np.int32)
        self._check(self.L.mpmb_set_rigid_samples(self.h, C.c_int32(len(rigid["inv_mass"])), C.c_int64(len(rid)), _ptr(off), _ptr(tri), _ptr(rid)))
        self.rigid_coupled = len(rid) > 0
        if len(rid):
            self._check(self.L.mpmb_set_rigid_coupling(self.h, C.c_float(rigid.get("penalty", 0.0)), C.c_float(rigid.get("pushing_force", 20000.0))))
            self.set_rigid_state(rigid)

    def set_rigid_state(self, rigid):
        nb, arr = self._rigid_records(rigid)
        self._check(self.L.mpmb_set_rigid_state(self.h, C.c_int32(nb), arr))

    def get_rigid_state(self, n_bodies):
        arr = (MpmbRigidBody * n_bodies)()
        self._check(self.L.mpmb_get_rigid_state(self.h, C.c_int32(n_bodies), arr))
        # rot and inv_inertia also column-major flattened, the layout of scenes.make_rigid (what the next substep reads)
        return dict(velocity=np.array([list(a.velocity) for a in arr], np.float32), angular_velocity=np.array([list(a.angular_velocity) for a in arr], np.float32),
                    position=np.array([list(a.position) for a in arr], np.float32),
                    rotation=np.array([np.reshape(list(a.rot), (3, 3)).T for a in arr], np.float32),
                    rot=np.array([list(a.rot) for a in arr], np.float32), inv_mass=np.array([a.inv_mass for a in arr], np.float32),
                    inv_inertia=np.array([list(a.inv_inertia) for a in arr], np.float32), frictions=np.array([list(a.frictions) for a in arr], np.float32))

    def set_rigid_motion(self, motion, levelset_collision=False):
        """Device advection of the bodies (mpmb_set_rigid_motion).  motion: one dict per body, row 0 = the background body
        (ignored), with mass, inv_inertia_body (3x3, body frame), rotation_axis, linear_damping, angular_damping, restitution,
        scripted_position, scripted_rotation; missing keys are 0.  An empty list switches device advection off."""
        nb = len(motion)
        arr = (MpmbRigidMotion * max(nb, 1))()
        for b, m in enumerate(motion):
            arr[b].mass = float(m.get("mass", 0.0))
            arr[b].inv_inertia_body[:] = [float(v) for v in np.asarray(m.get("inv_inertia_body", np.zeros((3, 3))), np.float64).T.reshape(9)]
            arr[b].rotation_axis[:] = [float(v) for v in m.get("rotation_axis", (0.0, 0.0, 0.0))]
            arr[b].linear_damping = float(m.get("linear_damping", 0.0))
            arr[b].angular_damping = float(m.get("angular_damping", 0.0))
            arr[b].restitution = float(m.get("restitution", 0.0))
            arr[b].scripted_position = int(bool(m.get("scripted_position", False)))
            arr[b].scripted_rotation = int(bool(m.get("scripted_rotation", False)))
        self._check(self.L.mpmb_set_rigid_motion(self.h, C.c_int32(nb), arr, C.c_int32(int(bool(levelset_collision)))))

    def set_rigid_script(self, poses):
        """poses[n_substeps][n_bodies][18] (float64): position, rotation (3x3 flattened column-major), velocity, angular
        velocity at the end of each substep; only the scripted parts are read."""
        poses = np.ascontiguousarray(poses, np.float64)
        n = poses.shape[0] if poses.ndim == 3 else 0
        self._check(self.L.mpmb_set_rigid_script(self.h, C.c_int32(n), _ptr(poses)))

    def set_particle_states(self, states):
        st = np.ascontiguousarray(states, np.uint32)
        self._check(self.L.mpmb_set_particle_states(self.h, C.c_int64(len(st)), _ptr(st)))

    def get_particle_cdf(self, n):
        out = dict(states=np.zeros(n, np.uint32), bnormal=np.zeros((n, 3), np.float32), bdist=np.zeros(n, np.float32), near=np.zeros(n, np.uint8))
        self._check(self.L.mpmb_get_particle_cdf(self.h, C.c_int64(n), _ptr(out["states"]), _ptr(out["bnormal"]), _ptr(out["bdist"]), _ptr(out["near"])))
        return out

    def download_cdf(self):
        nn = tuple(r + 1 for r in self.res)
        st, d = np.zeros(nn, np.uint32), np.zeros(nn, np.float32)
        self._check(self.L.mpmb_download_cdf(self.h, _ptr(st), _ptr(d)))
        return dict(node_state=st, node_dist=d)

    def sort_particles_and_populate_grid(self):
        self._check(self.L.mpmb_sort_particles_and_populate_grid(self.h))

    def rasterize(self):
        self._check(self.L.mpmb_rasterize(self.h))

    def resample(self):
        self._check(self.L.mpmb_resample(self.h))

    def rasterize_part(self, part):
        self._check(self.L.mpmb_rasterize_part(self.h, C.c_int32(part)))

    def resample_part(self, part):
        self._check(self.L.mpmb_resample_part(self.h, C.c_int32(part)))

    def download_grid(self, which):
        g = np.zeros(tuple(r + 1 for r in self.res) + (4,), np.float32)
        self._check(self.L.mpmb_download_grid(self.h, C.c_int32(which), _ptr(g)))
        return g

    # --- z-slab exchange (device pointers owned by the caller)
    def halo_bytes(self):
        return int(self.L.mpmb_halo_bytes(self.h))

    def migrate_bytes(self):
        return int(self.L.mpmb_migrate_bytes(self.h))

    def halo_pack(self, face, dev_ptr):
        self._check(self.L.mpmb_halo_pack(self.h, C.c_int32(face), C.c_void_p(int(dev_ptr))))

    def halo_unpack(self, face, dev_ptr):
        self._check(self.L.mpmb_halo_unpack(self.h, C.c_int32(face), C.c_void_p(int(dev_ptr))))

    def migrate_pack(self, face, dev_ptr):
        self._check(self.L.mpmb_migrate_pack(self.h, C.c_int32(face), C.c_void_p(int(dev_ptr))))

    def migrate_unpack(self, face, dev_ptr):
        self._check(self.L.mpmb_migrate_unpack(self.h, C.c_int32(face), C.c_void_p(int(dev_ptr))))

    # --- peer-memory exchange
    def xchg_buffer(self, kind, face):
        p = C.c_void_p()
        self._check(self.L.mpmb_xchg_buffer(self.h, C.c_int32(kind), C.c_int32(face), C.byref(p)))
        return p.value

    def xchg_ipc_handle(self, kind, face):
        buf = (C.c_ubyte * 64)()
        self._check(self.L.mpmb_xchg_ipc_handle(self.h, C.c_int32(kind), C.c_int32(face), buf))
        return bytes(buf)

    def xchg_connect(self, kind, face, handle=None, ptr=None):
        hb = (C.c_ubyte * 64).from_buffer_copy(handle) if handle is not None else None
        self._check(self.L.mpmb_xchg_connect(self.h, C.c_int32(kind), C.c_int32(face), hb, C.c_void_p(ptr) if ptr else None))

    def halo_send(self, face):
        self._check(self.L.mpmb_halo_send(self.h, C.c_int32(face)))

    def halo_recv(self, face):
        self._check(self.L.mpmb_halo_recv(self.h, C.c_int32(face)))

    def migrate_send(self, face):
        self._check(self.L.mpmb_migrate_send(self.h, C.c_int32(face)))

    def migrate_recv(self, face):
        self._check(self.L.mpmb_migrate_recv(self.h, C.c_int32(face)))

    # --- rigid impulses of z-slab ranks: summed over the ranks after each transfer
    def rigid_impulse_bytes(self):
        return int(self.L.mpmb_rigid_impulse_bytes(self.h))

    def rigid_impulse_pack(self, dev_ptr):
        """This rank's partial impulse sums of the last transfer into a device buffer of rigid_impulse_bytes()."""
        self._check(self.L.mpmb_rigid_impulse_pack(self.h, C.c_void_p(int(dev_ptr))))

    def rigid_impulse_apply(self, dev_ptr):
        """Sums the world ranks' partials (consecutive blocks in rank order, device memory) and applies them."""
        self._check(self.L.mpmb_rigid_impulse_apply(self.h, C.c_void_p(int(dev_ptr))))

    def rigid_mailbox(self):
        p = C.c_void_p()
        self._check(self.L.mpmb_rigid_mailbox(self.h, C.byref(p)))
        return p.value

    def rigid_mailbox_ipc_handle(self):
        buf = (C.c_ubyte * 64)()
        self._check(self.L.mpmb_rigid_mailbox_ipc_handle(self.h, buf))
        return bytes(buf)

    def rigid_connect(self, rank, handle=None, ptr=None):
        hb = (C.c_ubyte * 64).from_buffer_copy(handle) if handle is not None else None
        self._check(self.L.mpmb_rigid_connect(self.h, C.c_int32(rank), hb, C.c_void_p(ptr) if ptr else None))

    def rigid_send(self):
        self._check(self.L.mpmb_rigid_send(self.h))

    def rigid_recv(self):
        self._check(self.L.mpmb_rigid_recv(self.h))

    # --- re-cut of a z-slab run (device buffers: anything with data_ptr(), numel() and element_size(), e.g. torch tensors)
    def tile_range(self):
        """The tile layers [tile_z0, tile_z1) this engine owns now."""
        return int(self.cfg.tile_z0), int(self.cfg.tile_z1)

    def layer_counts(self):
        """This engine's live particles per tile layer of the whole domain (int64 array)."""
        out = np.zeros((self.res[2] + 4) // 4 + 1, np.int64)
        self._check(self.L.mpmb_layer_counts(self.h, C.c_int32(len(out)), _ptr(out)))
        return out

    def recut_pack(self, cuts, buf=None):
        """Departing particles of the new cuts (world + 1 tile layers, rank r owns [cuts[r], cuts[r + 1])): their number per
        destination rank; with `buf` also packed there (RECORD_BYTES each, by destination in rank order).  Changes nothing."""
        cuts = np.ascontiguousarray(cuts, np.int32)
        counts = np.zeros(len(cuts) - 1, np.int64)
        ptr, cap = (None, 0) if buf is None else (C.c_void_p(buf.data_ptr()), buf.numel() * buf.element_size() // RECORD_BYTES)
        self._check(self.L.mpmb_recut_pack(self.h, _ptr(cuts), ptr, C.c_int64(cap), _ptr(counts)))
        return counts

    def recut_apply(self, z0, z1, buf, n_in):
        """Owns tile layers [z0, z1) from now on: keeps the particles that stay, appends the n_in records of `buf`."""
        ptr = C.c_void_p(buf.data_ptr()) if buf is not None and n_in > 0 else None
        self._check(self.L.mpmb_recut_apply(self.h, C.c_int32(int(z0)), C.c_int32(int(z1)), C.c_int64(int(n_in)), ptr))
        self.cfg.tile_z0, self.cfg.tile_z1 = int(z0), int(z1)

    # --- profiling
    def set_profiling(self, enabled):
        self._check(self.L.mpmb_set_profiling(self.h, C.c_int32(int(enabled))))

    def get_profile(self, reset=True):
        ms = (C.c_double * MPMB_N_STAGES)()
        ln = (C.c_int64 * MPMB_N_STAGES)()
        self._check(self.L.mpmb_get_profile(self.h, ms, ln, C.c_int32(int(reset))))
        return list(ms), list(ln)

    def get_ordering_stats(self):
        a, b, c = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        self._check(self.L.mpmb_get_ordering_stats(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(rows=a.value, movers=b.value, ghost_tiles=c.value)

    def debug_check(self):
        """Bounds-checked builds only (-DMPMB_CHECKED, build.CHECKED_LIB): [site, a, b, c] of the first index check that
        failed (site 0: none failed), then n_store, n_alive, n_movers, n_tiles."""
        f = getattr(self.L, "mpmb_debug_check", None)
        if f is None:
            raise RuntimeError("mpmb_debug_check is exported by the bounds-checked build only")
        out = (C.c_int32 * 8)()
        self._check(f(self.h, out))
        return list(out)

    def get_counters(self):
        a, b, c = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        self._check(self.L.mpmb_get_counters(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(active_tiles=a.value, alive=b.value, kernel_launches=c.value)


class Engine2D(Engine):
    """A 2-D handle (MpmbConfig.dim = 2, MPM<2>): res = (r0, r1), gravity = (g_x, g_y); particle arrays are dim-packed
    (x, v [n, 2]; F, b [n, 4] column-major) and dense node arrays are (r0 + 1, r1 + 1, 4) with the z component 0.  The
    entry points include/mpmb.h lists for dim = 2 work; every other method returns the engine's error."""

    def __init__(self, res, dx, dt, gravity=(0.0, -10.0), particle_gravity=True, clean_boundary=True, device=0, capacity=0,
                 no_graph=False, apic_damping=0.0, rpic_damping=0.0):
        res = tuple(int(r) for r in res)
        if len(res) != 2 or len(gravity) != 2:
            raise ValueError("a 2-D engine takes res = (r0, r1) and gravity = (g_x, g_y)")
        super().__init__(res, dx, dt, gravity, particle_gravity, clean_boundary, device=device, capacity=capacity, no_graph=no_graph,
                         dim=2, apic_damping=apic_damping, rpic_damping=rpic_damping)
        self.res = res

    def upload(self, x, v, mass, vol, F=None, b=None, scalar=None, group=None):
        x = _f32(x).reshape(-1, 2)
        n = len(x)
        v, F, b = _f32(v, (n, 2)), _f32(F, (n, 4)), _f32(b, (n, 4))
        mass, vol, scalar = _f32(mass, (n,)), _f32(vol, (n,)), _f32(scalar, (n,))
        group = None if group is None else np.ascontiguousarray(group, np.int32).reshape(n)
        self._check(self.L.mpmb_upload_particles(self.h, C.c_int64(n), _ptr(x), _ptr(v), _ptr(F), _ptr(b), _ptr(mass), _ptr(vol),
                                                 _ptr(scalar), _ptr(group)))

    def download(self, cap=None, sort_by_id=True):
        """Returns dict(id,x,v,F,b,mass,vol,ps,group) of the live particles (x, v [n, 2]; F, b [n, 4])."""
        if cap is None:
            cap = max(self.num_particles(), 1)
        out = dict(id=np.zeros(cap, np.uint32), x=np.zeros((cap, 2), np.float32), v=np.zeros((cap, 2), np.float32),
                   F=np.zeros((cap, 4), np.float32), b=np.zeros((cap, 4), np.float32), mass=np.zeros(cap, np.float32),
                   vol=np.zeros(cap, np.float32), ps=np.zeros(cap, np.float32), group=np.zeros(cap, np.int32))
        n = C.c_int64(0)
        self._check(self.L.mpmb_download_particles(self.h, C.c_int64(cap), C.byref(n), _ptr(out["id"]), _ptr(out["x"]), _ptr(out["v"]),
                                                   _ptr(out["F"]), _ptr(out["b"]), _ptr(out["mass"]), _ptr(out["vol"]), _ptr(out["ps"]),
                                                   _ptr(out["group"])))
        out = {k: a[: n.value] for k, a in out.items()}
        if sort_by_id:
            o = np.argsort(out["id"], kind="stable")
            out = {k: a[o] for k, a in out.items()}
        return out
