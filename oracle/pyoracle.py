"""ctypes front-end of the CPU oracle (oracle/mpm_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

MAT_LINEAR, MAT_JELLY, MAT_SNOW, MAT_WATER, MAT_SAND, MAT_ELASTIC, MAT_VON_MISES, MAT_VISCO = range(8)
N_MAT_PARAMS = 8


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "mpm_oracle.cpp")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.oracle_fast_create.restype = C.c_void_p
        _LIB.oracle_fast_substeps.restype = C.c_int64
        _LIB.oracle_fast_num_threads.restype = C.c_int
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _suf(dtype):
    return "f32" if np.dtype(dtype) == np.float32 else "f64"


def _scalar(dtype):
    return C.c_float if np.dtype(dtype) == np.float32 else C.c_double


def quadratic_kernel(x, dtype=np.float32):
    w = np.zeros(3, dtype)
    dw = np.zeros(3, dtype)
    getattr(lib(), "oracle_quadratic_kernel_" + _suf(dtype))(_scalar(dtype)(x), _p(w), _p(dw))
    return w, dw


def cubic_kernel(x, dtype=np.float32):
    w = np.zeros(4, dtype)
    dw = np.zeros(4, dtype)
    getattr(lib(), "oracle_cubic_kernel_" + _suf(dtype))(_scalar(dtype)(x), _p(w), _p(dw))
    return w, dw


def mls_fast_kernel(rel, dtype=np.float32):
    rel = np.ascontiguousarray(rel, dtype)
    w = np.zeros(27, dtype)
    getattr(lib(), "oracle_mls_fast_kernel_" + _suf(dtype))(_p(rel), _p(w))
    return w.reshape(3, 3, 3)


def svd3(A, dtype=np.float64):
    """A: 3x3 numpy (row/col as math). Returns U, s, V with A = U diag(s) V^T."""
    a = np.ascontiguousarray(np.asarray(A, dtype).T)  # column-major storage
    U = np.zeros((3, 3), dtype)
    s = np.zeros(3, dtype)
    V = np.zeros((3, 3), dtype)
    getattr(lib(), "oracle_svd3_" + _suf(dtype))(_p(a), _p(U), _p(s), _p(V))
    return U.T.copy(), s, V.T.copy()


def polar3(A, dtype=np.float64):
    a = np.ascontiguousarray(np.asarray(A, dtype).T)
    R = np.zeros((3, 3), dtype)
    S = np.zeros((3, 3), dtype)
    getattr(lib(), "oracle_polar3_" + _suf(dtype))(_p(a), _p(R), _p(S))
    return R.T.copy(), S.T.copy()


def calculate_force(kind, params, F, ps, vol, dtype=np.float64):
    """F: 3x3 math layout. Returns -vol*P*F^T (3x3 math layout)."""
    prm = np.zeros(N_MAT_PARAMS, dtype)
    prm[: len(params)] = params
    f = np.ascontiguousarray(np.asarray(F, dtype).T)
    out = np.zeros((3, 3), dtype)
    sc = _scalar(dtype)
    getattr(lib(), "oracle_calculate_force_" + _suf(dtype))(C.c_int(kind), _p(prm), _p(f), sc(ps), sc(vol), _p(out))
    return out.T.copy()


def plasticity(kind, params, cdg, F, ps, dtype=np.float64):
    prm = np.zeros(N_MAT_PARAMS, dtype)
    prm[: len(params)] = params
    c = np.ascontiguousarray(np.asarray(cdg, dtype).T)
    f = np.ascontiguousarray(np.asarray(F, dtype).T)
    p = np.array([ps], dtype)
    getattr(lib(), "oracle_plasticity_" + _suf(dtype))(C.c_int(kind), _p(prm), _p(c), _p(f), _p(p))
    return f.T.copy(), p[0]


def friction_project(vel, base, n, friction, dtype=np.float64):
    vel = np.ascontiguousarray(vel, dtype)
    base = np.ascontiguousarray(base, dtype)
    n = np.ascontiguousarray(n, dtype)
    out = np.zeros(3, dtype)
    getattr(lib(), "oracle_friction_project_" + _suf(dtype))(_p(vel), _p(base), _p(n), _scalar(dtype)(friction), _p(out))
    return out


def substep(scene, state, dtype=np.float64, want_grids=True):
    """One reference substep on a dense grid.

    scene: dict(res, dx, dt, gravity, particle_gravity, mat_kind[int32 G], mat_params[G,8],
                sdf (nx,ny,nz,4) or None, friction, clean_boundary (default 1; 0 skips clear_boundary_particles
                and drops a particle whose stencil leaves the node grid, the engine's rule))
    state: dict(x[N,3], v[N,3], F[N,9] col-major, b[N,9] col-major, mass[N], vol[N], ps[N],
                group[N] int32, alive[N] uint8)  -- converted to `dtype`, returned as new dict.
    Returns (new_state, grid_rast, grid_vel); grids are (nx,ny,nz,4).
    """
    res = np.asarray(scene["res"], np.int32)
    st = {k: np.ascontiguousarray(np.asarray(state[k], dtype)) for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
    st = {k: a.copy() for k, a in st.items()}
    st["group"] = np.ascontiguousarray(state["group"], np.int32)
    st["alive"] = np.ascontiguousarray(state.get("alive", np.ones(len(st["mass"]), np.uint8)), np.uint8).copy()
    n = len(st["mass"])
    mk = np.ascontiguousarray(scene["mat_kind"], np.int32)
    mp = np.ascontiguousarray(scene["mat_params"], dtype)
    sdf = scene.get("sdf")
    sdf = None if sdf is None else np.ascontiguousarray(sdf, dtype)
    g = np.ascontiguousarray(scene["gravity"], dtype)
    nn = tuple(int(r) + 1 for r in res)
    grid_rast = np.zeros(nn + (4,), dtype) if want_grids else None
    grid_vel = np.zeros(nn + (4,), dtype) if want_grids else None
    sc = _scalar(dtype)
    getattr(lib(), "oracle_substep_" + _suf(dtype))(
        _p(res), sc(scene["dx"]), sc(scene["dt"]), _p(g), C.c_int(int(scene.get("particle_gravity", 1))),
        C.c_int(int(scene.get("clean_boundary", 1))), C.c_int(len(mk)), _p(mk), _p(mp), _p(sdf), sc(scene.get("friction", 0.0)), C.c_int64(n),
        _p(st["x"]), _p(st["v"]), _p(st["F"]), _p(st["b"]), _p(st["mass"]), _p(st["vol"]), _p(st["ps"]), _p(st["group"]),
        _p(st["alive"]), _p(grid_rast), _p(grid_vel))
    return st, grid_rast, grid_vel


def substep_coupled(scene, state, rigid, dtype=np.float64):
    """One reference substep WITH rigid bodies (CPIC): rigid pages, CDF rasterisation, gather_cdf, block_op_rigid transfers
    (oracle/mpm_oracle.cpp, section "CPIC rigid-coupled path"), at a fixed rigid pose — the host-side rigid dynamics
    (rigidify / articulate / advect_rigid_bodies) are not part of it.

    rigid: dict(position[nr,3], rot[nr,9] col-major, velocity[nr,3], angular_velocity[nr,3], inv_mass[nr],
                inv_inertia[nr,9] world-space col-major, frictions[nr,2]  (row 0 = the background body, unused),
                sample_offset[ns,3], sample_tri[ns,9], sample_rigid[ns] int32, penalty, pushing_force)
    state additionally carries "states"[N] uint32 (MPMParticle::states; zeros if absent).
    Returns (new_state, grid_rast, grid_vel, rigid_out, cdf) with new_state["states"/"bnormal"/"bdist"/"near"],
    rigid_out = dict(velocity, angular_velocity) after both transfers, cdf = dict(node_state, node_dist)."""
    return _coupled("oracle_substep_coupled_", scene, state, rigid, dtype, True)


def p2g_coupled(scene, state, rigid, dtype=np.float64):
    """Only the coupled rasterize of substep_coupled(): ordering, rigid pages, the colour field, gather_cdf and the coupled P2G
    with its impulses (apply_tmp_velocity after rasterize, src/transfer.cpp:578-580).  Same arguments.
    Returns (state, grid_rast, rigid_out, cdf): state carries "states"/"bnormal"/"bdist"/"near" and, for the particles of rigid
    pages, v with the gravity kick the rasterize stores back; rigid_out = dict(velocity, angular_velocity) after the rasterize's
    impulses only."""
    st, grid_rast, _, rig, cdf = _coupled("oracle_p2g_coupled_", scene, state, rigid, dtype, False)
    return st, grid_rast, rig, cdf


def _coupled(entry, scene, state, rigid, dtype, with_grid_vel):
    res = np.asarray(scene["res"], np.int32)
    st = {k: np.ascontiguousarray(np.asarray(state[k], dtype)).copy() for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
    st["group"] = np.ascontiguousarray(state["group"], np.int32)
    n = len(st["mass"])
    st["alive"] = np.ascontiguousarray(state.get("alive", np.ones(n, np.uint8)), np.uint8).copy()
    st["states"] = np.ascontiguousarray(state.get("states", np.zeros(n, np.uint32)), np.uint32).copy()
    st["bnormal"], st["bdist"], st["near"] = np.zeros((n, 3), dtype), np.zeros(n, dtype), np.zeros(n, np.uint8)
    mk = np.ascontiguousarray(scene["mat_kind"], np.int32)
    mp = np.ascontiguousarray(scene["mat_params"], dtype)
    sdf = scene.get("sdf")
    sdf = None if sdf is None else np.ascontiguousarray(sdf, dtype)
    g = np.ascontiguousarray(scene["gravity"], dtype)
    nn = tuple(int(r) + 1 for r in res)
    grid_rast = np.zeros(nn + (4,), dtype)
    grid_vel = np.zeros(nn + (4,), dtype) if with_grid_vel else None
    node_state, node_dist = np.zeros(nn, np.uint32), np.zeros(nn, dtype)
    r = {k: np.ascontiguousarray(np.asarray(rigid[k], dtype)).copy() for k in ("position", "rot", "velocity", "angular_velocity", "inv_mass",
                                                                             "inv_inertia", "frictions", "sample_offset", "sample_tri")}
    sr = np.ascontiguousarray(rigid["sample_rigid"], np.int32)
    sc = _scalar(dtype)
    getattr(lib(), entry + _suf(dtype))(
        _p(res), sc(scene["dx"]), sc(scene["dt"]), _p(g), C.c_int(int(scene.get("particle_gravity", 1))), C.c_int(len(mk)),
        _p(mk), _p(mp), _p(sdf), sc(scene.get("friction", 0.0)), C.c_int64(n),
        _p(st["x"]), _p(st["v"]), _p(st["F"]), _p(st["b"]), _p(st["mass"]), _p(st["vol"]), _p(st["ps"]), _p(st["group"]),
        _p(st["alive"]), _p(grid_rast), *([_p(grid_vel)] if with_grid_vel else []), C.c_int(len(r["inv_mass"])), _p(r["position"]), _p(r["rot"]),
        _p(r["velocity"]), _p(r["angular_velocity"]), _p(r["inv_mass"]), _p(r["inv_inertia"]), _p(r["frictions"]), C.c_int64(len(sr)),
        _p(r["sample_offset"]), _p(r["sample_tri"]), _p(sr), sc(rigid.get("penalty", 0.0)), sc(rigid.get("pushing_force", 20000.0)),
        _p(st["states"]), _p(st["bnormal"]), _p(st["bdist"]), _p(st["near"]), _p(node_state), _p(node_dist))
    return st, grid_rast, grid_vel, dict(velocity=r["velocity"], angular_velocity=r["angular_velocity"]), dict(node_state=node_state, node_dist=node_dist)


class FastOracle:
    """fp32 OpenMP restatement of the reference's optimized CPU path (the timed CPU baseline)."""

    def __init__(self, scene, state, threads=None, reorder_interval=0):
        """reorder_interval: physical re-ordering of the particle storage every that many substeps
        (sort_allocator, src/mpm.cpp:753-768,811; the reference's default is 1000); 0 keeps storage
        index == caller index, which the parity tests rely on for identical tie order."""
        self.scene = scene
        self.res = np.asarray(scene["res"], np.int32)
        self.h = C.c_void_p(lib().oracle_fast_create(_p(self.res)))
        if reorder_interval:
            lib().oracle_fast_set_reorder(self.h, C.c_int(int(reorder_interval)))
        if threads:
            lib().oracle_fast_set_threads(C.c_int(threads))
        self.threads = lib().oracle_fast_num_threads()
        f32 = np.float32
        self.st = {k: np.ascontiguousarray(np.asarray(state[k], f32)).copy() for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
        self.st["group"] = np.ascontiguousarray(state["group"], np.int32)
        self.st["alive"] = np.ascontiguousarray(state.get("alive", np.ones(len(self.st["mass"]), np.uint8)), np.uint8).copy()
        self.mk = np.ascontiguousarray(scene["mat_kind"], np.int32)
        self.mp = np.ascontiguousarray(scene["mat_params"], f32)
        sdf = scene.get("sdf")
        self.sdf = None if sdf is None else np.ascontiguousarray(sdf, f32)
        self.g = np.ascontiguousarray(scene["gravity"], f32)

    def substeps(self, nsub):
        """Returns (particle_updates, timings[sort,p2g,grid,g2p,harness_io] seconds)."""
        t = np.zeros(5, np.float64)
        st = self.st
        sc = self.scene
        upd = lib().oracle_fast_substeps(
            self.h, C.c_int(nsub), _p(self.res), C.c_float(sc["dx"]), C.c_float(sc["dt"]), _p(self.g),
            C.c_int(int(sc.get("particle_gravity", 1))), C.c_int(int(sc.get("clean_boundary", 1))), _p(self.mk), _p(self.mp), _p(self.sdf),
            C.c_float(sc.get("friction", 0.0)),
            C.c_int64(len(st["mass"])), _p(st["x"]), _p(st["v"]), _p(st["F"]), _p(st["b"]), _p(st["mass"]), _p(st["vol"]),
            _p(st["ps"]), _p(st["group"]), _p(st["alive"]), _p(t))
        return int(upd), t

    def download_grid(self):
        nn = tuple(int(r) + 1 for r in self.res)
        g = np.zeros(nn + (4,), np.float32)
        lib().oracle_fast_download_grid(self.h, _p(g))
        return g

    def __del__(self):
        try:
            lib().oracle_fast_destroy(self.h)
        except Exception:
            pass


def mpm88_advance(n, dt, x, v, F, C_, Jp, E=1e4, nu=0.2, hardening=10.0, gravity_y=-200.0, plastic=False, dtype=np.float64):
    """One step of the 88-line 2D algorithm (mls-mpm88.cpp:16-69). Arrays are modified copies."""
    x = np.ascontiguousarray(x, dtype).copy()
    v = np.ascontiguousarray(v, dtype).copy()
    F = np.ascontiguousarray(F, dtype).copy()
    C_ = np.ascontiguousarray(C_, dtype).copy()
    Jp = np.ascontiguousarray(Jp, dtype).copy()
    grid = np.zeros((n + 1, n + 1, 3), dtype)
    sc = _scalar(dtype)
    getattr(lib(), "oracle_mpm88_advance_" + _suf(dtype))(
        C.c_int(n), sc(dt), sc(E), sc(nu), sc(hardening), sc(gravity_y), C.c_int(int(plastic)), C.c_int64(len(Jp)),
        _p(x), _p(v), _p(F), _p(C_), _p(Jp), _p(grid))
    return x, v, F, C_, Jp, grid


# ---- the reference's own frame writer (vendored Partio compiled from /root/reference, `make ref`)
_PARTIO = None


def partio_ref_available():
    """True when oracle/_ref/libpartio_ref.so exists or can be built (the reference tree is present)."""
    so = os.path.join(_HERE, "_ref", "libpartio_ref.so")
    return os.path.exists(so) or os.path.isdir("/root/reference/external/partio/src")


def partio_ref():
    global _PARTIO
    if _PARTIO is None:
        so = os.path.join(_HERE, "_ref", "libpartio_ref.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-C", _HERE, "-s", "ref"])
        _PARTIO = C.CDLL(so)
    return _PARTIO


def ref_write_partio(path, pos, v, type_, index, limit, verbose=None):
    """MPM<dim>::write_partio (src/visualize.cpp:16-100) through the reference's Partio.
    verbose: None or dict(m, boundary_normal, debug, states, boundary_distance, near_boundary, apic_frobenius_norm)."""
    f32, i32 = np.float32, np.int32
    pos = np.ascontiguousarray(pos, f32); v = np.ascontiguousarray(v, f32)
    type_ = np.ascontiguousarray(type_, i32); index = np.ascontiguousarray(index, i32); limit = np.ascontiguousarray(limit, i32)
    extra = [None] * 7
    if verbose is not None:
        extra = [np.ascontiguousarray(verbose["m"], f32), np.ascontiguousarray(verbose["boundary_normal"], f32),
                 np.ascontiguousarray(verbose["debug"], f32), np.ascontiguousarray(verbose["states"], i32),
                 np.ascontiguousarray(verbose["boundary_distance"], f32), np.ascontiguousarray(verbose["near_boundary"], i32),
                 np.ascontiguousarray(verbose["apic_frobenius_norm"], f32)]
    partio_ref().ref_write_partio(str(path).encode(), C.c_int64(len(pos)), _p(pos), _p(v), _p(type_), _p(index), _p(limit),
                                  C.c_int(0 if verbose is None else 1), *[None if e is None else _p(e) for e in extra])


# ---- the reference's 88-line 2-D program executed here (oracle/mpm88_ref.cpp + taichi_stub/taichi.h)
_REF88 = None


def ref88_available():
    so = os.path.join(_HERE, "_ref", "libmpm88_ref.so")
    return os.path.exists(so) or os.path.exists("/root/reference/mls-mpm88.cpp")


def ref88():
    global _REF88
    if _REF88 is None:
        so = os.path.join(_HERE, "_ref", "libmpm88_ref.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-C", _HERE, "-s", "ref"])
        _REF88 = C.CDLL(so)
    return _REF88


def ref88_run(x, v, F, C_, Jp, steps, plastic):
    """advance(dt) of /root/reference/mls-mpm88.cpp:16-69, `steps` times, on the given particles
    (fp32; F, C row-major 2x2; n=80, dt=1e-4, E=1e4, nu=0.2, hardening=10 are the program's constants).
    Returns x, v, F, C, Jp, grid[(n+1),(n+1),3]."""
    L = ref88()
    f32 = np.float32
    x, v, F, C_, Jp = (np.ascontiguousarray(a, f32).copy() for a in (x, v, F, C_, Jp))
    L.ref88_set(C.c_int64(len(x)), _p(x), _p(v), _p(F), _p(C_), _p(Jp), C.c_int(int(plastic)))
    L.ref88_advance(C.c_int(int(steps)))
    L.ref88_get(_p(x), _p(v), _p(F), _p(C_), _p(Jp))
    n = L.ref88_n()
    g = np.zeros((n + 1, n + 1, 3), f32)
    L.ref88_grid(_p(g))
    return x, v, F, C_, Jp, g


# ---- the reference's constitutive models executed here (oracle/particles_ref.cpp + taichi_stub/taichi/*.h)
_REFP = None


def ref_particles_available():
    so = os.path.join(_HERE, "_ref", "libparticles_ref.so")
    return os.path.exists(so) or os.path.exists("/root/reference/src/particles.cpp")


def ref_particles():
    global _REFP
    if _REFP is None:
        so = os.path.join(_HERE, "_ref", "libparticles_ref.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-C", _HERE, "-s", "ref"])
        _REFP = C.CDLL(so)
        _REFP.ref_sand_alpha.restype = C.c_float
    return _REFP


def ref_particle_step(kind, params, cdg, F, ps, vol, do_plasticity=True):
    """<Type>Particle<3>::plasticity(cdg) (optional) followed by calculate_force() of the reference's
    src/particles.cpp, fp32.  cdg, F: 3x3 math layout.  Returns F', ps', force (math layout)."""
    prm = np.zeros(N_MAT_PARAMS, np.float32)
    prm[: len(params)] = params
    c = np.ascontiguousarray(np.asarray(cdg, np.float32).T).reshape(9)
    f = np.ascontiguousarray(np.asarray(F, np.float32).T).reshape(9).copy()
    s = np.array([ps], np.float32)
    force = np.zeros(9, np.float32)
    rc = ref_particles().ref_particle(C.c_int(kind), _p(prm), _p(c), _p(f), _p(s), C.c_float(vol), _p(force), C.c_int(int(do_plasticity)))
    assert rc == 0
    return f.reshape(3, 3).T.copy(), float(s[0]), force.reshape(3, 3).T.copy()


def ref_allowed_dt(kind, params, F, ps, mass, vol, v, dx):
    """MPMParticle::get_allowed_dt of the reference's own particle classes (oracle/particles_ref.cpp)."""
    L = ref_particles()
    L.ref_allowed_dt.restype = C.c_float
    prm = np.zeros(N_MAT_PARAMS, np.float32)
    prm[: len(params)] = params
    f = np.ascontiguousarray(F, np.float32).reshape(9)
    vv = np.ascontiguousarray(v, np.float32)
    return float(L.ref_allowed_dt(C.c_int(kind), _p(prm), _p(f), C.c_float(ps), C.c_float(mass), C.c_float(vol), _p(vv), C.c_float(dx)))


def ref_default_params(kind):
    out = np.zeros(N_MAT_PARAMS, np.float32)
    assert ref_particles().ref_default_params(C.c_int(kind), _p(out)) == 0
    return out


def ref_friction_project(vel, base, n, friction):
    vel, base, n = (np.ascontiguousarray(a, np.float32) for a in (vel, base, n))
    out = np.zeros(3, np.float32)
    ref_particles().ref_friction_project(_p(vel), _p(base), _p(n), C.c_float(friction), _p(out))
    return out


# ---- the reference's interpolation kernels executed here (oracle/kernel_ref.cpp)
_REFK = None


def ref_kernel_available():
    so = os.path.join(_HERE, "_ref", "libkernel_ref.so")
    return os.path.exists(so) or os.path.exists("/root/reference/src/kernel.h")


def ref_kernels():
    global _REFK
    if _REFK is None:
        so = os.path.join(_HERE, "_ref", "libkernel_ref.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-C", _HERE, "-s", "ref"])
        _REFK = C.CDLL(so)
        _REFK.ref_inv_D.restype = C.c_float
    return _REFK


def ref_kernel(order, pos, inv_dx=1.0):
    """MPMKernel<3,order>(pos, inv_dx) of src/kernel.h: returns (stencil start[3], w[k,k,k], dw[k,k,k,3])."""
    k = order + 1
    pos = np.ascontiguousarray(pos, np.float32)
    start = np.zeros(3, np.int32)
    w = np.zeros(k ** 3, np.float32)
    dw = np.zeros(k ** 3 * 3, np.float32)
    assert ref_kernels().ref_kernel(C.c_int(order), _p(pos), C.c_float(inv_dx), _p(start), _p(w), _p(dw)) == 0
    return start, w.reshape(k, k, k), dw.reshape(k, k, k, 3)


def ref_fast_kernel32(pos, inv_dx=1.0):
    pos = np.ascontiguousarray(pos, np.float32)
    w = np.zeros(27, np.float32)
    dw = np.zeros(81, np.float32)
    ref_kernels().ref_fast_kernel32(_p(pos), C.c_float(inv_dx), _p(w), _p(dw))
    return w.reshape(3, 3, 3), dw.reshape(3, 3, 3, 3)


# ---- the reference's 3-D transfer loops executed here (oracle/transfer_ref.cpp)
_REFT = None


def ref_transfer_available():
    so = os.path.join(_HERE, "_ref", "libtransfer_ref.so")
    return os.path.exists(so) or os.path.exists("/root/reference/src/transfer.cpp")


def ref_transfer():
    global _REFT
    if _REFT is None:
        so = os.path.join(_HERE, "_ref", "libtransfer_ref.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-C", _HERE, "-s", "ref"])
        _REFT = C.CDLL(so)
        _REFT.reft_create.restype = C.c_void_p
        _REFT.reft_num_particles.restype = C.c_int64
    return _REFT


class RefSolver:
    """The reference's MPM<3> object with particles loaded directly (oracle/transfer_ref.cpp): single transfers,
    the grid update, or whole substeps by MPM<3>::substep().  fp32; material groups as in the oracle's scenes."""

    def __init__(self, scene, state):
        L = ref_transfer()
        L.reft_substep.restype = C.c_int64
        f32 = np.float32
        self.L = L
        self.res = np.ascontiguousarray(scene["res"], np.int32)
        g = np.ascontiguousarray(scene["gravity"], f32)
        self.h = C.c_void_p(L.reft_create(_p(self.res), C.c_float(scene["dx"]), C.c_float(scene["dt"]), _p(g),
                                          C.c_int(int(scene.get("particle_gravity", 1)))))
        kinds = np.asarray(scene["mat_kind"], np.int32)
        prms = np.zeros((len(kinds), N_MAT_PARAMS), f32)
        for g, q in enumerate(scene["mat_params"]):
            prms[g, : len(q)] = q
        st = {k: np.ascontiguousarray(state[k], f32) for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
        group = np.asarray(state.get("group", np.zeros(len(st["x"]), np.int32)), np.int64)
        self.n = len(st["x"])
        L.reft_add_particles.restype = C.c_int64
        if self.n and (group == group[0]).all():          # one material: bulk loader
            g = int(group[0])
            assert L.reft_add_particles(self.h, C.c_int(int(kinds[g])), _p(prms[g]), C.c_int64(self.n), _p(st["x"]), _p(st["v"]), _p(st["mass"]),
                                        _p(st["vol"]), _p(st["F"]), _p(st["b"]), _p(st["ps"])) == self.n
        else:
            for i in range(self.n):
                g = int(group[i])
                pid = L.reft_add_particle(self.h, C.c_int(int(kinds[g])), _p(prms[g]), _p(st["x"][i]), _p(st["v"][i]), C.c_float(st["mass"][i]),
                                          C.c_float(st["vol"][i]), _p(st["F"][i]), _p(st["b"][i]), C.c_float(st["ps"][i]))
                assert pid == i
        if scene.get("planes") is not None:      # grid units, (n, d) per plane — what scenes.planes_sdf rasterises
            pl = np.ascontiguousarray(scene["planes"], f32).reshape(-1, 4)
            L.reft_set_planes(self.h, C.c_int(len(pl)), _p(pl), C.c_float(scene.get("friction", 0.0)))

    @classmethod
    def from_benchmark(cls, res, dt, gravity, type_name, benchmark=125, density=400.0, particle_gravity=1):
        """A solver seeded by the reference's own add_particles(type=..., benchmark=...) (src/mpm.cpp:155-186), the way
        scripts/benchmark/benchmark_3d.py sets its scene up."""
        L = ref_transfer()
        L.reft_substep.restype = C.c_int64
        L.reft_add_benchmark.restype = C.c_int64
        self = cls.__new__(cls)
        self.L = L
        self.res = np.array([res] * 3, np.int32)
        g = np.ascontiguousarray(gravity, np.float32)
        self.h = C.c_void_p(L.reft_create(_p(self.res), C.c_float(1.0 / res), C.c_float(dt), _p(g), C.c_int(int(particle_gravity))))
        self.n = int(L.reft_add_benchmark(self.h, type_name.encode(), C.c_int(int(benchmark)), C.c_float(density)))
        return self

    def set_threads(self, n):
        """Threads of the stand-in's parallel loops; 1 (default) = serial, what every pin runs with."""
        self.L.reft_set_threads(self.h, C.c_int(int(n)))

    def p2g(self, optimized=True):
        """Ordering + P2G.  g2p() must follow a p2g() of the same particle positions (it reads that ordering)."""
        self.L.reft_p2g(self.h, C.c_int(int(optimized)))

    def grid_update(self):
        """normalize_grid_and_apply_external_force + apply_grid_boundary_conditions (src/mpm.cpp:277-372)"""
        self.L.reft_grid_update(self.h)

    def g2p(self, optimized=True):
        self.L.reft_g2p(self.h, C.c_int(int(optimized)))

    def get_grid(self):
        grid = np.zeros(tuple(int(r) + 1 for r in self.res) + (4,), np.float32)
        self.L.reft_get_grid(self.h, _p(grid))
        return grid

    def set_grid(self, grid):
        gv = np.ascontiguousarray(grid, np.float32)
        assert gv.shape == tuple(int(r) + 1 for r in self.res) + (4,)
        self.L.reft_set_grid(self.h, _p(gv))

    def substep(self, n=1):
        """MPM<3>::substep() n times (src/mpm.cpp:452-575).  Returns the number of live particles."""
        return int(self.L.reft_substep(self.h, C.c_int(int(n))))

    def step(self, dt):
        """MPM<3>::step(dt) (src/mpm.cpp:428-450).  Returns (substep_counter, current_t, request_t), the clocks as the
        reference's `real` (float32) members hold them."""
        self.L.reft_step.restype = C.c_int64
        cur, req = C.c_float(0), C.c_float(0)
        n = int(self.L.reft_step(self.h, C.c_float(float(dt)), C.byref(cur), C.byref(req)))
        return n, np.float32(cur.value), np.float32(req.value)

    def substep_via_mpmb(self, lib_path, n=1):
        """The drop-in, executed (INTEGRATION.md §2): the reference's MPM<3> object hands its AoS pool to libmpmb through the
        C-ABI (mpmb_upload_aos with the slot layout taken by offsetof on the reference's own classes), the engine runs n
        substeps, and pool + index vector are refreshed (mpmb_download_aos).  lib_path: libmpmb.so or its SIMT-emulator
        build.  Single material.  Returns the number of survivors."""
        self.L.reft_substep_via_mpmb.restype = C.c_int64
        err = C.create_string_buffer(512)
        r = int(self.L.reft_substep_via_mpmb(self.h, str(lib_path).encode(), C.c_int(int(n)), err, C.c_int(512)))
        if r < 0:
            raise RuntimeError("mpmb through the reference's pool failed (%d): %s" % (r, err.value.decode(errors="replace")))
        return r

    def particles(self):
        """dict(x, v, F, b, ps) indexed by particle id (rows of deleted particles are zero) + alive ids."""
        n, f32 = self.n, np.float32
        out = dict(x=np.zeros((n, 3), f32), v=np.zeros((n, 3), f32), F=np.zeros((n, 9), f32), b=np.zeros((n, 9), f32), ps=np.zeros(n, f32))
        self.L.reft_get_particles(self.h, _p(out["x"]), _p(out["v"]), _p(out["F"]), _p(out["b"]), _p(out["ps"]))
        na = int(self.L.reft_num_particles(self.h))
        ids = np.zeros(na, np.int32)
        self.L.reft_alive_ids(self.h, _p(ids))
        out["alive_ids"] = np.sort(ids)
        return out

    # ---- rigid bodies (CPIC): src/rigid_transfer.cpp and the block_op_rigid branches of src/transfer.cpp, run by the
    # reference's own solver object against the stand-in RigidBody (oracle/taichi_stub/taichi/dynamics/rigid_body.h)
    def set_rigid(self, rigid):
        f32 = np.float32
        r = {k: np.ascontiguousarray(rigid[k], f32) for k in ("position", "rot", "velocity", "angular_velocity", "inv_mass", "inv_inertia", "frictions",
                                                               "sample_offset", "sample_tri")}
        sr = np.ascontiguousarray(rigid["sample_rigid"], np.int32)
        rc = self.L.reft_set_rigid(self.h, C.c_int(len(r["inv_mass"])), _p(r["position"]), _p(r["rot"]), _p(r["velocity"]), _p(r["angular_velocity"]),
                                   _p(r["inv_mass"]), _p(r["inv_inertia"]), _p(r["frictions"]), C.c_int64(len(sr)), _p(r["sample_offset"]),
                                   _p(r["sample_tri"]), _p(sr), C.c_float(rigid.get("penalty", 0.0)), C.c_float(rigid.get("pushing_force", 20000.0)))
        assert rc == 0
        self.n_bodies = len(r["inv_mass"])

    def set_rigid_state(self, rigid):
        f32 = np.float32
        r = {k: np.ascontiguousarray(rigid[k], f32) for k in ("position", "rot", "velocity", "angular_velocity")}
        self.L.reft_set_rigid_state(self.h, _p(r["position"]), _p(r["rot"]), _p(r["velocity"]), _p(r["angular_velocity"]))

    def rigid_state(self):
        v, w = np.zeros((self.n_bodies, 3), np.float32), np.zeros((self.n_bodies, 3), np.float32)
        self.L.reft_get_rigid_state(self.h, _p(v), _p(w))
        return dict(velocity=v, angular_velocity=w)

    def set_states(self, states):
        st = np.ascontiguousarray(states, np.uint32)
        assert len(st) == self.n
        self.L.reft_set_states(self.h, _p(st))

    def coupled_stage(self, stage):
        """0: ordering + rigid pages + rasterize_rigid_boundary + gather_cdf; 1: rasterize_optimized; 2: grid update;
        3: resample_optimized + clear_boundary_particles (the calls of MPM<3>::substep, src/mpm.cpp:464-565)."""
        self.L.reft_coupled_stage(self.h, C.c_int(int(stage)))

    def cdf_particles(self):
        n = self.n
        out = dict(states=np.zeros(n, np.uint32), bnormal=np.zeros((n, 3), np.float32), bdist=np.zeros(n, np.float32), near=np.zeros(n, np.uint8))
        self.L.reft_get_cdf_particles(self.h, _p(out["states"]), _p(out["bnormal"]), _p(out["bdist"]), _p(out["near"]))
        return out

    def cdf_grid(self):
        nn = tuple(int(r) + 1 for r in self.res)
        st, d = np.zeros(nn, np.uint32), np.zeros(nn, np.float32)
        self.L.reft_get_cdf_grid(self.h, _p(st), _p(d))
        return dict(node_state=st, node_dist=d)

    def is_rigid_page(self, node):
        return bool(self.L.reft_is_rigid_page(self.h, C.c_int(int(node[0])), C.c_int(int(node[1])), C.c_int(int(node[2]))))

    def write_partio(self, path):
        """MPM<3>::write_partio (src/visualize.cpp:16-100) on the solver's current particles."""
        self.L.reft_write_partio(self.h, str(path).encode())

    def close(self):
        if self.h is not None:
            self.L.reft_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RefAsyncSolver:
    """The reference's AsyncMPM<3> object (src/async/async_mpm.{h,cpp} compiled in place, oracle/transfer_ref.cpp): its own
    scheduler — per-block power-of-two time levels, backup pools, update_dt_limits / advance / step — around MPM<3>::substep(),
    which runs either as the reference's own code or, after route_through(lib), on libmpmb through the C-ABI (the drop-in patch
    point; base_delta_t changes from call to call).  One material; fp32."""

    def __init__(self, scene, state, unit_delta_t, max_units=8192, cfl_dt_mul=1.0, strength_dt_mul=1.0):
        L = ref_transfer()
        f32 = np.float32
        self.L = L
        self.res = np.ascontiguousarray(scene["res"], np.int32)
        g = np.ascontiguousarray(scene["gravity"], f32)
        L.reft_create_async.restype = C.c_void_p
        self.h = C.c_void_p(L.reft_create_async(_p(self.res), C.c_float(scene["dx"]), _p(g), C.c_int(int(scene.get("particle_gravity", 1))),
                                                C.c_float(unit_delta_t), C.c_int64(int(max_units)), C.c_float(cfl_dt_mul), C.c_float(strength_dt_mul)))
        kinds = np.asarray(scene["mat_kind"], np.int32)
        prm = np.zeros(N_MAT_PARAMS, f32)
        prm[: len(scene["mat_params"][0])] = scene["mat_params"][0]
        st = {k: np.ascontiguousarray(state[k], f32) for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
        self.n = len(st["x"])
        L.reft_add_particles.restype = C.c_int64
        assert L.reft_add_particles(self.h, C.c_int(int(kinds[0])), _p(prm), C.c_int64(self.n), _p(st["x"]), _p(st["v"]), _p(st["mass"]), _p(st["vol"]),
                                    _p(st["F"]), _p(st["b"]), _p(st["ps"])) == self.n
        if scene.get("planes") is not None:
            pl = np.ascontiguousarray(scene["planes"], f32).reshape(-1, 4)
            L.reft_set_planes(self.h, C.c_int(len(pl)), _p(pl), C.c_float(scene.get("friction", 0.0)))
        L.reft_async_distribute(self.h)

    def route_through(self, lib_path):
        self.L.reft_route_through(self.h, str(lib_path or "").encode())

    def step(self, dt):
        """AsyncMPM<3>::step(dt).  Returns dict(alive, update_counter, current_t_int, min_level, max_level, routed_substeps)."""
        self.L.reft_async_step.restype = C.c_int64
        self.L.reft_routed_substeps.restype = C.c_int64
        out = np.zeros(4, np.int64)
        n = int(self.L.reft_async_step(self.h, C.c_float(float(dt)), _p(out)))
        if n < 0:
            self.L.reft_route_error.restype = C.c_char_p
            raise RuntimeError("routed substep failed: " + self.L.reft_route_error(self.h).decode(errors="replace"))
        return dict(alive=n, update_counter=int(out[0]), current_t_int=int(out[1]), min_level=int(out[2]), max_level=int(out[3]),
                    routed_substeps=int(self.L.reft_routed_substeps(self.h)))

    def particles(self):
        n, f32 = self.n, np.float32
        out = dict(x=np.zeros((n, 3), f32), v=np.zeros((n, 3), f32), F=np.zeros((n, 9), f32), b=np.zeros((n, 9), f32), ps=np.zeros(n, f32),
                   alive=np.zeros(n, np.uint8))
        self.L.reft_async_get_particles.restype = C.c_int64
        self.L.reft_async_get_particles(self.h, _p(out["x"]), _p(out["v"]), _p(out["F"]), _p(out["b"]), _p(out["ps"]), _p(out["alive"]))
        return out

    def close(self):
        if self.h is not None:
            self.L.reft_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def ref_transfer_substep(scene, state, grid_vel, optimized=True):
    """One substep's two transfers by the reference's own code (src/transfer.cpp), fp32:
    P2G = rasterize_optimized / rasterize on the given particles -> dense node (momentum, mass);
    then the node values are replaced by `grid_vel` (dense [(res+1)^3][4] node velocities) and
    G2P = resample_optimized / resample moves the particles.  Returns grid_after_p2g, dict(x, v, F, b, ps)."""
    s = RefSolver(scene, state)
    try:
        s.p2g(optimized)
        grid = s.get_grid()
        s.set_grid(grid_vel)
        s.g2p(optimized)
        p = s.particles()
        p.pop("alive_ids")
        return grid, p
    finally:
        s.close()


def ref_substep_coupled(scene, state, rigid):
    """One coupled substep by the REFERENCE's own code (src/mpm.cpp ordering and rigid pages, src/rigid_transfer.cpp,
    src/transfer.cpp block_op_switch) at a fixed rigid pose, fp32.  Same return shape as substep_coupled()."""
    s = RefSolver(scene, state)
    try:
        s.set_rigid(rigid)
        if state.get("states") is not None:
            s.set_states(state["states"])
        s.coupled_stage(0)
        cdf, pc = s.cdf_grid(), s.cdf_particles()
        s.coupled_stage(1)
        grid_rast = s.get_grid()
        s.coupled_stage(2)
        grid_vel = s.get_grid()
        s.coupled_stage(3)
        p = s.particles()
        alive = np.zeros(s.n, np.uint8)
        alive[p.pop("alive_ids")] = 1
        new = dict(p, alive=alive, states=pc["states"], bnormal=pc["bnormal"], bdist=pc["bdist"], near=pc["near"])
        return new, grid_rast, grid_vel, s.rigid_state(), cdf
    finally:
        s.close()


def ref_benchmark_particles(res, type_name="sand", benchmark=125, density=400.0):
    """MPM<3>::add_particles with `benchmark` (src/mpm.cpp:155-186) run by the reference itself: returns
    dict(x, v, F, mass, vol) of the lattice it seeds (benchmark 125: a cube of res*0.2 cells, 8000: res*0.8)."""
    L = ref_transfer()
    L.reft_add_benchmark.restype = C.c_int64
    f32 = np.float32
    r = np.array([res] * 3, np.int32)
    g = np.array([0, -10, 0], f32)
    h = C.c_void_p(L.reft_create(_p(r), C.c_float(1.0 / res), C.c_float(1e-4), _p(g), C.c_int(1)))
    try:
        n = int(L.reft_add_benchmark(h, type_name.encode(), C.c_int(benchmark), C.c_float(density)))
        out = dict(x=np.zeros((n, 3), f32), v=np.zeros((n, 3), f32), F=np.zeros((n, 9), f32), mass=np.zeros(n, f32), vol=np.zeros(n, f32))
        b, ps = np.zeros((n, 9), f32), np.zeros(n, f32)
        L.reft_get_particles(h, _p(out["x"]), _p(out["v"]), _p(out["F"]), _p(b), _p(ps))
        L.reft_get_mass_vol(h, _p(out["mass"]), _p(out["vol"]))
        return out
    finally:
        L.reft_destroy(h)
