"""ctypes front-end of the 2-D oracle (oracle/mpm2d_oracle.cpp -> liboracle2d.so) and of the reference's own MPM<2> compiled
in place (oracle/transfer2d_ref.cpp -> _ref/libtransfer2d_ref.so, only where the reference tree exists).

TEST INFRASTRUCTURE ONLY: imported by tests/, bench_2d.py's CPU baselines and tests/golden/make_mpm2d_golden.py.  The product
package never imports this module.  The libraries are built with the flags oracle/Makefile uses for liboracle.so and
_ref/libtransfer_ref.so.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.pyoracle import N_MAT_PARAMS, _p, _scalar, _suf

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_REF = None
REFERENCE = "/root/reference"
LIB = os.path.join(_HERE, "liboracle2d.so")
REF_LIB = os.path.join(_HERE, "_ref", "libtransfer2d_ref.so")
_CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"   # not $CXX: see oracle/Makefile


def _stale(out, deps):
    return not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps)


def build(force=False):
    """liboracle2d.so: mpm2d_oracle.cpp (which includes mpm_oracle.cpp)."""
    deps = [os.path.join(_HERE, f) for f in ("mpm2d_oracle.cpp", "mpm_oracle.cpp")]
    if force or _stale(LIB, deps):
        subprocess.check_call([_CXX, "-O3", "-march=x86-64-v3", "-mfma", "-std=c++17", "-fopenmp", "-fPIC", "-ffp-contract=off", "-Wall",
                               "-Wno-unused-function", "-shared", "-o", LIB, deps[0]], cwd=_HERE)
    return LIB


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


def ref_available():
    return os.path.exists(REF_LIB) or os.path.exists(os.path.join(REFERENCE, "src", "mpm.cpp"))


def ref_build(force=False):
    """_ref/libtransfer2d_ref.so: transfer2d_ref.cpp (which includes transfer_ref.cpp) against the reference's sources where
    they lie, the command line of oracle/Makefile's _ref/libtransfer_ref.so."""
    stub = os.path.join(_HERE, "taichi_stub")
    deps = [os.path.join(_HERE, f) for f in ("transfer2d_ref.cpp", "transfer_ref.cpp")]
    deps += [os.path.join(d, f) for d, _, fs in os.walk(stub) for f in fs if f.endswith(".h")]
    if not (force or _stale(REF_LIB, deps)):
        return REF_LIB
    R = REFERENCE
    src, ext, partio = os.path.join(R, "src"), os.path.join(R, "external"), os.path.join(R, "external", "partio", "src")
    partio_src = [os.path.join(partio, p) for p in ("core/Particle.cpp", "core/ParticleCaching.cpp", "core/ParticleHeaders.cpp",
                                                     "core/ParticleSimple.cpp", "core/ParticleSimpleInterleave.cpp", "io/BGEO.cpp",
                                                     "io/ParticleIO.cpp", "io/ZIP.cpp")]
    os.makedirs(os.path.dirname(REF_LIB), exist_ok=True)
    defs = {"REF_TRANSFER_SOURCE": "transfer.cpp", "REF_MPM_SOURCE": "mpm.cpp", "REF_VISUALIZE_SOURCE": "visualize.cpp",
            "REF_PARTICLES_SOURCE": "particles.cpp", "REF_RIGID_TRANSFER_SOURCE": "rigid_transfer.cpp",
            "REF_BOUNDARY_PARTICLE_SOURCE": "boundary_particle.cpp", "REF_ASYNC_SOURCE": "async/async_mpm.cpp"}
    cmd = [_CXX, "-O2", "-std=c++17", "-fopenmp", "-fPIC", "-shared", "-mavx2", "-mfma", "-ffp-contract=off", "-w", "-include", "cstdint",
           "-include", "cstring", "-I" + stub, "-I" + ext, "-I" + src, "-I" + partio]
    cmd += ['-D%s="%s"' % (k, os.path.join(src, v)) for k, v in defs.items()]
    cmd += ["-o", REF_LIB, deps[0], os.path.join(ext, "SPGrid", "Core", "SPGrid_Utilities.cpp"),
            os.path.join(ext, "SPGrid", "Core", "SPGrid_Geometry.cpp")] + partio_src + ["-ldl"]
    subprocess.check_call(cmd, cwd=_HERE)
    return REF_LIB


def ref_lib():
    global _REF
    if _REF is None:
        _REF = C.CDLL(REF_LIB if os.path.exists(REF_LIB) and not os.path.exists(os.path.join(REFERENCE, "src")) else ref_build())
    return _REF


def substep2d(scene, state, dtype=np.float64, want_grids=True):
    """One MPM<2> substep on a dense grid (oracle_substep2d).

    scene: dict(res (r0, r1), dx, dt, gravity (gx, gy), particle_gravity, clean_boundary, apic_damping, rpic_damping,
                mat_kind[int32 G], mat_params[G,8], sdf (nx,ny,4) = (n_x, n_y, 0, phi) or None, friction)
    state: dict(x[N,2], v[N,2], F[N,4] col-major, b[N,4] col-major, mass[N], vol[N], ps[N], group[N] int32, alive[N] uint8).
    Returns (new_state, grid_rast, grid_vel); grids are (nx,ny,4).
    """
    res = np.asarray(scene["res"], np.int32)[:2].copy()
    st = {k: np.ascontiguousarray(np.asarray(state[k], dtype)).copy() for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
    st["group"] = np.ascontiguousarray(state["group"], np.int32)
    st["alive"] = np.ascontiguousarray(state.get("alive", np.ones(len(st["mass"]), np.uint8)), np.uint8).copy()
    n = len(st["mass"])
    mk = np.ascontiguousarray(scene["mat_kind"], np.int32)
    mp = np.ascontiguousarray(scene["mat_params"], dtype)
    sdf = scene.get("sdf")
    sdf = None if sdf is None else np.ascontiguousarray(sdf, dtype)
    g = np.ascontiguousarray(scene["gravity"][:2], dtype)
    nn = tuple(int(r) + 1 for r in res)
    grid_rast = np.zeros(nn + (4,), dtype) if want_grids else None
    grid_vel = np.zeros(nn + (4,), dtype) if want_grids else None
    sc = _scalar(dtype)
    getattr(lib(), "oracle_substep2d_" + _suf(dtype))(
        _p(res), sc(scene["dx"]), sc(scene["dt"]), _p(g), C.c_int(int(scene.get("particle_gravity", 1))),
        C.c_int(int(scene.get("clean_boundary", 1))), sc(scene.get("apic_damping", 0.0)), sc(scene.get("rpic_damping", 0.0)),
        _p(mk), _p(mp), _p(sdf), sc(scene.get("friction", 0.0)), C.c_int64(n),
        _p(st["x"]), _p(st["v"]), _p(st["F"]), _p(st["b"]), _p(st["mass"]), _p(st["vol"]), _p(st["ps"]), _p(st["group"]),
        _p(st["alive"]), _p(grid_rast), _p(grid_vel))
    return st, grid_rast, grid_vel


def calculate_force2d(kind, params, F, ps, vol, dtype=np.float64):
    """F: 2x2 math layout. Returns -vol*P*F^T (2x2 math layout) of the dim = 2 model."""
    prm = np.zeros(N_MAT_PARAMS, dtype)
    prm[: len(params)] = params
    f = np.ascontiguousarray(np.asarray(F, dtype).T)
    out = np.zeros((2, 2), dtype)
    sc = _scalar(dtype)
    getattr(lib(), "oracle_calculate_force2d_" + _suf(dtype))(C.c_int(kind), _p(prm), _p(f), sc(ps), sc(vol), _p(out))
    return out.T.copy()


def plasticity2d(kind, params, cdg, F, ps, dtype=np.float64):
    prm = np.zeros(N_MAT_PARAMS, dtype)
    prm[: len(params)] = params
    c = np.ascontiguousarray(np.asarray(cdg, dtype).T)
    f = np.ascontiguousarray(np.asarray(F, dtype).T)
    p = np.array([ps], dtype)
    getattr(lib(), "oracle_plasticity2d_" + _suf(dtype))(C.c_int(kind), _p(prm), _p(c), _p(f), _p(p))
    return f.T.copy(), p[0]


class RefSolver2D:
    """The reference's MPM<2> object (oracle/transfer_ref.cpp, reft2_*) with particles loaded directly: its own ordering,
    scalar transfers, grid update and deletion stage by stage, whole substeps by MPM<2>::substep(), and write_partio.  fp32;
    one material; the scene and state dicts of substep2d (planes from scene["planes"] = [(n_x, n_y, 0, d)], grid units)."""

    def __init__(self, scene, state):
        L = ref_lib()
        L.reft2_create.restype = C.c_void_p
        L.reft2_substep.restype = C.c_int64
        L.reft2_add_particles.restype = C.c_int64
        L.reft2_num_particles.restype = C.c_int64
        f32 = np.float32
        self.L = L
        self.res = np.ascontiguousarray(scene["res"][:2], np.int32)
        g = np.ascontiguousarray(scene["gravity"][:2], f32)
        self.h = C.c_void_p(L.reft2_create(_p(self.res), C.c_float(scene["dx"]), C.c_float(scene["dt"]), _p(g),
                                           C.c_int(int(scene.get("particle_gravity", 1))), C.c_int(int(scene.get("clean_boundary", 1))),
                                           C.c_float(scene.get("apic_damping", 0.0)), C.c_float(scene.get("rpic_damping", 0.0))))
        kinds = np.asarray(scene["mat_kind"], np.int32)
        assert len(kinds) == 1, "one material"
        prm = np.zeros(N_MAT_PARAMS, f32)
        prm[: len(scene["mat_params"][0])] = scene["mat_params"][0]
        st = {k: np.ascontiguousarray(state[k], f32) for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
        self.n = len(st["x"])
        assert L.reft2_add_particles(self.h, C.c_int(int(kinds[0])), _p(prm), C.c_int64(self.n), _p(st["x"]), _p(st["v"]), _p(st["mass"]),
                                     _p(st["vol"]), _p(st["F"]), _p(st["b"]), _p(st["ps"])) == self.n
        if scene.get("planes") is not None:
            pl = np.ascontiguousarray(np.asarray(scene["planes"], f32).reshape(-1, 4)[:, [0, 1, 3]])
            L.reft2_set_planes(self.h, C.c_int(len(pl)), _p(pl), C.c_float(scene.get("friction", 0.0)))

    def set_threads(self, n):
        """Threads of the stand-in's parallel loops; 1 (default) = serial, what every pin runs with."""
        self.L.reft2_set_threads(self.h, C.c_int(int(n)))

    def stage(self, k):
        """1: sort_particles_and_populate_grid + rasterize_optimized; 2: the grid update; 3: resample_optimized + deletion."""
        self.L.reft2_stage(self.h, C.c_int(int(k)))

    def get_grid(self):
        """Dense (res0+1, res1+1, 4) = (p_x | v_x, p_y | v_y, 0, m)."""
        g = np.zeros((int(self.res[0]) + 1, int(self.res[1]) + 1, 4), np.float32)
        self.L.reft2_get_grid(self.h, _p(g))
        return g

    def substep(self, n=1):
        return int(self.L.reft2_substep(self.h, C.c_int(int(n))))

    def particles(self):
        """dict(x, v, F, b, ps, alive) indexed by particle id (rows of deleted particles are zero, alive 0)."""
        n, f32 = self.n, np.float32
        out = dict(x=np.zeros((n, 2), f32), v=np.zeros((n, 2), f32), F=np.zeros((n, 4), f32), b=np.zeros((n, 4), f32), ps=np.zeros(n, f32),
                   alive=np.zeros(n, np.uint8))
        self.L.reft2_get_particles(self.h, _p(out["x"]), _p(out["v"]), _p(out["F"]), _p(out["b"]), _p(out["ps"]), _p(out["alive"]))
        return out

    def write_partio(self, path):
        self.L.reft2_write_partio(self.h, str(path).encode())

    def close(self):
        if self.h is not None:
            self.L.reft2_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
