"""ctypes front-end of the drop-in for pools that mix particle types (oracle/transfer_mixed_ref.cpp ->
_ref/libtransfer_mixed_ref.so, built only where the reference tree exists): the reference's own MPM<3> and AsyncMPM<3>
objects of oracle/pyoracle.py, loaded from that library, with every particle added under its own group's type and
parameters, and substeps routed to libmpmb with one material group per distinct (type, parameters) and per-kind
plastic-scalar offsets in MpmbAosLayout.

TEST INFRASTRUCTURE ONLY: imported by tests/ and bench_dropin_mixed.py.  The product package never imports this module.  The
library is built with the command line of oracle/Makefile's _ref/libtransfer_ref.so.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyoracle as O
from oracle.pyoracle import N_MAT_PARAMS, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF = None
REFERENCE = "/root/reference"
REF_LIB = os.path.join(_HERE, "_ref", "libtransfer_mixed_ref.so")
_CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"   # not $CXX: see oracle/Makefile


def _stale(out, deps):
    return not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps)


def ref_available():
    return os.path.exists(REF_LIB) or os.path.exists(os.path.join(REFERENCE, "src", "mpm.cpp"))


def ref_build(force=False):
    """_ref/libtransfer_mixed_ref.so: transfer_mixed_ref.cpp (which includes transfer_ref.cpp) against the reference's sources
    where they lie.  AsyncMPM's source comes in through async_route_mixed.h."""
    stub = os.path.join(_HERE, "taichi_stub")
    deps = [os.path.join(_HERE, f) for f in ("transfer_mixed_ref.cpp", "transfer_ref.cpp", "async_route_mixed.h")]
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
            "REF_BOUNDARY_PARTICLE_SOURCE": "boundary_particle.cpp", "REF_ASYNC_ROUTED_SOURCE": "async/async_mpm.cpp"}
    cmd = [_CXX, "-O2", "-std=c++17", "-fopenmp", "-fPIC", "-shared", "-mavx2", "-mfma", "-ffp-contract=off", "-w", "-include", "cstdint",
           "-include", "cstring", "-I" + stub, "-I" + ext, "-I" + src, "-I" + partio]
    cmd += ['-D%s="%s"' % (k, os.path.join(src, v)) for k, v in defs.items()]
    cmd += ['-DREF_ASYNC_SOURCE="%s"' % os.path.join(_HERE, "async_route_mixed.h")]
    cmd += ["-o", REF_LIB, deps[0], os.path.join(ext, "SPGrid", "Core", "SPGrid_Utilities.cpp"),
            os.path.join(ext, "SPGrid", "Core", "SPGrid_Geometry.cpp")] + partio_src + ["-ldl"]
    subprocess.check_call(cmd, cwd=_HERE)
    return REF_LIB


def ref_lib():
    global _REF
    if _REF is None:
        L = C.CDLL(REF_LIB if os.path.exists(REF_LIB) and not os.path.exists(os.path.join(REFERENCE, "src")) else ref_build())
        L.reft_create.restype = C.c_void_p
        L.reft_create_async.restype = C.c_void_p
        L.reft_num_particles.restype = C.c_int64
        L.reft_substep.restype = C.c_int64
        L.reft_substep_via_mpmb_mixed.restype = C.c_int64
        _REF = L
    return _REF


def aos_scalar_offsets():
    """offsetof() of SnowParticle::Jp, WaterParticle::j, SandParticle::logJp, ViscoParticle::visco_tau: the reference's
    MpmbAosLayout.off_scalar_by_kind."""
    out = np.zeros(4, np.int32)
    ref_lib().reft_aos_scalar_offsets(_p(out))
    return out


def aos_layout(kind=-1):
    """The slot layout of the reference's pool (reft_aos_layout): stride, pos, v_and_m, dg_e, apic_b, col_pitch, vol, scalar."""
    out = np.zeros(8, np.int32)
    ref_lib().reft_aos_layout(C.c_int(int(kind)), _p(out))
    return out


def _add_particles(L, h, scene, state):
    """Every particle under its group's type and parameters (reft_add_particle), ids = row of `state`.  Returns n."""
    f32 = np.float32
    kinds = np.asarray(scene["mat_kind"], np.int32)
    prms = np.zeros((len(kinds), N_MAT_PARAMS), f32)
    for g, q in enumerate(scene["mat_params"]):
        prms[g, : len(q)] = q
    st = {k: np.ascontiguousarray(state[k], f32) for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
    group = np.asarray(state.get("group", np.zeros(len(st["x"]), np.int32)), np.int64)
    for i in range(len(st["x"])):
        g = int(group[i])
        pid = L.reft_add_particle(h, C.c_int(int(kinds[g])), _p(prms[g]), _p(st["x"][i]), _p(st["v"][i]), C.c_float(st["mass"][i]),
                                  C.c_float(st["vol"][i]), _p(st["F"][i]), _p(st["b"][i]), C.c_float(st["ps"][i]))
        assert pid == i
    if scene.get("planes") is not None:
        pl = np.ascontiguousarray(scene["planes"], f32).reshape(-1, 4)
        L.reft_set_planes(h, C.c_int(len(pl)), _p(pl), C.c_float(scene.get("friction", 0.0)))
    return len(st["x"])


class MixedRefSolver(O.RefSolver):
    """The reference's MPM<3> object (pyoracle.RefSolver) whose substep_via_mpmb routes a pool of several particle types."""

    def __init__(self, scene, state):
        self.L = L = ref_lib()
        self.res = np.ascontiguousarray(scene["res"], np.int32)
        g = np.ascontiguousarray(scene["gravity"], np.float32)
        self.h = C.c_void_p(L.reft_create(_p(self.res), C.c_float(scene["dx"]), C.c_float(scene["dt"]), _p(g),
                                          C.c_int(int(scene.get("particle_gravity", 1)))))
        self.n = _add_particles(L, self.h, scene, state)

    def substep_via_mpmb(self, lib_path, n=1):
        """The drop-in for a mixed pool: one group per distinct (type, parameters), per-kind scalar offsets, n substeps on
        libmpmb (lib_path: libmpmb.so or its SIMT-emulator build).  Returns the number of survivors."""
        err = C.create_string_buffer(512)
        r = int(self.L.reft_substep_via_mpmb_mixed(self.h, str(lib_path).encode(), C.c_int(int(n)), err, C.c_int(512)))
        if r < 0:
            raise RuntimeError("mpmb through the reference's pool failed (%d): %s" % (r, err.value.decode(errors="replace")))
        return r


class MixedRefAsyncSolver(O.RefAsyncSolver):
    """The reference's AsyncMPM<3> object (pyoracle.RefAsyncSolver) holding several particle types; after route_through(lib)
    every substep its scheduler asks for goes to one libmpmb engine through reft_substep_via_mpmb_mixed."""

    def __init__(self, scene, state, unit_delta_t, max_units=8192, cfl_dt_mul=1.0, strength_dt_mul=1.0):
        self.L = L = ref_lib()
        self.res = np.ascontiguousarray(scene["res"], np.int32)
        g = np.ascontiguousarray(scene["gravity"], np.float32)
        self.h = C.c_void_p(L.reft_create_async(_p(self.res), C.c_float(scene["dx"]), _p(g), C.c_int(int(scene.get("particle_gravity", 1))),
                                                C.c_float(unit_delta_t), C.c_int64(int(max_units)), C.c_float(cfl_dt_mul), C.c_float(strength_dt_mul)))
        self.n = _add_particles(L, self.h, scene, state)
        L.reft_async_distribute(self.h)
