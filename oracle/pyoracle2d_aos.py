"""ctypes front-end of the 2-D drop-in (oracle/transfer2d_aos_ref.cpp -> _ref/libtransfer2d_aos_ref.so, built only where the
reference tree exists): the reference's own MPM<2> object of oracle/pyoracle2d.py, loaded from that library, whose substeps
can be handed to libmpmb through mpmb_upload_aos / mpmb_download_aos on its own ParticleContainer<2> pool.

TEST INFRASTRUCTURE ONLY: imported by tests/.  The product package never imports this module.  The library is built with the
command line of oracle/pyoracle2d.py's _ref/libtransfer2d_ref.so.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pyoracle2d as O2
from oracle.pyoracle import N_MAT_PARAMS, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF = None
REFERENCE = O2.REFERENCE
REF_LIB = os.path.join(_HERE, "_ref", "libtransfer2d_aos_ref.so")
_CXX = O2._CXX


def ref_available():
    return os.path.exists(REF_LIB) or os.path.exists(os.path.join(REFERENCE, "src", "mpm.cpp"))


def ref_build(force=False):
    """_ref/libtransfer2d_aos_ref.so: transfer2d_aos_ref.cpp (which includes transfer2d_ref.cpp and transfer_ref.cpp) against the
    reference's sources where they lie."""
    stub = os.path.join(_HERE, "taichi_stub")
    deps = [os.path.join(_HERE, f) for f in ("transfer2d_aos_ref.cpp", "transfer2d_ref.cpp", "transfer_ref.cpp")]
    deps += [os.path.join(os.path.dirname(_HERE), "include", "mpmb.h")]
    deps += [os.path.join(d, f) for d, _, fs in os.walk(stub) for f in fs if f.endswith(".h")]
    if not (force or O2._stale(REF_LIB, deps)):
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
        L = C.CDLL(REF_LIB if os.path.exists(REF_LIB) and not os.path.exists(os.path.join(REFERENCE, "src")) else ref_build())
        L.reft2_create.restype = C.c_void_p
        L.reft2_substep.restype = C.c_int64
        L.reft2_add_particles.restype = C.c_int64
        L.reft2_num_particles.restype = C.c_int64
        L.reft2_substep_via_mpmb.restype = C.c_int64
        _REF = L
    return _REF


# the order of MpmbAosLayout's int32 fields
LAYOUT_FIELDS = ("stride", "off_pos", "off_v_and_m", "off_dg_e", "off_apic_b", "col_pitch", "off_vol", "off_scalar")


def aos_layout(kind=-1):
    """The reference's ParticleContainer<2> slot layout (reft2_aos_layout) as an int32[12] in MpmbAosLayout's field order:
    kind >= 0 the single-offset layout of that type, -1 the per-kind layout of a mixed pool."""
    out = np.zeros(12, np.int32)
    ref_lib().reft2_aos_layout(C.c_int(int(kind)), _p(out))
    return out


class AosRefSolver2D(O2.RefSolver2D):
    """The reference's MPM<2> object (pyoracle2d.RefSolver2D) built from this module's library, with any number of materials:
    row k of `state` becomes particle k under the type and parameters of its group (state["group"], default 0)."""

    def __init__(self, scene, state):
        self.L = L = ref_lib()
        f32 = np.float32
        self.res = np.ascontiguousarray(scene["res"][:2], np.int32)
        g = np.ascontiguousarray(scene["gravity"][:2], f32)
        self.h = C.c_void_p(L.reft2_create(_p(self.res), C.c_float(scene["dx"]), C.c_float(scene["dt"]), _p(g),
                                           C.c_int(int(scene.get("particle_gravity", 1))), C.c_int(int(scene.get("clean_boundary", 1))),
                                           C.c_float(scene.get("apic_damping", 0.0)), C.c_float(scene.get("rpic_damping", 0.0))))
        kinds = np.asarray(scene["mat_kind"], np.int32)
        st = {k: np.ascontiguousarray(state[k], f32) for k in ("x", "v", "F", "b", "mass", "vol", "ps")}
        self.n = len(st["x"])
        group = np.asarray(state.get("group", np.zeros(self.n, np.int32)), np.int64)
        cuts = np.flatnonzero(np.diff(group)) + 1
        for lo, hi in zip(np.r_[0, cuts], np.r_[cuts, self.n]):   # runs of one group, in row order: ids = rows
            gi = int(group[lo])
            prm = np.zeros(N_MAT_PARAMS, f32)
            prm[: len(scene["mat_params"][gi])] = scene["mat_params"][gi]
            run = {k: np.ascontiguousarray(a[lo:hi]) for k, a in st.items()}
            assert L.reft2_add_particles(self.h, C.c_int(int(kinds[gi])), _p(prm), C.c_int64(hi - lo), _p(run["x"]), _p(run["v"]), _p(run["mass"]),
                                         _p(run["vol"]), _p(run["F"]), _p(run["b"]), _p(run["ps"])) == hi - lo
        if scene.get("planes") is not None:
            pl = np.ascontiguousarray(np.asarray(scene["planes"], f32).reshape(-1, 4)[:, [0, 1, 3]])
            L.reft2_set_planes(self.h, C.c_int(len(pl)), _p(pl), C.c_float(scene.get("friction", 0.0)))

    def substep_via_mpmb(self, lib_path, n=1):
        """The 2-D drop-in: n substeps of this MPM<2> object on libmpmb (lib_path: libmpmb.so or its SIMT-emulator build), its
        pool and `particles` handed over through mpmb_upload_aos and written back through mpmb_download_aos.  Returns the
        number of survivors."""
        err = C.create_string_buffer(512)
        r = int(self.L.reft2_substep_via_mpmb(self.h, str(lib_path).encode(), C.c_int(int(n)), err, C.c_int(512)))
        if r < 0:
            raise RuntimeError("mpmb through the reference's 2-D pool failed (%d): %s" % (r, err.value.decode(errors="replace")))
        return r
