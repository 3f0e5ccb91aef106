"""The device math header (taichi_mpm_b200/csrc/mpmb_math.cuh) compiled for sm_90a with the product's flags
(tests/device_math/device_math.cu) and run on the GPU against the fp64 oracle: the arithmetic test_host_math.py
checks with IEEE stand-ins, here with rsqrt.approx.ftz, __expf, __fdividef and nvcc's FMA contraction, over the
host-math CASES and the edge regimes of tests/material_states.py."""
import ctypes as C
import os

import numpy as np
import pytest

from taichi_mpm_b200 import scenes
from tests import material_states as MS
from tests import test_host_math as H
from tests.device_math import build_device_math


def test_device_math_compiles_for_sm90a():
    # CPU-side: the harness builds with the product's nvcc flags (the GPU tests below load it)
    import subprocess
    lib = build_device_math.build()
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump" if os.path.exists("/usr/local/cuda/bin/cuobjdump") else "cuobjdump", "-lelf", lib],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0 and "sm_90a" in out.stdout, out.stdout


@pytest.fixture(scope="module")
def dm():
    L = C.CDLL(build_device_math.build())
    for f in ("dm_material_step", "dm_plasticity", "dm_calculate_force", "dm_sand_step_series", "dm_eig_sym3"):
        getattr(L, f).restype = C.c_int
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def run_device_step(dm, kind, prm, F, cdg, ps, vol):
    n = len(F)
    Fd, psd, force = H._cm(F), ps.copy(), np.zeros((n, 9), np.float32)
    assert dm.dm_material_step(C.c_int64(n), C.c_int(kind), _p(prm), _p(H._cm(cdg)), _p(Fd), _p(psd), _p(vol), _p(force)) == 0
    return H._math(Fd), psd, H._math(force)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,regime,strain", H.edge_cases())
def test_sm90a_material_step_edges_match_oracle(dm, kind, regime, strain):
    F, cdg, ps, vol, prm, Fo, pso, fo = H.edge_batch(kind, regime, strain)
    Fd, psd, fd = run_device_step(dm, kind, prm, F, cdg, ps, vol)
    err = H.edge_errors(kind, regime, F, cdg, Fd, psd, fd, Fo, pso, fo)
    tol = dict(H.EDGE_TOL[regime])
    if regime == "rotated":
        tol["force"] = H.rotated_force_tol(kind, prm, cdg, F, ps, vol, fo)
    print("sm_90a", kind, regime, strain, {k: "%.2e" % v for k, v in err.items()})
    for k, v in err.items():
        assert v <= tol[k], (k, v, tol[k])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,kw,strain,rate", H.CASES)
def test_sm90a_material_step_matches_oracle(dm, kind, kw, strain, rate):
    # the host-math CASES, same states, same tolerances
    n = 400
    F, cdg, ps, vol = H._random_states(kind, n, 11 + kind, strain, rate)
    prm = H._params8(kind, **kw)
    Fd, psd, fd = run_device_step(dm, kind, prm, F, cdg, ps, vol)
    Fo, pso, fo = H._oracle_step(kind, prm.astype(np.float64), cdg, F, ps, vol)
    if kind != scenes.MAT_WATER:
        assert np.abs(Fd - Fo).max() <= 2e-5
    assert np.abs(psd - pso).max() <= 1e-5 * max(1.0, np.abs(pso).max())
    assert np.abs(fd - fo).max() <= 2e-4 * np.abs(fo).max()
    # and the two-call form (upload-time calculate_force after plasticity) agrees with the fused step
    F2, ps2, f2 = H._cm(F), ps.copy(), np.zeros((n, 9), np.float32)
    assert dm.dm_plasticity(C.c_int64(n), C.c_int(kind), _p(prm), _p(H._cm(cdg)), _p(F2), _p(ps2)) == 0
    assert dm.dm_calculate_force(C.c_int64(n), C.c_int(kind), _p(prm), _p(F2), _p(ps2), _p(vol), _p(f2)) == 0
    assert np.abs(H._math(F2) - Fd).max() <= 2e-6 * max(1.0, np.abs(Fd).max())
    assert np.abs(ps2 - psd).max() <= 2e-6 * max(1.0, np.abs(psd).max())


@pytest.mark.gpu
@pytest.mark.parametrize("strain", [1e-4, 1e-2])
def test_sm90a_sand_series_path_alone(dm, strain):
    # the decomposition-free path on its own, rotated states included: where it accepts a lane it must match the
    # oracle; it must refuse inverted elements (det Ft < 0), which only the eigen path un-inverts
    kind = scenes.MAT_SAND
    F, cdg, ps, vol = MS.states(kind, "rotated", 256, 3, strain)
    Fi, cdgi, psi, voli = MS.states(kind, "inverted", 64, 3)
    F, cdg, ps, vol = np.concatenate([F, Fi]), np.concatenate([cdg, cdgi]), np.concatenate([ps, psi]), np.concatenate([vol, voli])
    prm = H._params8(kind)
    n = len(F)
    Fd, psd, fd, ok = H._cm(F), ps.copy(), np.zeros((n, 9), np.float32), np.zeros(n, np.int32)
    assert dm.dm_sand_step_series(C.c_int64(n), _p(prm), _p(H._cm(cdg)), _p(Fd), _p(psd), _p(vol), _p(fd), _p(ok)) == 0
    Fo, pso, fo = MS.expected_batch(kind, prm, cdg, F, ps, vol)
    inv = np.linalg.det(np.einsum("nij,njk->nik", cdg.astype(np.float64), F.astype(np.float64))) < 0
    assert not ok[inv].any()
    acc = ok.astype(bool)
    assert acc.sum() >= 200
    scale = np.abs(fo[acc]).max()
    err_F, err_f = np.abs(H._math(Fd)[acc] - Fo[acc]).max(), np.abs(H._math(fd)[acc] - fo[acc]).max() / scale
    print("series", strain, "F %.2e force %.2e" % (err_F, err_f))
    assert err_F <= 2e-5 and np.abs(psd[acc] - pso[acc]).max() <= 1e-5
    assert err_f <= H.rotated_force_tol(kind, prm, cdg[acc], F[acc], ps[acc], vol[acc], fo[acc])


@pytest.mark.gpu
def test_sm90a_eigensystem(dm):
    # as test_host_math.py::test_device_eigensystem, plus F F^T - I of rotated states near a half turn
    rng = np.random.default_rng(5)
    n = 500
    A = rng.normal(size=(n, 3, 3))
    A = (A + np.transpose(A, (0, 2, 1))) * 0.5 * (10.0 ** rng.uniform(-5, 0, size=(n, 1, 1)))
    A[0] = 0.0
    A[1] = np.diag([1e-3, 1e-3, 1e-3])
    A[2] = np.diag([2e-3, 2e-3, -1e-3])
    A6 = np.ascontiguousarray(np.stack([A[:, 0, 0], A[:, 1, 1], A[:, 2, 2], A[:, 0, 1], A[:, 0, 2], A[:, 1, 2]], 1), np.float32)
    U9, e3 = np.zeros((n, 9), np.float32), np.zeros((n, 3), np.float32)
    assert dm.dm_eig_sym3(C.c_int64(n), _p(A6), _p(U9), _p(e3)) == 0
    U = H._math(U9).astype(np.float64)
    rec = np.einsum("nij,nj,nkj->nik", U, e3.astype(np.float64), U)
    nrm = np.maximum(np.abs(A).reshape(n, -1).max(1), 1e-30)
    assert (np.abs(rec - A).reshape(n, -1).max(1) <= 4e-6 * nrm + 1e-12).all()
    assert np.abs(np.einsum("nji,njk->nik", U, U) - np.eye(3)[None]).max() <= 5e-6
    assert np.abs(np.linalg.det(U) - 1).max() <= 1e-5           # a rotation: the sign convention of DESIGN.md §2 needs it
