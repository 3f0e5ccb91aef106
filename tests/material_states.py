"""Deformation gradients at the edges of the constitutive models: one seeded generator for the host build of
the device math header (test_host_math.py), its sm_90a build (test_gpu_device_math.py) and the engine's own
kernels (test_gpu_material_edges.py, test_material_edges_simt.py).

`states(kind, regime, n, seed)` returns float32 batches (F, cdg, ps, vol), math layout [n,3,3]:
  rotated        F = R (I + N(0, strain)), R uniform on SO(3), a quarter of them within 1e-3 of a half turn
  large          sigma log-uniform in [0.2, 5]; sand with |F F^T - I| within 1e-3 of the series' 0.15 limit;
                 snow beyond both clamps with Jp at 0.6 and at 20
  degenerate     R diag(a, a, b) Q^T, a R Q^T, exact rotations, and inverted R diag(a, a, -b) Q^T, b < a
  near_singular  R diag(a, b, s_min) Q^T with s_min in {1e-2, 1e-3, 1e-4, 0}
  inverted       det F < 0, the smallest |sigma| at least 1e-2 below the next: R in SO(3) is unique
Everything but `rotated` and `inverted` uses cdg = I so that the constructed spectrum is the one the step sees.
"""
import numpy as np

from taichi_mpm_b200 import scenes

KINDS = (scenes.MAT_LINEAR, scenes.MAT_JELLY, scenes.MAT_SNOW, scenes.MAT_WATER, scenes.MAT_SAND, scenes.MAT_ELASTIC,
         scenes.MAT_VON_MISES, scenes.MAT_VISCO)
REGIMES = ("rotated", "large", "degenerate", "near_singular", "inverted")
HENCKY = (scenes.MAT_SAND, scenes.MAT_ELASTIC, scenes.MAT_VON_MISES)
# strain of the rotated regime per kind: the moderate strains of the host-math CASES; sand on the series path (1e-4)
# and with more series terms (1e-2)
ROTATED_STRAIN = {scenes.MAT_LINEAR: (0.02,), scenes.MAT_JELLY: (0.05,), scenes.MAT_SNOW: (0.02,), scenes.MAT_WATER: (0.0,),
                  scenes.MAT_SAND: (1e-4, 1e-2), scenes.MAT_ELASTIC: (0.05,), scenes.MAT_VON_MISES: (0.02,), scenes.MAT_VISCO: (0.05,)}
NEAR_SINGULAR = (1e-2, 1e-3, 1e-4, 0.0)
VOL = (1.0 / 256) ** 3 / 8


def rotations(rng, n, near_pi=0.25):
    """uniform rotations (unit quaternions); the first round(near_pi * n) turn by pi - U(0, 1e-3)"""
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    m = int(round(near_pi * n))
    if m:
        ax = rng.normal(size=(m, 3))
        ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        half = 0.5 * (np.pi - rng.uniform(0, 1e-3, size=m))
        q[:m] = np.concatenate([np.cos(half)[:, None], np.sin(half)[:, None] * ax], 1)
    w, x, y, z = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], 1)


def plastic_scalar(kind, rng, n):
    """Jp / j / logJp / visco_tau around the values a run carries (as tests/test_host_math.py::_random_states)"""
    if kind == scenes.MAT_SNOW:
        return 1.0 + rng.normal(size=n) * 0.05
    if kind == scenes.MAT_WATER:
        return 1.0 + rng.normal(size=n) * 0.02
    if kind == scenes.MAT_SAND:
        return np.abs(rng.normal(size=n)) * 2e-3 * (rng.random(n) < 0.5)
    if kind == scenes.MAT_VISCO:
        return 1000.0 * (0.5 + rng.random(n))
    return np.zeros(n)


def _usv(rng, sig):
    n = len(sig)
    return np.einsum("nij,nj,nkj->nik", rotations(rng, n, 0.0), sig, rotations(rng, n, 0.0))


def states(kind, regime, n=256, seed=0, strain=None):
    rng = np.random.default_rng(seed * 7919 + 101 * kind + REGIMES.index(regime))
    eye = np.broadcast_to(np.eye(3), (n, 3, 3))
    cdg = eye.copy()
    ps = plastic_scalar(kind, rng, n)
    if regime == "rotated":
        strain = ROTATED_STRAIN[kind][0] if strain is None else strain
        F = np.einsum("nij,njk->nik", rotations(rng, n), eye + rng.normal(size=(n, 3, 3)) * strain)
        cdg = eye + rng.normal(size=(n, 3, 3)) * min(1e-3, max(strain, 1e-5))
    elif regime == "large":
        if kind == scenes.MAT_SAND:
            # |F F^T - I|_F = 0.15 + U(-1e-3, 1e-3): both sides of the series' limit, under rotation
            d = rng.normal(size=(n, 3))
            d *= (0.15 + rng.uniform(-1e-3, 1e-3, size=(n, 1))) / np.linalg.norm(d, axis=1, keepdims=True)
            F = _usv(rng, np.sqrt(1.0 + d))
        elif kind == scenes.MAT_SNOW:
            # every axis beyond a clamp (theta_c = 2.5e-2, theta_s = 7.5e-3), Jp at both bounds
            sig = np.where(rng.random((n, 3)) < 0.5, rng.uniform(0.9, 0.97, (n, 3)), rng.uniform(1.01, 1.1, (n, 3)))
            F = _usv(rng, sig)
            ps = np.where(rng.random(n) < 0.5, 0.6, 20.0)
        else:
            F = _usv(rng, np.exp(rng.uniform(np.log(0.2), np.log(5.0), size=(n, 3))))
    elif regime == "degenerate":
        a = rng.uniform(0.8, 1.2, size=n)
        b = a * rng.uniform(0.85, 0.97, size=n)
        form = np.arange(n) % 4
        sig = np.stack([a, a, np.where(form == 0, b, np.where(form == 3, -b, a))], 1)
        sig[form == 2] = 1.0                                                  # exact rotations
        F = _usv(rng, sig)
    elif regime == "near_singular":
        smin = np.array(NEAR_SINGULAR)[np.arange(n) % len(NEAR_SINGULAR)]
        F = _usv(rng, np.stack([rng.uniform(1.05, 1.3, n), rng.uniform(0.75, 0.95, n), smin], 1))
    elif regime == "inverted":
        # |sigma| descending with gaps >= 0.05, the smallest negated
        s2 = rng.uniform(0.5, 1.0, n)
        s1 = s2 + rng.uniform(0.05, 0.3, n)
        s0 = s1 + rng.uniform(0.05, 0.3, n)
        F = _usv(rng, np.stack([s0, s1, -s2], 1))
        cdg = eye + rng.normal(size=(n, 3, 3)) * 1e-3
    else:
        raise ValueError(regime)
    vol = np.full(n, VOL)
    return F.astype(np.float32), np.ascontiguousarray(cdg, np.float32), ps.astype(np.float32), vol.astype(np.float32)


def min_abs_sigma(F):
    return np.linalg.svd(np.asarray(F, np.float64), compute_uv=False).min(-1)


# ---------------------------------------------------------------- fp64 expectation
def _approx_exponent(dt, m, depth=0):
    """ViscoParticle::approximate_exponent (src/particles.cpp:89-102), as the oracle restates it"""
    s = m * dt
    r = (s * 0.5 + np.eye(3)) @ s + np.eye(3)
    if np.linalg.det(r) > 0 or depth >= 16:
        return r
    t = _approx_exponent(dt * 0.5, m, depth + 1)
    return t @ t


def visco_abs_sigma(prm, cdg, F, ps, vol):
    """The device's visco step for any det: the oracle's return map (src/particles.cpp:104-137) on |sigma| of F^ (the
    reference's pow(det, 1/3) is NaN for det < 0), the reflection of F^ kept; |P(F_old)| and the stress of the new
    state are the fixed-corotated ones with R in SO(3) and signed J."""
    from oracle import pyoracle as O
    mu, la, nu, kappa, dt = (float(v) for v in prm[:5])
    P = -np.asarray(O.calculate_force(scenes.MAT_VISCO, prm, F, ps, 1.0, np.float64)) @ np.linalg.inv(F.T)
    pnorm = np.sqrt((P * P).sum())
    Fh = _approx_exponent(dt, (cdg - np.eye(3)) / dt) @ F
    w, U = np.linalg.eigh(Fh @ Fh.T)
    sg = np.sqrt(np.maximum(w, 0.0))
    gamma = min(max(dt * nu * (pnorm - ps) / pnorm, 0.0), 1.0) if pnorm > 1e-5 else 0.0
    det = sg.prod()
    scale = 1.0 / np.cbrt(det) if abs(det) > 1e-5 else 1.0
    mid = (sg * scale) ** gamma
    sn = np.clip(sg / np.where(np.abs(mid) > 1e-5, mid, 1.0), 0.1, 10.0)
    F1 = U @ np.diag(sn / sg) @ U.T @ Fh
    ps1 = ps + kappa * gamma * pnorm
    return F1, ps1, np.asarray(O.calculate_force(scenes.MAT_VISCO, prm, F1, ps1, vol, np.float64))


REFLECT = np.diag([1.0, 1.0, -1.0])


def expected_step(kind, prm, cdg, F, ps, vol):
    """fp64 plasticity(cdg) + calculate_force() of one state.  The oracle's (svd3 puts det F's sign on the smallest
    singular value, U, V in SO(3), as the reference's polar_decomp / svd do) wherever the reference is defined.  For an
    inverted element the Hencky kinds elastic and von Mises read |sigma| and keep the reflection: their step depends on
    F F^T only, so it is the oracle's step of F Q (Q a reflection, det F Q > 0) with Q taken off again on the right."""
    from oracle import pyoracle as O
    prm = np.asarray(prm, np.float64)
    cdg, F = np.asarray(cdg, np.float64), np.asarray(F, np.float64)
    if kind == scenes.MAT_VISCO and (np.linalg.det(F) < 0 or np.linalg.det(cdg @ F) < 0):
        return visco_abs_sigma(prm, cdg, F, float(ps), vol)
    if kind in (scenes.MAT_ELASTIC, scenes.MAT_VON_MISES) and np.linalg.det(cdg @ F) < 0:
        F1, ps1, f1 = expected_step(kind, prm, cdg, F @ REFLECT, ps, vol)
        return F1 @ REFLECT, ps1, f1
    F1, ps1 = O.plasticity(kind, prm, cdg, F, float(ps), np.float64)
    return np.asarray(F1), float(ps1), np.asarray(O.calculate_force(kind, prm, F1, ps1, float(vol), np.float64))


def expected_batch(kind, prm, cdg, F, ps, vol):
    out = [expected_step(kind, prm, cdg[i], F[i], ps[i], float(vol[i])) for i in range(len(F))]
    return np.array([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out])
