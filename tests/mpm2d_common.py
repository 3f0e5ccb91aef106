"""2-D scenes shared by the 2-D tests and tests/golden/make_mpm2d_golden.py: a seeded lattice block perturbed so that every
term of P2G, the grid update and G2P with the return map is exercised, as tests/common.py builds them in 3-D."""
import numpy as np

from taichi_mpm_b200 import scenes


def perturb2d(st, kind, dx, seed, strain=0.02, vel=0.5):
    """Random affine velocity field, apic_b, F perturbation and plastic scalars (the 2-D twin of common.perturb_state)."""
    rng = np.random.default_rng(seed)
    x = st["x"]
    n = len(x)
    A = rng.normal(size=(2, 2)) * vel * 4
    st["v"] = (rng.normal(size=2) * vel + (x - x.mean(0)) @ A.T + rng.normal(size=(n, 2)) * 0.05 * vel).astype(np.float32)
    st["b"] = (rng.normal(size=(n, 4)) * vel * dx * 0.1).astype(np.float32)
    if kind != scenes.MAT_WATER:
        st["F"] = (st["F"] + rng.normal(size=(n, 4)) * strain).astype(np.float32)
    if kind == scenes.MAT_SNOW:
        st["ps"] = (1.0 + rng.normal(size=n) * 0.02).astype(np.float32)
    if kind == scenes.MAT_WATER:
        st["ps"] = (1.0 + rng.normal(size=n) * 0.01).astype(np.float32)
    if kind == scenes.MAT_SAND:
        st["ps"] = (np.abs(rng.normal(size=n)) * 1e-3 * (rng.random(n) < 0.3)).astype(np.float32)
    if kind == scenes.MAT_VISCO:
        st["ps"] = (1000.0 * (0.2 + 1.6 * rng.random(n))).astype(np.float32)
    return st


def scene2d(kind, res=(32, 32), dx=None, blocks=None, gravity=(0.0, -10.0), levelset="floor", friction=0.4, clean_boundary=1,
            apic=0.0, rpic=0.0, dt=None, seed=0, strain=0.02, vel=0.5, jitter=0.2, particle_gravity=1, **matkw):
    """levelset: None; "floor" (a plane two thirds of a cell under the block); ("planes", planes[k, 4]); ("shapes", [...]);
    ("dense", [...]) (set_sdf of scenes.shapes_sdf2d).  The oracle always gets the dense twin."""
    res = tuple(int(r) for r in res)
    dx = float(np.float32(1.0 / res[0] if dx is None else dx))
    if blocks is None:
        lo = ((res[0] - 8) // 2, 9)
        blocks = [(lo, (lo[0] + 8, lo[1] + 8))]
    parts = [scenes.lattice_block2d(res, lo, hi, jitter=jitter, seed=seed + 1 + k, dx=dx) for k, (lo, hi) in enumerate(blocks)]
    x, mass, vol = (np.concatenate([p[i] for p in parts]) for i in range(3))
    st = perturb2d(scenes.make_state2d(x, mass, vol, kind), kind, dx, seed, strain, vel)
    if kind == scenes.MAT_VON_MISES and "yield_stress" not in matkw:
        matkw["yield_stress"] = 1.0
    if dt is None:
        dt = {scenes.MAT_SAND: 2e-5, scenes.MAT_WATER: 5e-5}.get(kind, 1e-4)
    scene = dict(res=res, dx=dx, dt=dt, gravity=tuple(float(g) for g in gravity), particle_gravity=particle_gravity,
                 clean_boundary=clean_boundary, apic_damping=apic, rpic_damping=rpic, mat_kind=np.array([kind], np.int32),
                 mat_params=scenes.material_params(kind, **matkw)[None], friction=0.0, sdf=None)
    if levelset == "floor":
        levelset = ("planes", [[0.0, 1.0, 0.0, -(blocks[0][0][1] + 0.6)]])
    if levelset is not None:
        route, desc = levelset
        scene["friction"] = friction
        scene["route"] = levelset
        scene["sdf"] = scenes.planes_sdf2d(res, desc) if route == "planes" else scenes.shapes_sdf2d(res, desc)
        if route == "planes":
            scene["planes"] = np.asarray(desc, np.float32).reshape(-1, 4)
    return scene, st


def state_of(got):
    """The engine's download as oracle input (rows in id order)."""
    st = {k: got[k].copy() for k in ("x", "v", "F", "b", "mass", "vol", "ps", "group")}
    st["alive"] = np.ones(len(st["x"]), np.uint8)
    return st
