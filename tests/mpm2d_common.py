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


# ---------------------------------------------------------------------------------------------------- bench_2d.py's column
def bench_column(res):
    """bench_2d.py's sand column at any res: the column is res / 2 cells wide and high on the 8-cell floor, dt = 5e-6 * 1024 / res
    (bench_2d.SIZES at 1024 and 2048, where bench_2d.column itself is used).  Returns (state, dt, scene for the oracle)."""
    import bench_2d
    if res in bench_2d.SIZES:
        st, dt = bench_2d.column(res)
    else:
        cells, dt = res // 2, 5e-6 * 1024 / res
        lo = ((res - cells) // 2, bench_2d.FLOOR)
        x, mass, vol = scenes.lattice_block2d((res, res), lo, (lo[0] + cells, lo[1] + cells), density=400.0)
        st = scenes.make_state2d(x, mass, vol, scenes.MAT_SAND)
    planes = [[0.0, 1.0, 0.0, -float(bench_2d.FLOOR)]]
    scene = dict(res=(res, res), dx=1.0 / res, dt=dt, gravity=(0.0, -10.0), particle_gravity=1, clean_boundary=1, apic_damping=0.0,
                 rpic_damping=0.0, mat_kind=np.array([scenes.MAT_SAND], np.int32), mat_params=scenes.material_params(scenes.MAT_SAND)[None],
                 sdf=scenes.planes_sdf2d((res, res), planes), friction=0.4, route=("planes", planes))
    return st, dt, scene


def _math2(a4):
    """Column-major [N, 4] -> [N, 2, 2] in math layout, fp64."""
    return np.asarray(a4, np.float64).reshape(-1, 2, 2).transpose(0, 2, 1)


def trial_F2d(scene, F, b):
    """The trial F = cdg F of G2P, cdg = I + dt b (-4 / dx), from the stored F and the substep's undamped apic_b, fp64."""
    S = -4.0 / float(np.float32(scene["dx"])) * float(scene["dt"])
    return (np.eye(2) + S * _math2(b)) @ _math2(F)


def sand_case2d(Ft, prm, ps):
    """SandParticle::project's case with d = 2 (0: expansion, tr >= 0; 1: inside the cone, dg <= 0; 2: projected onto it) of
    the trial F [N, 2, 2], in fp64: eps = log|sigma| - cohesion, tr = sum(eps) + logJp, hat = eps - tr / 2,
    dg = |hat| + (2 lambda + 2 mu) / (2 mu) tr alpha."""
    prm = np.asarray(prm, np.float64)
    s = np.linalg.svd(Ft, compute_uv=False)
    eps = np.log(np.maximum(np.abs(s), 1e-4)) - prm[3]
    tr = eps.sum(1) + np.asarray(ps, np.float64)
    hat = eps - tr[:, None] / 2
    dg = np.linalg.norm(hat, axis=1) + (2 * prm[1] + 2 * prm[0]) / (2 * prm[0]) * tr * prm[2]
    return np.where(tr >= 0, 0, np.where(dg <= 0, 1, 2))


def regime2d(S_seed, S, ref, grid_rast, scene):
    """The numbers that show S (the whole state, rows in id order) is bench_2d.py's developed collapse, in fp64: the floor
    nodes' Coulomb branches (collapse.floor_branches, whose third components are 0 on a 2-D grid), the sand cases of the
    return map on the trial F of the oracle's substep `ref` of S, the most particles in one cell, the centre of mass's drop
    and the footprint width (occupied columns of cells) relative to the seeded column, and the fraction still alive."""
    from tests.collapse import floor_branches
    dx = float(scene["dx"])
    out = floor_branches(grid_rast, scene["sdf"], float(scene["friction"]))
    case = sand_case2d(trial_F2d(scene, S["F"], ref["b"]), scene["mat_params"][0], S["ps"])
    out.update({"case%d" % c: int((case == c).sum()) for c in range(3)})
    cell = np.floor(np.asarray(S["x"], np.float64) / dx).astype(np.int64)
    _, counts = np.unique(cell[:, 0] * int(scene["res"][1]) + cell[:, 1], return_counts=True)
    out["ppc_max"] = int(counts.max())
    out["com_drop"] = float(np.asarray(S_seed["x"], np.float64)[:, 1].mean() - np.asarray(S["x"], np.float64)[:, 1].mean()) / dx

    def width(x):
        return len(np.unique(np.floor(np.asarray(x, np.float64)[:, 0] / dx)))
    out["footprint"] = width(S["x"]) / width(S_seed["x"])
    out["alive"] = len(S["x"]) / len(S_seed["x"])
    return out


# The regime guards of tests/test_gpu_zz_mpm2d_bench.py: about half of what its first H100 run measured (the table in its
# header; footprint: half of the growth over the seeded column); ppc_max > 4 is compaction beyond the lattice's 4 per cell.
# Every case of the return map and every Coulomb branch of the floor must be reached.  bench_2d's developed states by res:
GUARDS_FULL = {1024: dict(stick=480, slide=42, separate=9, case0=99000, case1=138000, case2=285000, ppc_max=4, com_drop=3.5, footprint=1.023),
               2048: dict(stick=930, slide=96, separate=39, case0=500000, case1=719000, case2=875000, ppc_max=4, com_drop=6.7, footprint=1.025)}
# the reduced columns by (res, simulated seconds); tests/test_mpm2d_collapse_host.py shows the fp32 oracle reaches the 64^2 ones
GUARDS_REDUCED = {(64, 0.05): dict(stick=26, slide=6, separate=3, case0=560, case1=120, case2=1360, ppc_max=4, com_drop=0.19, footprint=1.03),
                  (128, 0.05): dict(stick=56, slide=8, separate=4, case0=2100, case1=670, case2=5400, ppc_max=4, com_drop=0.39, footprint=1.015),
                  (128, 0.3): dict(stick=94, slide=16, separate=6, case0=1030, case1=1530, case2=5100, ppc_max=4, com_drop=7.0, footprint=1.39),
                  (256, 0.05): dict(stick=117, slide=12, separate=5, case0=8000, case1=3800, case2=20900, ppc_max=4, com_drop=0.79, footprint=1.023),
                  (256, 0.3): dict(stick=199, slide=32, separate=13, case0=2087, case1=7536, case2=21818, ppc_max=4, com_drop=14.3, footprint=1.44)}
