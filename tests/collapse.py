"""The developed sand collapse that bench.py times, for the parity tests: the engine seeded as bench.py seeds it, the window
rule that lets the fp64 oracle check a few boxes of an 8 M state exactly, and the numbers that show a state really is the
developed collapse (tests/test_gpu_zz_collapse_parity.py, tests/test_collapse_window_host.py).

bench.py's default run (--warmup 20 --steps 200 --develop 20000) times the resting column over substeps 20 .. 220 (after
20 warm-up substeps), repeats those 200 with per-stage events, advances 20 000 substeps, warms up 20 more and times
substeps 20 440 .. 20 640; --dump-outputs writes the state after substep 20 640."""
import numpy as np

from taichi_mpm_b200 import capi, scenes, slab

NAME = "sand256"
QUIESCENT = 20        # the resting column: the end of the first warm-up
DEVELOPED = 20640     # the end of the collapse's timed region (bench.py's `developed_substeps`)
MARGIN = 2            # the quadratic stencil reaches nodes base .. base + 2


def scene_of(scale):
    """(scene with the floor's dense level set for the oracle, meta) of sand256 at `scale`."""
    cfg = scenes.config(NAME, scale, state=False)
    scene, meta = cfg["scene"], cfg["meta"]
    scene["clean_boundary"] = 1
    scene["sdf"] = scenes.planes_sdf(scene["res"], scene["planes"])
    return scene, meta


def _configure(e, scene, meta):
    e.set_material(0, meta["kind"], scene["mat_params"][0])
    e.set_planes(scene["planes"], scene["friction"])
    return e.seed_lattice(meta["lo"], meta["hi"], meta["vol"], meta["mass"], jitter=meta["jitter"], seed=meta["seed"])


def seeded_engine(scale, **kw):
    """bench.py's SlabJob at `scale`: the column seeded on the device (mpmb_seed_lattice), nothing uploaded, so that every
    later substep runs on the incremental ordering the engine keeps.  kw: rank, world, tile_z0, tile_z1, ... of
    capi.Engine.  Returns (engine, scene, meta, particles seeded)."""
    scene, meta = scene_of(scale)
    e = capi.Engine(scene["res"], scene["dx"], scene["dt"], scene["gravity"], scene["particle_gravity"], True, **kw)
    return e, scene, meta, _configure(e, scene, meta)


def seeded_state(scale):
    """The host twin of the seeded column (scenes.lattice_block_hashed, bit for bit what mpmb_seed_lattice writes)."""
    scene, meta = scene_of(scale)
    ids, x, mass, vol = scenes.lattice_block_hashed(scene["res"], meta["lo"], meta["hi"], meta["density"], meta["jitter"], meta["seed"])
    st = scenes.make_state(x, mass, vol, meta["kind"])
    st["id"] = ids
    return scene, meta, st


def port_collapse(scale, nsub):
    """The seeded column advanced `nsub` substeps by the fp32 OpenMP port: (scene, live state with the seeding ids)."""
    from oracle import pyoracle as O
    scene, _, st = seeded_state(scale)
    f = O.FastOracle(scene, st)
    f.substeps(nsub)
    alive = f.st["alive"].astype(bool)
    out = {k: np.ascontiguousarray(v[alive]) for k, v in f.st.items() if k != "alive"}
    out["id"] = st["id"][alive]
    return scene, out


def z_cuts(scale, world):
    """bench.py's slab cuts: slab.slab_partition of the seeded column's base tile layers."""
    scene, _, st = seeded_state(scale)
    return slab.slab_partition(slab.base_tile_z(st["x"][:, 2], scene["dx"]), slab.tile_layers(scene["res"][2]), world)


class SeededSlabs:
    """`world` z-slab engines of the seeded column in one process, connected through the engine's peer-memory buffers as
    bench.py --gpus N connects its ranks, the stages of a substep interleaved on one stream."""

    def __init__(self, scale, world, migrate_capacity=65536):
        self.world = world
        self.cuts = z_cuts(scale, world)
        self.eng, self.n = [], 0
        for rank, (z0, z1) in enumerate(self.cuts):
            e, self.scene, self.meta, n = seeded_engine(scale, rank=rank, world=world, tile_z0=z0, tile_z1=z1,
                                                        migrate_capacity=migrate_capacity)
            self.eng.append(e)
            self.n += n
        for r in range(world - 1):
            for k in (0, 1):
                self.eng[r].xchg_connect(k, 1, ptr=self.eng[r + 1].xchg_buffer(k, 0))
                self.eng[r + 1].xchg_connect(k, 0, ptr=self.eng[r].xchg_buffer(k, 1))
        self.faces = [[f for f in (0, 1) if 0 <= r + (1 if f else -1) < world] for r in range(world)]

    def _faces(self, call):
        for r, e in enumerate(self.eng):
            for f in self.faces[r]:
                call(e, f)

    def step(self, n):
        for _ in range(n):
            for e in self.eng:
                e.sort_particles_and_populate_grid()
                e.rasterize()
            self._faces(lambda e, f: e.halo_send(f))
            self._faces(lambda e, f: e.halo_recv(f))
            for e in self.eng:
                e.resample()
            self._faces(lambda e, f: e.migrate_send(f))
            self._faces(lambda e, f: e.migrate_recv(f))

    def union(self):
        parts = [e.download() for e in self.eng]
        U = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
        o = np.argsort(U["id"], kind="stable")
        return {k: v[o] for k, v in U.items()}

    def close(self):
        for e in self.eng:
            e.close()


# ---------------------------------------------------------------------------------------------------- the window rule
def base_nodes(x, dx):
    """The base node of every particle by the fp64 oracle's rule: int(x / dx - 0.5) in double precision."""
    X = np.asarray(x, np.float64) * (1.0 / float(dx))
    return (X - 0.5).astype(np.int64)


def window(S, lo, hi, margin=MARGIN, dx=None):
    """A node box [lo, hi) of a state S (dict of per-particle arrays; dx: the scene's cell size).  Returns
    (sub, mask, (nlo, nhi)):
      sub   the particles whose base node lies in [lo - margin, hi + margin);
      mask  over sub: the particles to compare, base node in [lo, hi);
      nodes the node box whose P2G sums and velocities are complete in sub: [lo, hi + 2).
    With margin = 2 every node a compared particle reads receives all its particles: the oracle's substep of sub is its
    substep of S for the compared particles and nodes (the visiting order of the contributions to a node is the same)."""
    lo, hi = np.asarray(lo, np.int64), np.asarray(hi, np.int64)
    base = base_nodes(S["x"], dx)
    near = ((base >= lo - margin) & (base < hi + margin)).all(1)
    sub = {k: np.ascontiguousarray(v[near]) for k, v in S.items()}
    mask = ((base[near] >= lo) & (base[near] < hi)).all(1)
    return sub, mask, (lo, hi + 2)


def box(a, nodes):
    """The node box `nodes` = (lo, hi) of a dense grid a[nx, ny, nz, ...]."""
    (x0, y0, z0), (x1, y1, z1) = nodes
    return a[x0:x1, y0:y1, z0:z1]


def clip_box(centre, size, res):
    """A node box of `size` nodes per axis around `centre`, inside the nodes a live particle can use as its base."""
    c = np.asarray(centre, np.int64)
    lo = np.clip(c - size // 2, 0, np.asarray(res) - 2 - size)
    return lo, lo + size


def floor_box(scene, band=3.0):
    """The node box of the floor band (phi in [-band, 0]) over the whole x-z extent: P2G's floor nodes."""
    res = np.asarray(scene["res"])
    d = -float(scene["planes"][0][3])
    y0, y1 = int(np.ceil(d - band)), int(np.floor(d))
    return np.array([0, y0, 0]), np.array([res[0] - 1, y1 - 1, res[2] - 1])   # complete nodes [lo, hi + 2)


# ---------------------------------------------------------------------------------------------------- the regime
def floor_branches(grid_rast, sdf, friction, band=3.0):
    """The Coulomb branch every floor-band node (phi in [-band, 0], mass > 0) takes in the grid update, from the P2G grid
    before projection (fp64): counts of sticking (the tangential velocity cancelled, scale = 0), sliding (Coulomb term
    active, 0 < scale < 1) and separating (moving off the floor) nodes."""
    g = np.asarray(grid_rast, np.float64)
    s = np.asarray(sdf, np.float64)
    m = g[..., 3]
    sel = (m > 0) & (s[..., 3] >= -band) & (s[..., 3] <= 0)
    v = g[sel][:, :3] / m[sel][:, None]
    n = s[sel][:, :3]
    nn = (v * n).sum(1)
    tang = v - nn[:, None] * n
    tn = np.sqrt((tang ** 2).sum(1))
    scale = np.maximum(tn + np.minimum(nn, 0.0) * friction, 0.0) / np.maximum(1e-30, tn)
    return dict(stick=int((scale == 0).sum()), slide=int(((scale > 0) & (nn < 0)).sum()), separate=int((nn >= 0).sum()))


def _math(a9):
    return np.asarray(a9, np.float64).reshape(-1, 3, 3).transpose(0, 2, 1)


def regime(S_seed, S, P, ref, grid_rast, scene, stats):
    """The numbers that show S is the developed collapse.
    S_seed: the seeded state (x); S: the whole downloaded state; P: the state (S or a window of it) the oracle stepped,
    ref: the oracle's substep of P; grid_rast: its P2G grid, complete over the floor band; stats: get_ordering_stats()
    of the engine after the substep before S."""
    from tests.test_gpu_next_p2g import _sand_case
    dx = float(scene["dx"])
    out = dict(movers=int(stats["movers"]), hole_fraction=float(stats["movers"]) / max(float(stats["rows"]), 1.0))
    cell = np.floor(np.asarray(S["x"], np.float64) / dx).astype(np.int64)
    res = np.asarray(scene["res"], np.int64)
    _, counts = np.unique((cell[:, 0] * res[1] + cell[:, 1]) * res[2] + cell[:, 2], return_counts=True)
    out["ppc_max"] = int(counts.max())
    out["ppc_p999"] = float(np.percentile(counts, 99.9))
    out.update(floor_branches(grid_rast, scene["sdf"], float(scene["friction"])))
    S_ = -4.0 / float(np.float32(dx)) * scene["dt"]
    Ft = (np.eye(3) + S_ * _math(ref["b"])) @ _math(P["F"])
    case, _ = _sand_case(Ft, np.asarray(scene["mat_params"][0], np.float64), np.asarray(P["ps"], np.float64))
    out.update({"case%d" % c: int((case == c).sum()) for c in range(3)})
    sig = np.concatenate([np.linalg.svd(_math(S["F"][i:i + (1 << 20)]), compute_uv=False) for i in range(0, len(S["F"]), 1 << 20)])
    out["resting"] = float((np.abs(np.log(sig)).max(1) < 1e-3).mean())
    out["ps_max"] = float(np.abs(S["ps"]).max())
    out["com_drop"] = float(np.asarray(S_seed["x"], np.float64)[:, 1].mean() - np.asarray(S["x"], np.float64)[:, 1].mean()) / dx

    def footprint(x):
        c = np.floor(np.asarray(x, np.float64)[:, [0, 2]] / dx).astype(np.int64)
        return len(np.unique(c[:, 0] * res[2] + c[:, 1]))
    out["footprint"] = footprint(S["x"]) / footprint(S_seed["x"])
    out["alive"] = len(S["x"]) / len(S_seed["x"])     # the flow reaches the clean_boundary band: particles are deleted
    return out
