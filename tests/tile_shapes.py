"""Scenes built tile by tile for the tile walks of k_p2g, k_grid and k_g2p (tests/test_gpu_tile_walk.py), and the guards
that prove each scene reaches the shapes where those loops change branch.

A tile is 4x4x4 cells of BASE nodes: particle x lies in tile i along an axis when int(x / dx - 0.5) // 4 == i, so tile i
spans x / dx in [4 i + 0.5, 4 i + 4.5).  The generator puts prescribed particle counts into chosen tiles of a res-64 grid,
at least MARGIN cells from the tile faces, except in crossing bands.  Whole lanes of tiles move along +x at one velocity
U, so a particle of a band at distance d below a +x face crosses it in substep ceil(d / DELTA): G2P gives a particle the
grid's velocity, which for a uniformly moving lane is U.  Lanes are one tile apart from each other and from the resting
tiles, so that no grid node is shared between a lane and anything moving at another velocity.

The guards rebuild each substep's layout in numpy from the engine's downloaded states, by the rule of k_order_c:
- the rows of tile t in substep s + 1 (which moves x_s to x_{s+1}) are its run, the rows it wrote in substep s (the
  particles with key(x_{s-1}) == t), followed by its arrivals (key(x_s) == t, key(x_{s-1}) != t);
- a run row whose particle left the tile or died is a hole;
- slots follow the dense tile index (x nt1 + y) nt2 + z; out_begin is the exclusive scan of stay + arrivals, and the
  next substep's run_begin is this out_begin;
- after an upload every particle is an arrival (no run).
They then list which edge categories occurred; a category that stops occurring fails the test that uses the scene."""
import numpy as np

from taichi_mpm_b200 import scenes
from tests import common as T

RES = 64
NT = RES // 4
DX = 1.0 / RES
DT = 2e-5                     # sand's substep
U = 2.5                       # lane velocity along +x
DELTA = U * DT / DX           # cells a lane moves per substep (0.0032)
MARGIN = 0.05                 # cells between a particle that does not cross and the tile faces
NSUB = 6
P2G_CH, G2P_CH = 576, 256     # rows per chunk of k_p2g and k_g2p (csrc/mpmb_engine.cu)
G2P_CTAS_PER_SM = 5           # k_g2p's __launch_bounds__(BLOCK, 5): its grid is SMs x 5
KINDS = (scenes.MAT_SAND, scenes.MAT_JELLY)

# run lengths around warp multiples, the k_g2p chunk (256) and its multiples, the k_p2g chunk (576) and its double
RUN_LENGTHS = (1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 511, 512, 513, 575, 576, 577, 767, 768, 769, 1151, 1152, 1153, 1700)
ARRIVALS_ONLY = (1, 255, 256, 257, 600)


def _band(rng, n, tile, d_lo, d_hi):
    """n positions (grid units) in `tile`, x at a distance in (d_lo, d_hi) cells below its +x face, y and z inside."""
    X = _inside(rng, n, tile)
    X[:, 0] = 4 * tile[0] + 4.5 - rng.uniform(d_lo, d_hi, n)
    return X


def _inside(rng, n, tile, x_lo=None):
    lo = 4 * np.asarray(tile, np.float64) + 0.5 + MARGIN
    hi = 4 * np.asarray(tile, np.float64) + 4.5 - MARGIN
    if x_lo is not None:
        lo[0] = x_lo
    return rng.uniform(lo, hi, (n, 3))


def _crossing(rng, tile, schedule):
    """Band particles of `tile` that cross its +x face in the given substeps: schedule = {substep: count}."""
    parts = [_band(rng, n, tile, (s - 0.7) * DELTA, (s - 0.3) * DELTA) for s, n in sorted(schedule.items()) if n]
    return np.concatenate(parts) if parts else np.zeros((0, 3))


def lanes():
    """(first tile, [(resting count, crossing schedule) per tile along +x]) of every moving lane; the tile after the last
    one is empty until the lane's bands reach it."""
    L = []
    for n in ARRIVALS_ONLY:                                    # a band that all crosses in substep 1: an arrivals-only tile
        L.append([(0, {1: n})])
    L.append([(100, {1: 20, 3: 5}), (0, {1: 40})])             # the 2nd tile's run is all holes in substep 2, with 20 arrivals
    every = {s: 12 for s in range(1, NSUB)}
    out = {2: 3, 3: 3, 4: 3, 5: 3}                             # holes in the last chunk of a multi-chunk run
    for bulk in (240, 248, 556, 568, 750, 1138):               # runs of bulk + 12: run + arrivals across 256, 576, 768, 1152
        L.append([(50, every), (bulk, out)])
    return L


def tile_scene(run_lengths=RUN_LENGTHS, seed=5):
    """The scene and its state: resting tiles with the prescribed counts and filler tiles, the moving lanes, and one
    particle past clean_boundary's 7-cell band in a multi-chunk tile.  Groups 0 (sand) and 1 (fixed-corotated jelly) are
    interleaved at random."""
    rng = np.random.default_rng(seed)
    X, vel = [], []

    def add(P, u):
        X.append(P)
        vel.append(np.tile([u, 0.0, 0.0], (len(P), 1)))

    # resting tiles: y tiles 2-3, x and z tiles 2-13; the prescribed counts first, small filler tiles around them
    rest = [(tx, ty, tz) for ty in (2, 3) for tx in range(2, 14) for tz in range(2, 14)]
    order = rng.permutation(len(rest))
    for i, k in enumerate(order):
        n = run_lengths[i] if i < len(run_lengths) else int(rng.integers(8, 65))
        add(_inside(rng, n, rest[k]), 0.0)
    # the dead particle: x tile 1 (cells 4.5-8.5) holds 600 particles at x >= 7.05 and one at 6.9, which k_g2p deletes
    P = _inside(rng, 600, (1, 2, 7), x_lo=7.05)
    P[0, 0] = 6.9
    add(P, 0.0)
    # lanes: y tiles 6, 8, 10, 12 and z tiles 2, 4, .., 12, from x tile 3
    slots = [(ty, tz) for ty in (6, 8, 10, 12) for tz in range(2, 14, 2)]
    for (ty, tz), lane in zip(slots, lanes()):
        for j, (bulk, schedule) in enumerate(lane):
            tile = (3 + j, ty, tz)
            # the resting part of a moving tile keeps MARGIN + the whole run's travel below the +x face
            P = _inside(rng, bulk, tile)
            P[:, 0] = np.minimum(P[:, 0], 4 * tile[0] + 4.5 - MARGIN - NSUB * DELTA)
            add(np.concatenate([P, _crossing(rng, tile, schedule)]), U)
    Xg = np.concatenate(X)
    x = (Xg * DX).astype(np.float32)
    n = len(x)
    vol = np.full(n, DX ** 3 / 8.0, np.float32)
    st = scenes.make_state(x, (vol * np.float32(400.0)).astype(np.float32), vol, scenes.MAT_SAND)
    st["group"] = rng.integers(0, 2, n).astype(np.int32)
    st["ps"] = np.zeros(n, np.float32)
    for g, kind in enumerate(KINDS):
        sel = np.nonzero(st["group"] == g)[0]
        sub = {k: np.ascontiguousarray(v[sel]) for k, v in st.items()}
        T.perturb_state(sub, kind, DX, seed + 7 * g)
        for key in ("b", "F", "ps"):
            st[key][sel] = sub[key]
    st["v"] = np.concatenate(vel).astype(np.float32)
    scene = dict(res=(RES, RES, RES), dx=DX, dt=DT, gravity=(0.0, -10.0, 0.0), particle_gravity=1, clean_boundary=1,
                 mat_kind=np.array(KINDS, np.int32), mat_params=np.stack([scenes.material_params(k) for k in KINDS]),
                 planes=None, friction=0.0, sdf=None)
    return scene, st


def tile_keys(x, res=RES):
    """Dense tile index of each position, as make_key computes it in fp32: base node int(x * inv_dx - 0.5), / 4."""
    inv_dx = np.float32(1.0) / np.float32(1.0 / res)
    X = np.asarray(x, np.float32) * inv_dx
    b = (X - np.float32(0.5)).astype(np.int64) // 4
    nt = res // 4
    return (b[:, 0] * nt + b[:, 1]) * nt + b[:, 2]


def layout(states, res=RES):
    """Per substep s = 1 .. len(states) - 1, the tile layout the engine walked, from the states before each substep
    (states[0] the upload, states[s] after s substeps; dicts with "id" and "x").  Returns a list of dicts of dense
    per-tile arrays: run_begin, run_len, stay, arr, holes, and `dead`, the tiles in which a particle died."""
    ntot = (res // 4) ** 3
    out = []
    prev_keys = None
    for s in range(len(states) - 1):
        a, b = states[s], states[s + 1]
        ka = tile_keys(a["x"], res)
        tot = np.bincount(ka, minlength=ntot)
        if prev_keys is None:
            run_len = np.zeros(ntot, np.int64)
            run_begin = np.zeros(ntot, np.int64)
            arr = tot
        else:
            pid, pk = prev_keys
            kp = pk[np.searchsorted(pid, a["id"])]  # the key each particle had one substep earlier (no appends)
            run_len = np.bincount(pk, minlength=ntot)
            run_begin = np.concatenate([[0], np.cumsum(run_len)[:-1]])
            arr = np.bincount(ka[kp != ka], minlength=ntot)
        stay = tot - arr
        died = ~np.isin(a["id"], b["id"])
        out.append(dict(run_begin=run_begin, run_len=run_len, stay=stay, arr=arr, holes=run_len - stay,
                        dead=np.bincount(ka[died], minlength=ntot)))
        prev_keys = (np.asarray(a["id"]), ka)
    return out


def categories(lay):
    """The edge categories the layouts reach, and the fewest active tiles of any substep."""
    found = set()
    min_active = None
    for s, L in enumerate(lay, start=1):
        run_len, arr, stay, holes = L["run_len"], L["arr"], L["stay"], L["holes"]
        tot = run_len + arr
        act = np.nonzero(stay + arr)[0]
        min_active = len(act) if min_active is None else min(min_active, len(act))
        for t in act:
            rl, ar, n = int(run_len[t]), int(arr[t]), int(tot[t])
            if ar == 0:
                found.add(("run_len", rl if rl < 1600 else "~1700" if rl < 1800 else rl))
            if rl == 0 and s >= 2:
                found.add(("arrivals_only", ar if ar < 590 else "~600" if ar < 610 else ar))
            if rl > 0 and stay[t] == 0 and ar > 0:
                found.add(("holes_only_run_with_arrivals",))
            if rl > G2P_CH and holes[t] > 0:
                found.add(("holes_in_multi_chunk_run",))
            if L["dead"][t] and n > G2P_CH:
                found.add(("dead_in_multi_chunk_tile",))
            for ch, name in ((G2P_CH, "g2p"), (P2G_CH, "p2g")):
                if 0 < rl < ch < n:
                    found.add((name, "chunk_end_in_arrivals"))
                for c0 in range(ch, n, ch):   # later chunks that hold run rows and arrivals
                    if c0 < rl < min(c0 + ch, n):
                        found.add((name, "run_arrival_boundary_in_later_chunk"))
            if rl > 0:
                found.add(("sh", int(run_begin_shift(L, t))))
                if n > G2P_CH:
                    found.add(("sh_multi_chunk", int(run_begin_shift(L, t))))
    return found, min_active


def run_begin_shift(L, t):
    return L["run_begin"][t] & 3


def required():
    """Every category the tile-walk scene must reach."""
    req = {("run_len", n) for n in RUN_LENGTHS if n < 1600} | {("run_len", "~1700")}
    req |= {("arrivals_only", n) for n in ARRIVALS_ONLY if n < 590} | {("arrivals_only", "~600")}
    req |= {("holes_only_run_with_arrivals",), ("holes_in_multi_chunk_run",), ("dead_in_multi_chunk_tile",)}
    req |= {(k, c) for k in ("g2p", "p2g") for c in ("chunk_end_in_arrivals", "run_arrival_boundary_in_later_chunk")}
    req |= {(k, s) for k in ("sh", "sh_multi_chunk") for s in range(4)}
    return req


def missing(states, res=RES):
    """Required categories that the run given by `states` did not reach, and its fewest active tiles."""
    found, min_active = categories(layout(states, res))
    return sorted(required() - found, key=str), min_active
