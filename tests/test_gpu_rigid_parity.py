"""The rigid-coupled (CPIC) transfers against the fp64 oracle.
a. One coupled substep for all eight material kinds (scripted and free plate), eight kinds interleaved in every rigid tile,
   grid gravity only.
b. The next coupled P2G after k_g2p_rigid, whose cached A and apic_b k_p2g_rigid turns back into dt * force for the bodies'
   impulses ((A - 4 m apic_b) * (-dx / 4)): all eight kinds after substep(1), (2) and (7) calls with host launches and with
   graph replay, and a fast rotating, drifting block where that recovery cancels and rows arrive in rigid tiles.
c. The transfer edges of the rigid kernels: two free bodies in one stencil, eleven bodies, every friction mode with a
   different one on each side of a body, the penalty window with and without the pushing force, the row strides of
   k_p2g_rigid.
d. Coupled runs against a chained fp64 oracle: 20 substeps of a scripted plate (graph replay and the per-substep contract),
   10 substeps of a free plate advanced on the device against HostRigidBody.advect.
Runs on the SIMT emulator too, in all three scheduling orders (tests/test_rigid_parity_simt.py).

Stress errors are measured as in tests/test_gpu_next_p2g.py: against the stress part of the result, the oracle's result minus
its result at F = I and the fresh plastic scalar.  That holds for the bodies too: at zero stress tf = 0, and the velocity
change a body takes from the rasterize loses exactly the stress term of its impulses."""
import numpy as np
import pytest

from taichi_mpm_b200 import scenes
from tests import common as T
from tests.test_gpu_next_p2g import GUARD, KINDS, _assert_grid, _free_state, _grid_errors, _math, _sand_case
from tests.test_gpu_rigid import G, _engine
from tests.test_gpu_rigid_motion import _host_bodies, _motion, _scripted_pose_table

pytestmark = pytest.mark.gpu

# one coupled substep against the oracle: grid relative to max(|p|, m); x absolute; v, apic_b relative to their largest
# component; F absolute; the plastic scalar as T.ps_err; a body's velocity change from the rasterize, from the resample and
# from the substep relative to the largest component of the oracle's change.  About 4-5 x the worst errors measured on an
# H100 and on the SIMT emulator (DESIGN §2), tighter than the shared single-substep tolerances of tests/common.py.
TOL_ONE = dict(grid=6e-6, x=8e-7, v=2.5e-5, b=4e-5, F=4e-6, ps=3e-5, body=3e-5)
# next coupled P2G: the grid's error relative to its stress part (measured worst 2.9e-4 on an H100, von Mises; 2.0e-4 on the
# emulator), and the body's change from the rasterize relative to the stress part of that change (measured worst 1.2e-3)
TOL_STRESS_RIGID = 1e-3
TOL_BODY_STRESS = 5e-3


def _kind_scene(kind, variant="dynamic", vel=0.3, j_floor=True):
    """The golden plate through a block of `kind` at its T.KIND_KW strain; water with half its particles at the j = 0.1 floor
    (`j_floor`; their pressure is 1e7 times that of j = 1)."""
    scene, st, rigid = G.golden_scene(variant, kind=kind, vel=vel)
    if kind == scenes.MAT_WATER and j_floor:
        st["ps"][::2] = 0.1
    return scene, st, rigid


def _rel(a, b, floor=1e-7):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), floor))


def _rigid_now(rigid, rs):
    """`rigid` with the pose, velocities, inverse masses and world inverse inertia the engine holds (get_rigid_state)."""
    out = dict(rigid)
    for k in ("position", "rot", "velocity", "angular_velocity", "inv_mass", "inv_inertia", "frictions"):
        out[k] = np.asarray(rs[k], np.float32)
    return out


def _pages(scene, rigid):
    """rigid_page_map (update_rigid_page_map, the rule test_rigid_pages_are_the_reference_s_including_its_one_sided_dilation
    pins): the 4x4x8-node blocks of the samples' base nodes and their {0,1}^3 upper neighbours.  Returns a boolean
    [nb_x, nb_y, nb_z] array."""
    res = np.asarray(scene["res"])
    nb = ((res[0] + 3) // 4 + 1, (res[1] + 3) // 4 + 1, (res[2] + 7) // 8 + 1)
    rid = rigid["sample_rigid"]
    rot = np.asarray(rigid["rot"], np.float64).reshape(-1, 3, 3).transpose(0, 2, 1)[rid]
    pos = np.asarray(rigid["position"], np.float64)[rid] + np.einsum("nij,nj->ni", rot, rigid["sample_offset"])
    base = np.floor(pos / scene["dx"] - 0.5).astype(int)
    page = np.zeros(nb, bool)
    for i in (0, 1):
        for j in (0, 1):
            for k in (0, 1):
                b = (base >> np.array([2, 2, 3])) + (i, j, k)
                ok = (b >= 0).all(1) & (b < nb).all(1)
                page[b[ok, 0], b[ok, 1], b[ok, 2]] = True
    return page


def _tile(scene, x):
    return np.floor(np.asarray(x, np.float64) / scene["dx"] - 0.5).astype(int) >> 2


def _in_rigid_tile(page, tiles):
    t = np.asarray(tiles)
    ok = (t >= 0).all(1) & (t[:, 0] < page.shape[0]) & (t[:, 1] < page.shape[1]) & ((t[:, 2] >> 1) < page.shape[2])
    out = np.zeros(len(t), bool)
    out[ok] = page[t[ok, 0], t[ok, 1], t[ok, 2] >> 1]
    return out


def _rigid_arena_nodes(scene, page):
    """The nodes of the arenas (6x6x6 nodes from 4 t) of every 4x4x4-node tile whose page is a rigid page."""
    nn = tuple(int(r) + 1 for r in scene["res"])
    mask = np.zeros(nn, bool)
    for tx, ty, pz in zip(*np.nonzero(page)):
        for tz in (2 * pz, 2 * pz + 1):
            mask[4 * tx: 4 * tx + 6, 4 * ty: 4 * ty + 6, 4 * tz: 4 * tz + 6] = True
    return mask


def _body_errors(rigid, r_eng, r_ref, floor=1e-4):
    out = {}
    for b in np.nonzero(np.asarray(rigid["inv_mass"]) > 0)[0]:
        for k, name in (("velocity", "dv"), ("angular_velocity", "dw")):
            d_ref = np.asarray(r_ref[k][b], np.float64) - rigid[k][b]
            d_eng = np.asarray(r_eng[k][b], np.float64) - rigid[k][b]
            if floor is None and not d_ref.any():      # no impulse (the resample's come from the penalty window only)
                out["%s%d" % (name, b)] = float(np.abs(d_eng).max())
                continue
            assert np.abs(d_ref).max() > (floor or 0.0), (b, k, d_ref)
            out["%s%d" % (name, b)] = _rel(d_eng, d_ref)
    return out


def _fmt(err):
    return {k: ("%.3g" % v if isinstance(v, float) else v) for k, v in err.items()}


# ---------------------------------------------------------------------------------------------------- a. one coupled substep
def coupled_substep(scene, st, rigid, label, tol=None):
    """One coupled substep, stage by stage, on the engine and the fp64 oracle; asserts the colours, the rasterized grid, the
    bodies' changes from the rasterize, from the resample and from the whole substep, and every particle's state.  `tol`
    overrides entries of TOL_ONE.  Returns (oracle state, engine state, oracle colour field)."""
    from oracle import pyoracle as O
    tol = dict(TOL_ONE, **(tol or {}))
    n = len(st["x"])
    ref, grid_rast, _, rref, cdf = O.substep_coupled(scene, st, rigid, np.float64)
    _, _, rp2g, _ = O.p2g_coupled(scene, st, rigid, np.float64)
    e = _engine(scene, st, rigid, states=st.get("states"))
    e.sort_particles_and_populate_grid()
    assert np.array_equal(e.download_cdf()["node_state"], cdf["node_state"])
    pc = e.get_particle_cdf(n)
    assert np.array_equal(pc["states"], ref["states"]) and np.array_equal(pc["near"], ref["near"]) and ref["near"].sum() > 0
    e.rasterize()
    g0 = e.download_grid(0).astype(np.float64)
    nb = len(rigid["inv_mass"])
    r1 = e.get_rigid_state(nb)
    e.resample()
    got = e.download()
    r2 = e.get_rigid_state(nb)
    e.close()
    ids = got["id"].astype(np.int64)
    assert np.array_equal(np.sort(ids), np.nonzero(ref["alive"])[0])
    pmax = max(np.abs(grid_rast[..., :3]).max(), grid_rast[..., 3].max())
    err = dict(grid=float(np.abs(g0 - grid_rast).max() / pmax), x=float(np.abs(got["x"] - ref["x"][ids]).max()),
               v=_rel(got["v"], ref["v"][ids]), b=_rel(got["b"], ref["b"][ids], 1e-30), F=float(np.abs(got["F"] - ref["F"][ids]).max()),
               ps=T.ps_err(got["ps"], ref["ps"][ids]), deleted=int(n - len(ids)))
    err.update({"p2g_" + k: v for k, v in _body_errors(rigid, r1, rp2g).items()})
    err.update({"g2p_" + k: v for k, v in _body_errors(_rigid_now(rigid, r1), r2, dict(velocity=rref["velocity"] - rp2g["velocity"] + r1["velocity"],
               angular_velocity=rref["angular_velocity"] - rp2g["angular_velocity"] + r1["angular_velocity"]), floor=None).items()})
    err.update({"sub_" + k: v for k, v in _body_errors(rigid, r2, rref).items()})
    print(label, _fmt(err))
    for k in ("grid", "x", "v", "b", "F", "ps"):
        assert err[k] <= tol[k], (k, err)
    for k, v in err.items():
        if k.startswith(("p2g_", "g2p_", "sub_")):
            assert v <= tol["body"], (k, err)
    for b in range(1, nb):
        if rigid["inv_mass"][b] == 0:      # scripted bodies take no impulse
            assert np.array_equal(r2["velocity"][b], rigid["velocity"][b]) and np.array_equal(r2["angular_velocity"][b], rigid["angular_velocity"][b])
    return ref, got, cdf


def _branch_counts(scene, st, rigid, ref):
    """Which material branches the oracle's substep took on particles of rigid pages that are not near a boundary (their stored
    apic_b is the B of their cdg, so the trial F = (I + S apic_b) F is known), with numpy."""
    kind = int(scene["mat_kind"][0])
    prm = scene["mat_params"][0].astype(np.float64)
    page = _pages(scene, rigid)
    sel = _in_rigid_tile(page, _tile(scene, st["x"])) & (ref["near"] == 0) & (ref["alive"] == 1)
    S_ = -4.0 / float(np.float32(scene["dx"])) * scene["dt"]
    Ft = (np.eye(3) + S_ * _math(ref["b"][sel])) @ _math(st["F"][sel])
    ps0 = st["ps"][sel].astype(np.float64)
    if kind == scenes.MAT_SAND:
        case, _ = _sand_case(Ft, prm, ps0)
        return {"expansion": int((case == 0).sum()), "inside": int((case == 1).sum()), "projected": int((case == 2).sum())}
    if kind == scenes.MAT_SNOW:
        s = np.linalg.svd(Ft, compute_uv=False)
        return {"compress_clamp": int((s.min(1) < 1 - prm[3]).sum()), "stretch_clamp": int((s.max(1) > 1 + prm[4]).sum())}
    if kind == scenes.MAT_WATER:
        return {"j_floor": int((ref["ps"][sel] == 0.1).sum()), "above": int((ref["ps"][sel] > 0.1).sum())}
    if kind == scenes.MAT_VON_MISES:
        eps = np.log(np.linalg.svd(Ft, compute_uv=False))
        n2 = ((eps - eps.mean(1, keepdims=True)) ** 2).sum(1)
        y = n2 > prm[2] / (2 * prm[0])
        return {"yield": int(y.sum()), "elastic": int((~y).sum())}
    return {"rigid_page_particles": int(sel.sum())}


@pytest.mark.parametrize("variant", ["kinematic", "dynamic"], ids=["scripted", "free"])
@pytest.mark.parametrize("name,kind", KINDS)
def test_coupled_substep_every_kind(name, kind, variant):
    scene, st, rigid = _kind_scene(kind, variant)
    # water next to a body: the pushing force makes tr(cdg) - 2, the factor of j, reach 25 in one substep, and j carries that
    # factor's relative rounding (measured 1.2e-5)
    ref, _, _ = coupled_substep(scene, st, rigid, "%s %s" % (name, variant), dict(ps=5e-5) if kind == scenes.MAT_WATER else None)
    counts = _branch_counts(scene, st, rigid, ref)
    print("  branches in rigid pages", counts)
    assert min(counts.values()) > 0, counts


def test_coupled_substep_kinds_interleaved_in_rigid_tiles():
    # every particle's material by the group of its tag: eight kinds interleaved row by row in the tiles of k_g2p_rigid
    from tests.test_gpu_next_p2g import mixed_state
    kinds = [k for _, k in KINDS]
    scene, _, rigid = G.golden_scene("dynamic")
    st = mixed_state(32, (13, 9, 13), (19, 15, 19), kinds, seed=5, strain=0.01, vel=0.3)
    scene = dict(scene, mat_kind=np.array(kinds, np.int32), mat_params=np.array([scenes.material_params(k, **({"kappa": 0.3} if k == scenes.MAT_VISCO else {}))
                                                                               for k in kinds], np.float32), dt=2e-5)
    coupled_substep(scene, st, rigid, "8 kinds interleaved")
    tiles = _tile(scene, st["x"])
    inside = _in_rigid_tile(_pages(scene, rigid), tiles)
    key = (tiles[:, 0] * 64 + tiles[:, 1]) * 64 + tiles[:, 2]
    per_tile = [len(np.unique(st["group"][inside & (key == k)])) for k in np.unique(key[inside])]
    print("  groups per rigid tile", sorted(per_tile))
    assert len(per_tile) >= 8 and min(per_tile) == 8, per_tile      # every rigid tile holds all eight kinds


def test_coupled_substep_with_grid_gravity_only():
    # particle_gravity = 0: no kick in either rigid kernel (pv of k_g2p_rigid, v of k_p2g_rigid), gravity on the grid instead
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY, "dynamic")
    scene = dict(scene, particle_gravity=0, gravity=(3.0, -40.0, 5.0))
    coupled_substep(scene, st, rigid, "grid gravity")


# ---------------------------------------------------------------------------------------------------- b. the next coupled P2G
def next_p2g_coupled(e, scene, rigid, n, label, tol=TOL_STRESS_RIGID, guard=GUARD, tol_body=TOL_BODY_STRESS):
    """The engine's next coupled P2G (grid and the bodies' change from the rasterize) against pyoracle.p2g_coupled of the state,
    colours and bodies downloaded between substeps; then the engine finishes the substep.  Returns the errors."""
    from oracle import pyoracle as O
    nb = len(rigid["inv_mass"])
    S = e.download()
    S["states"] = e.get_particle_cdf(n)["states"][S["id"].astype(np.int64)]
    R = _rigid_now(rigid, e.get_rigid_state(nb))
    e.sort_particles_and_populate_grid()
    e.rasterize()
    g = e.download_grid(0).astype(np.float64)
    r_eng = e.get_rigid_state(nb)
    e.resample()
    _, g_ref, r_ref, _ = O.p2g_coupled(scene, S, R, np.float64)
    _, g_free, r_free, _ = O.p2g_coupled(scene, _free_state(scene, S), R, np.float64)
    err = _grid_errors(g, g_ref, g_free)
    arena = _rigid_arena_nodes(scene, _pages(scene, R)) & (g_ref[..., 3] > 0)
    err.update({"rigid_" + k: v for k, v in _grid_errors(g, g_ref, g_free, arena).items()})
    for b in np.nonzero(R["inv_mass"] > 0)[0]:
        for k, name in (("velocity", "dv"), ("angular_velocity", "dw")):
            d_ref, d_free = r_ref[k][b] - R[k][b], r_free[k][b] - R[k][b]
            d_eng = np.asarray(r_eng[k][b], np.float64) - R[k][b]
            stress = np.abs(d_ref - d_free).max()
            err["%s%d_stress" % (name, b)] = float(np.abs(d_eng - d_ref).max() / stress)
            err["%s%d_visible" % (name, b)] = float(stress / np.abs(d_ref).max())
    print(label, _fmt(err))
    _assert_grid(err, tol, guard)
    _assert_grid({k[6:]: v for k, v in err.items() if k.startswith("rigid_")}, tol, guard)
    for k, v in err.items():
        if k.endswith("_stress") and k[:2] in ("dv", "dw"):
            assert v <= tol_body, (k, err)
            assert err[k.replace("_stress", "_visible")] >= 1e-4, (k, err)
    return err, S, R


def _row_guards(scene, prev, S, R):
    """Rows the last k_g2p_rigid wrote (particles of rigid tiles before the substep) that the next P2G reads from rigid tiles:
    (rows that stayed in their tile, arrival rows: particles that changed tile)."""
    t0 = _tile(scene, prev["x"][np.searchsorted(prev["id"], S["id"])])
    t1 = _tile(scene, S["x"])
    moved = (t0 != t1).any(1)
    in_now = _in_rigid_tile(_pages(scene, R), t1)
    return int((in_now & ~moved).sum()), int((in_now & moved).sum())


@pytest.mark.parametrize("mode", ["host", "graph"])
@pytest.mark.parametrize("name,kind", KINDS)
def test_next_coupled_p2g_after_substeps(name, kind, mode):
    # substep(1), then (2), then (7) calls between the checks (each check runs one substep itself).  host: no graphs, the host
    # sets the bodies before every substep (translation at the read-back velocity); graph: device advection with a script
    # table, pairs of substeps replayed as CUDA graphs.  Slow particles: the stress is a larger part of the momentum.
    scene, st, rigid = _kind_scene(kind, "dynamic", vel=0.05, j_floor=False)
    if kind == scenes.MAT_WATER:
        # the pushing force drives water next to the plate to ~1 m/s within a few substeps, and its stress (pressure only)
        # then falls below GUARD of the momentum: without it the check still sees the stress
        rigid["pushing_force"] = 0.0
    n = len(st["x"])
    dt = float(np.float32(scene["dt"]))
    if mode == "graph":
        e = _engine(scene, st, rigid)
        bodies = _host_bodies(rigid)
        e.set_rigid_motion(_motion(bodies))
        table, _ = _scripted_pose_table(bodies, 13, dt)
        e.set_rigid_script(table)
    else:
        e = T.make_engine(scene, st, no_graph=True)
        e.set_rigid(rigid)
    stay = arr = 0
    for nsub in (1, 2, 7):
        if mode == "graph":
            e.substep(nsub)
        else:
            for _ in range(nsub):
                prev = e.download()
                r = _rigid_now(rigid, e.get_rigid_state(len(rigid["inv_mass"])))
                r["position"] = r["position"] + r["velocity"] * np.float32(dt)
                e.set_rigid_state(r)
                e.substep(1)
        _, S, R = next_p2g_coupled(e, scene, rigid, n, "%s %s nsub=%d" % (name, mode, nsub))
        if mode == "host":      # the state before the last substep is known here
            s, a = _row_guards(scene, prev, S, R)
            stay, arr = stay + s, arr + a
    e.close()
    if mode == "host":
        print("  rows of k_g2p_rigid read by k_p2g_rigid: %d stayed, %d arrived" % (stay, arr))
        # no arrivals here: at 0.05 m/s a particle moves 2e-4 cells per substep, and the jittered lattice keeps every particle
        # 0.05 cells or more from a tile face; the rotating block below guards the arrival rows
        assert stay > 40, (stay, arr)


# the rotating block: next-P2G stress error of the grid inside rigid tiles, where k_p2g_rigid recovers dt * force as the small
# difference A - 4 m apic_b.  Measured worst 4.9e-4 (grid) and 1.0e-4 (body), on an H100 and on the emulator.
TOL_ROT = 2e-3
TOL_ROT_BODY = 5e-4


def test_next_coupled_p2g_of_a_fast_rotating_block():
    # |4 m apic_b| >= 100 x the stress term of A inside the rigid tiles: the recovery (A - 4 m apic_b) * (-dx / 4) cancels, and
    # the error of the bodies' stress impulses and of the grid is measured there.  Fast enough that rows change tile: arrival
    # rows in rigid tiles, next to rows k_g2p_rigid wrote that stayed.
    from oracle import pyoracle as O
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY, "dynamic")
    rng = np.random.default_rng(7)
    c = st["x"].mean(0)
    W = np.array([[0.0, -70.0, 25.0], [70.0, 0.0, -40.0], [-25.0, 40.0, 0.0]])       # angular velocity (40, 25, 70) rad/s
    st["v"] = ((st["x"] - c) @ W.T).astype(np.float32)
    st["F"] = (np.eye(3).reshape(9) + rng.normal(size=(len(st["x"]), 9)) * 1e-4).astype(np.float32)
    # a drift of 18 m/s along the plate, and positions off the lattice (which keeps particles 0.05 cells from tile faces):
    # about 25 rows arrive in rigid tiles per substep, each with a large apic_b, next to the plate
    st["x"] = (st["x"] + rng.uniform(-0.5, 0.5, st["x"].shape) * scene["dx"]).astype(np.float32)
    st["v"] = (st["v"] + np.array([15.0, 0.0, 10.0], np.float32)).astype(np.float32)
    n = len(st["x"])
    dt = float(np.float32(scene["dt"]))
    e = T.make_engine(scene, st, no_graph=True)
    e.set_rigid(rigid)
    stay = arr = 0
    ratios = []
    for nsub in (1, 1, 1, 1, 1):
        for _ in range(nsub):
            prev = e.download()
            e.substep(1)
        S = e.download()
        R = _rigid_now(rigid, e.get_rigid_state(len(rigid["inv_mass"])))
        near = e.get_particle_cdf(n)["near"][S["id"].astype(np.int64)] != 0      # apic_b is zero next to a boundary
        sel = _in_rigid_tile(_pages(scene, R), _tile(scene, S["x"])) & ~near
        Fm = _math(S["F"][sel])
        stress = np.stack([O.calculate_force(scenes.MAT_JELLY, scene["mat_params"][0], Fm[i], float(S["ps"][sel][i]), float(S["vol"][sel][i]))
                           for i in range(len(Fm))]) * (-4.0 / float(np.float32(scene["dx"])) * scene["dt"])
        apic = 4.0 * S["mass"][sel].astype(np.float64)[:, None, None] * _math(S["b"][sel])
        ratio = float(np.median(np.abs(apic).max((1, 2)) / np.abs(stress).max((1, 2))))
        err, _, _ = next_p2g_coupled(e, scene, rigid, n, "rotating block nsub=%d (|4 m apic_b| / |stress| median %.0f)" % (nsub, ratio),
                                     tol=TOL_ROT, tol_body=TOL_ROT_BODY)
        ratios.append(ratio)
        s, a = _row_guards(scene, prev, S, R)
        stay, arr = stay + s, arr + a
    e.close()
    print("  rows of k_g2p_rigid read by k_p2g_rigid: %d stayed, %d arrived" % (stay, arr))
    assert ratios[0] >= 100, ratios          # the stress grows as the plate stops the block: the first check is the one that cancels
    assert stay > 500 and arr > 50, (stay, arr)


# ---------------------------------------------------------------------------------------------------- c. transfer edges
def _plate(c, off, friction=0.2, free=True, half=0.1, euler=(3.0, 8.0, 2.0)):
    b = dict(tris=scenes.plate_mesh(half, half, axis=1), position=np.asarray(c) + np.asarray(off), rotation=scenes.euler_rotation(euler),
             velocity=(0.1, -0.6, 0.05), angular_velocity=(0.2, 0.0, -0.3), friction=friction)
    if free:
        b.update(inv_mass=1 / 3.0, inv_inertia=np.diag([40.0, 25.0, 40.0]))
    return b


def _incompatible(scene, st, rigid, ref, cdf):
    """[n, 27] body ids (0: none) of the stencil nodes whose colour differs from the particle's in the transfers (the nodes
    that give a body an impulse instead of taking the particle's momentum), for the particles of rigid tiles."""
    X = np.asarray(st["x"], np.float64) / scene["dx"]
    base = np.floor(X - 0.5).astype(int)
    off = np.stack(np.meshgrid(*[np.arange(3)] * 3, indexing="ij"), -1).reshape(27, 3)
    nodes = base[:, None, :] + off[None]
    words = cdf["node_state"][nodes[..., 0], nodes[..., 1], nodes[..., 2]].astype(np.int64)
    gs, pst = words & 0xFFFFFF, ref["states"].astype(np.int64)[:, None]
    mask = (gs & pst & 0xAAAAAAAA) >> 1
    rid = np.where((gs & mask) != (pst & mask), (words >> 24) - 1, 0)      # the word holds body + 1
    rid[rid < 0] = 0
    rid[~_in_rigid_tile(_pages(scene, rigid), _tile(scene, st["x"]))] = 0
    return rid


def test_two_free_bodies_in_one_stencil():
    # two free plates 0.6 cells apart: rows whose stencil holds incompatible nodes of both, so that ImpulseAcc switches body
    # in the middle of a row, in k_p2g_rigid and (penalty window) k_g2p_rigid
    scene, st, _ = _kind_scene(scenes.MAT_JELLY)
    c = st["x"].mean(0)
    rigid = scenes.make_rigid([_plate(c, (0.0, 0.0, 0.0), 0.3), _plate(c, (0.0, 0.6 * scene["dx"], 0.0), 0.1)], scene["dx"], penalty=1e3)
    ref, _, cdf = coupled_substep(scene, st, rigid, "two free plates")
    rid = _incompatible(scene, st, rigid, ref, cdf)
    both = ((rid == 1).any(1) & (rid == 2).any(1)).sum()
    print("  rows with incompatible nodes of both bodies:", int(both))
    assert both > 50, both


def test_eleven_bodies():
    # ten scripted plates and an eleventh, free, through the block: its tag bits are 22-23, the last the 24-bit tag word holds
    scene, st, _ = _kind_scene(scenes.MAT_JELLY)
    c = st["x"].mean(0)
    bodies = [_plate(c, (x, 0.06, z), 0.2, free=False, half=0.02) for x in (-0.07, 0.07) for z in (-0.08, -0.04, 0.0, 0.04, 0.08)]
    bodies.append(_plate(c, (0.003, -0.01, 0.002), 0.3, half=0.06, euler=(11.0, 4.0, -7.0)))
    rigid = scenes.make_rigid(bodies, scene["dx"], penalty=1e3)
    assert len(rigid["inv_mass"]) == 12
    ref, _, cdf = coupled_substep(scene, st, rigid, "eleven bodies")
    rid = _incompatible(scene, st, rigid, ref, cdf)
    coloured = ((ref["states"] >> 22) & 3 != 0).sum()
    print("  particles coloured by body 11: %d, rows with its incompatible nodes: %d, bodies seen: %s" %
          (coloured, (rid == 11).any(1).sum(), np.unique(cdf["node_state"] >> 24)))
    assert coloured > 50 and (rid == 11).any(1).sum() > 50 and len(np.unique(cdf["node_state"] >> 24)) == 12


@pytest.mark.parametrize("frictions", [(-1.0, 0.4), (-2.5, 0.0), (0.0, -1.0), (0.4, -3.0)], ids=["sticky|0.4", "slip|0", "0|sticky", "0.4|slip"])
def test_friction_modes_on_both_sides_of_a_body(frictions):
    # friction_project's modes: -1 sticky, <= -2 slip with friction -f - 2, 0, > 0; a different one on each side of the plate,
    # chosen by the particle's side bit (B.fric[(pst >> 2 rid) & 1])
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY)
    rigid["frictions"] = rigid["frictions"].copy()
    rigid["frictions"][1] = frictions
    ref, _, cdf = coupled_substep(scene, st, rigid, "frictions %s" % (frictions,))
    rid = _incompatible(scene, st, rigid, ref, cdf)
    touch = (rid == 1).any(1)
    side = (ref["states"] >> 2) & 1
    counts = (int((touch & (side == 0)).sum()), int((touch & (side == 1)).sum()))
    print("  rows projected against the plate, side 0 / side 1:", counts)
    assert min(counts) > 50, counts


@pytest.mark.parametrize("pushing_force", [0.0, 20000.0])
def test_penalty_window(pushing_force):
    # the position correction of near particles with -0.3 dx < boundary distance < -0.05 dx (src/transfer.cpp:823-832), and its
    # impulse on a light, fast body, taken at the particle's new position; the resample's change of the body is compared alone
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY, vel=1.0)
    st["states"] = np.full(len(st["x"]), 0b1000, np.uint32)    # every particle brings the colour "positive side of body 1":
    rigid["pushing_force"] = pushing_force                    # those below the plate have a negative boundary distance
    rigid["inv_mass"] = rigid["inv_mass"] * 10
    rigid["inv_inertia"] = rigid["inv_inertia"] * 10
    # (body: the impulse is dv m with dv = bdist n penalty, and bdist carries the fp32 error of the reconstruction; measured
    # 5.1e-5 relative to the resample's change of the body)
    ref, _, _ = coupled_substep(scene, st, rigid, "penalty window, pushing force %g" % pushing_force, dict(body=2.5e-4))
    dx = scene["dx"]
    hit = (ref["near"] == 1) & (ref["bdist"] < -0.05 * dx) & (ref["bdist"] > -0.3 * dx)
    print("  particles in the penalty window:", int(hit.sum()))
    assert hit.sum() > 50, hit.sum()


def test_row_strides_of_k_p2g_rigid():
    # k_p2g_rigid walks a tile's rows with stride 61, or 67 when the count is a multiple of 61, or 1 when it is a multiple of
    # both (4087): rigid tiles with 122 (67), 134 (61), 4087 (1) and 200 rows (more than the 128-thread CTA)
    scene, _, rigid = _kind_scene(scenes.MAT_JELLY)
    page = _pages(scene, rigid)
    rng = np.random.default_rng(23)
    dx = scene["dx"]
    c = np.floor(rigid["position"][1] / dx - 0.5).astype(int) >> 2     # the tile of the plate's centre and three neighbours
    tiles = [c, c + (1, 0, 0), c + (0, 0, 1), c + (1, 0, 1)]
    counts = [122, 134, 4087, 200]
    assert _in_rigid_tile(page, np.array(tiles)).all()
    X = np.concatenate([4 * np.asarray(t) + 0.5 + rng.uniform(0.0, 4.0, (k, 3)) for t, k in zip(tiles, counts)])
    n = len(X)
    x = (X * dx).astype(np.float32)
    vol = np.full(n, dx ** 3 / 8, np.float32)
    st = scenes.make_state(x, (vol * 400).astype(np.float32), vol, scenes.MAT_JELLY)
    T.perturb_state(st, scenes.MAT_JELLY, dx, 29, 0.01, 0.3)
    got = np.unique(_tile(scene, st["x"]), axis=0, return_counts=True)
    assert sorted(got[1].tolist()) == sorted(counts), got
    for k in counts:
        stride = 61 if k % 61 else (67 if k % 67 else 1)
        assert len(np.unique(np.arange(k) * stride % k)) == k
    coupled_substep(scene, st, rigid, "row strides")


# ---------------------------------------------------------------------------------------------------- d. coupled runs
def _chain_errors(got, pc, cur, label):
    """The engine's survivors by id against the chained oracle's, without the particles whose colour flipped (a colour decided
    by two nearly equal weighted distances may flip in fp32, gather_cdf 200-205)."""
    ids = got["id"].astype(np.int64)
    assert np.array_equal(ids, np.nonzero(cur["alive"])[0])
    flip = pc["states"][ids] != cur["states"][ids]
    keep = ~flip
    err = dict(flips=float(flip.mean()), x=float(np.abs(got["x"][keep] - cur["x"][ids][keep]).max()), v=_rel(got["v"][keep], cur["v"][ids][keep]),
               b=_rel(got["b"][keep], cur["b"][ids][keep], 1e-30), F=float(np.abs(got["F"][keep] - cur["F"][ids][keep]).max()),
               ps=T.ps_err(got["ps"][keep], cur["ps"][ids][keep]))
    print(label, _fmt(err))
    assert err["flips"] <= MAX_FLIPS, err
    for k in ("x", "v", "b", "F", "ps"):
        assert err[k] <= TOL_CHAIN[k], (k, err)
    return err


# 20 (10) coupled substeps against the chained fp64 oracle, the measures of TOL_ONE; the body's velocities relative to the
# oracle's, its position absolute.  About 5 x the worst measured on an H100 and on the emulator (DESIGN §2).
TOL_CHAIN = dict(x=1.2e-6, v=5e-6, b=6e-5, F=7e-6, ps=3e-5)
TOL_CHAIN_BODY = 3e-6
MAX_FLIPS = 0.005


@pytest.mark.parametrize("mode", ["host", "graph"])
def test_scripted_plate_twenty_substeps_against_the_chained_oracle(mode):
    # a scripted plate sweeping through a strained jelly block.  graph: device advection with the script table, pairs replayed
    # as CUDA graphs; host: the per-substep contract (set_rigid_state with the same pose, substep(1)).  The oracle chains
    # substep_coupled with the pose of each substep: the script table's entries, in fp32 as the engine holds them.
    from oracle import pyoracle as O
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY, "kinematic")
    rigid["velocity"] = rigid["velocity"].copy()
    rigid["velocity"][1] = (2.0, -0.5, 1.0)
    n, nsub = len(st["x"]), 20
    dt = float(np.float32(scene["dt"]))
    bodies = _host_bodies(rigid)
    table, _ = _scripted_pose_table(bodies, nsub, dt)

    def pose(k):
        r = dict(rigid)
        if k:
            for key, sl in (("position", slice(0, 3)), ("rot", slice(3, 12)), ("velocity", slice(12, 15)), ("angular_velocity", slice(15, 18))):
                r[key] = rigid[key].copy()
                r[key][1:] = table[k - 1, 1:, sl].astype(np.float32)
        return r
    if mode == "graph":
        e = _engine(scene, st, rigid)
        e.set_rigid_motion(_motion(bodies))
        e.set_rigid_script(table)
        e.substep(nsub)
    else:
        e = T.make_engine(scene, st, no_graph=True)
        e.set_rigid(rigid)
        for k in range(nsub):
            e.set_rigid_state(pose(k))
            e.substep(1)
    got, pc = e.download(), e.get_particle_cdf(n)
    e.close()
    cur = dict(st, states=np.zeros(n, np.uint32))
    for k in range(nsub):
        cur, _, _, _, _ = O.substep_coupled(scene, cur, pose(k), np.float64)
    assert (cur["states"] != 0).sum() > 500 and abs(table[-1, 1, 0] - rigid["position"][1][0]) > 0.1 * scene["dx"]
    _chain_errors(got, pc, cur, "scripted plate, 20 substeps, %s" % mode)


def test_free_plate_ten_substeps_against_the_chained_oracle():
    # a free plate: the engine advances it on the device (graph replay), the oracle chains substep_coupled with
    # HostRigidBody.advect (fp64) on its own body velocities; particles and the body's trajectory are compared every substep
    from oracle import pyoracle as O
    from tests.test_gpu_rigid_motion import _host_advect
    scene, st, rigid = _kind_scene(scenes.MAT_JELLY, "dynamic")
    n, nsub = len(st["x"]), 10
    dt = float(np.float32(scene["dt"]))
    bodies = _host_bodies(rigid)
    e = _engine(scene, st, rigid)
    e.set_rigid_motion(_motion(bodies))
    b = _host_bodies(rigid)[0]
    cur, r, t = dict(st, states=np.zeros(n, np.uint32)), rigid, 0.0
    worst = dict(position=0.0, velocity=0.0, angular_velocity=0.0)
    for k in range(nsub):
        e.substep(1)
        cur, _, _, rv, _ = O.substep_coupled(scene, cur, r, np.float64)
        b.velocity, b.angular_velocity = rv["velocity"][1].copy(), rv["angular_velocity"][1].copy()
        _host_advect(b, t, dt)
        t += dt
        r = dict(rigid, position=rigid["position"].copy(), rot=rigid["rot"].copy(), velocity=rigid["velocity"].copy(),
                 angular_velocity=rigid["angular_velocity"].copy(), inv_inertia=rigid["inv_inertia"].copy())
        r["position"][1], r["velocity"][1], r["angular_velocity"][1] = b.position, b.velocity, b.angular_velocity
        r["rot"][1] = b.rotation.T.reshape(9)
        r["inv_inertia"][1] = (b.rotation @ b.inv_inertia_body @ b.rotation.T).T.reshape(9)
        rs = e.get_rigid_state(len(rigid["inv_mass"]))
        for key in worst:
            worst[key] = max(worst[key], _rel(rs[key][1], getattr(b, key)) if key != "position" else float(np.abs(rs[key][1] - b.position).max()))
    got, pc = e.download(), e.get_particle_cdf(n)
    e.close()
    print("free plate, body trajectory over 10 substeps", _fmt(worst))
    _chain_errors(got, pc, cur, "free plate, 10 substeps")
    assert np.abs(b.velocity - rigid["velocity"][1]).max() > 1e-2          # the coupling and gravity moved the body
    assert worst["position"] <= 1.2e-7 and worst["velocity"] <= TOL_CHAIN_BODY and worst["angular_velocity"] <= TOL_CHAIN_BODY, worst
