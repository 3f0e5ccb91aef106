"""Every device allocation of the engine has an owner: on the SIMT emulator build (tests/simt), which counts its live
allocations and can make any one of them fail, a scenario that reaches every allocating entry point leaves nothing behind
once its engines are closed — after a clean run, and after a run in which the k-th allocation fails, for every k.  A
failed allocation must surface as an MpmbError (MPMB_ERR_CUDA, or creation refused).

The scenario runs in a child process (`python -m tests.test_device_memory_simt`) against the emulator build, so that the
product library this process may have loaded stays out of it."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES, DX, DT = 32, 1.0 / 32, 1e-4


def _sand(lo, hi, seed):
    from taichi_mpm_b200 import scenes
    x, mass, vol = scenes.lattice_block(RES, lo, hi, jitter=0.2, seed=seed)
    st = scenes.make_state(x, mass, vol, scenes.MAT_SAND)
    st["v"][:, 2] = 0.5
    return st


def _fields(st, sl=slice(None)):
    return [np.ascontiguousarray(st[k][sl]) for k in ("x", "v", "mass", "vol", "F", "b", "ps", "group")]


class _HostBytes:
    """numpy bytes in place of a device buffer (emulator: device memory is host memory)"""

    def __init__(self, n):
        self.a = np.zeros(max(int(n), 16), np.uint8)

    def data_ptr(self):
        return self.a.ctypes.data

    def numel(self):
        return self.a.size

    def element_size(self):
        return 1


def _aos(st):
    """st in the reference's 320-byte AoS slots (the layout of test_gpu_parity.test_aos_round_trip)"""
    from taichi_mpm_b200 import capi
    n = len(st["x"])
    L = capi.MpmbAosLayout()
    L.stride, L.off_v_and_m, L.off_pos, L.off_dg_e, L.off_apic_b, L.col_pitch = 320, 16, 32, 48, 96, 16
    L.off_vol, L.off_scalar = 164, 200
    slots = n + 3
    pool = np.zeros((slots, 320), np.uint8)
    indices = np.random.default_rng(1).permutation(slots)[:n].astype(np.uint32)
    f = pool.view(np.float32).reshape(slots, 80)
    for k, s in enumerate(indices):
        f[s, 4:7] = st["v"][k]; f[s, 7] = st["mass"][k]; f[s, 8:11] = st["x"][k]
        for c in range(3):
            f[s, 12 + 4 * c: 15 + 4 * c] = st["F"][k, 3 * c: 3 * c + 3]
        f[s, 41] = st["vol"][k]
    return pool, indices, L


def _box(half, y):
    from taichi_mpm_b200 import rigid as rigid_mod, scenes
    b = rigid_mod.HostRigidBody(scenes.box_mesh(half), density=400.0, position=(0.5, y, 0.5), velocity=(0.0, -0.5, 0.0), frictions=(0.3, 0.3))
    return b, rigid_mod.engine_records([b], DX, 0.0, 20000.0)


def scenario(opened):
    """Reaches every allocating entry point of the C-ABI; every engine it creates is appended to `opened`."""
    from taichi_mpm_b200 import capi, scenes, slab
    sand = scenes.material_params(scenes.MAT_SAND)

    def engine(**kw):
        e = capi.Engine((RES,) * 3, DX, DT, **kw)
        opened.append(e)
        e.set_material(0, scenes.MAT_SAND, sand)
        return e

    # one GPU, no configured capacity: uploads, edits, level sets, downloads, rigid bodies
    st = _sand((12, 12, 12), (16, 15, 16), 1)
    e = engine()
    e.upload(*_fields(st))
    e.append(*_fields(st, slice(0, 8)))
    e.append(*_fields(st, slice(0, 60)))            # grows the rows again
    e.set_planes(np.array([[0.0, 1.0, 0.0, -13.0]], np.float32), 0.4)
    e.delete_inside_levelset()
    e.set_levelset_shapes([(capi.SHAPE_PLANE, 0, (0.0, 1.0, 0.0, -8.0))], 0.4)
    e.seed_lattice((12, 12, 12), (15, 14, 15), DX ** 3 / 8, 400 * DX ** 3 / 8)
    pool, indices, L = _aos(st)
    e.upload_aos(pool, indices, L, group=np.zeros(len(indices), np.int32))
    e.sort_particles_and_populate_grid()
    e.rasterize()
    e.download_grid(0)
    e.resample()
    e.download_aos(pool, indices.copy(), L)
    e.download()
    e.download_bgeo_points(2 * len(st["x"]))
    body, rec = _box((0.06, 0.06, 0.06), 0.6)
    e.set_rigid(rec)
    body, rec = _box((0.1, 0.05, 0.08), 0.6)         # another sample count
    e.set_rigid(rec)
    e.set_rigid_motion([{}, body.motion_record()], levelset_collision=True)
    e.set_rigid_script(np.zeros((1, 2, capi.RIGID_SCRIPT_STRIDE)))
    e.set_rigid_script(np.zeros((3, 2, capi.RIGID_SCRIPT_STRIDE)))   # grows the table ...
    e.set_rigid_script(np.zeros((7, 2, capi.RIGID_SCRIPT_STRIDE)))   # ... twice
    e.substep(1)

    # a configured capacity
    c = engine(capacity=512)
    c.upload(*_fields(st))

    # AsyncMPM pools
    a = engine()
    nb = (RES + 1 + 3) // 4 + 1, (RES + 1 + 3) // 4 + 1, (RES + 1 + 7) // 8 + 1
    a.async_init(nb, 1.0 / DX)
    a.async_init(nb, 1.0 / DX)
    rec = {k: st[k] for k in ("x", "v", "F", "b", "mass", "vol", "ps", "group")}
    rec["id"] = np.arange(len(st["x"]), dtype=np.uint32)
    a.async_add(0, rec)
    a.async_block_limits(True)
    a.async_advance(np.full(int(np.prod(nb)), capi.ASYNC_EQUAL, np.uint8), DT)

    # two z-slab ranks in one process, peers connected by pointer; the re-cut thickens rank 1's slab (its tile arrays grow)
    st = _sand((14, 12, 8), (17, 14, 24), 2)
    nl = slab.tile_layers(RES)
    cuts = [(0, nl // 2), (nl // 2, nl)]
    tz = slab.base_tile_z(st["x"][:, 2], DX)
    ranks = []
    for r, (z0, z1) in enumerate(cuts):
        s = engine(rank=r, world=2, tile_z0=z0, tile_z1=z1, migrate_capacity=64)
        s.set_id_base(int((tz < z0).sum()))
        s.upload(*_fields(st, (tz >= z0) & (tz < z1)))
        ranks.append(s)
    for k in (0, 1):
        ranks[0].xchg_connect(k, 1, ptr=ranks[1].xchg_buffer(k, 0))
        ranks[1].xchg_connect(k, 0, ptr=ranks[0].xchg_buffer(k, 1))
    new = [(0, 3), (3, nl)]
    flat = [0, 3, nl]
    packs = []
    for s in ranks:
        counts = s.recut_pack(flat)
        b = _HostBytes(int(counts.sum()) * capi.RECORD_BYTES)
        s.recut_pack(flat, b)
        packs.append((counts, b))
    for r, s in enumerate(ranks):
        data = [b.a[int(cn[:r].sum()) * capi.RECORD_BYTES:int(cn[:r + 1].sum()) * capi.RECORD_BYTES] for cn, b in packs]
        buf = _HostBytes(0)
        buf.a = np.ascontiguousarray(np.concatenate(data + [np.zeros(16, np.uint8)]))
        s.recut_apply(new[r][0], new[r][1], buf, sum(int(cn[r]) for cn, _ in packs))


def _close(opened):
    for e in opened:
        e.close()
    opened.clear()


def main():
    """Clean run, then one run per allocation k with the k-th one failing; prints the counts as JSON."""
    from taichi_mpm_b200 import capi
    L = capi.lib()
    L.simt_device_allocations.restype = C.c_longlong
    L.simt_fail_allocation.restype = C.c_longlong
    live = L.simt_device_allocations
    fail_at = lambda k: L.simt_fail_allocation(C.c_longlong(k))
    baseline = live()
    opened = []
    # a clean run counts its allocations: the failure armed past its end tells how far it got
    far = 1 << 40
    fail_at(far)
    scenario(opened)
    n_alloc = far - fail_at(0)
    held = live() - baseline
    _close(opened)
    out = dict(allocations=n_alloc, held=held, after_close=live() - baseline, failures=[])
    for k in range(1, n_alloc + 1):
        before = live()
        fail_at(k)
        err = None
        try:
            scenario(opened)
        except capi.MpmbError as ex:
            err = ex.code
        fired = fail_at(0) == 0
        _close(opened)
        out["failures"].append(dict(k=k, fired=fired, code=err, leaked=live() - before))
    print("RESULT " + json.dumps(out))


@pytest.fixture(scope="module")
def report():
    from tests.simt import build_simt
    env = dict(os.environ, MPMB_LIB=build_simt.build(), MPMB_SIMT="1")
    r = subprocess.run([sys.executable, "-m", "tests.test_device_memory_simt"], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    assert r.returncode == 0 and lines, r.stdout[-4000:]
    return json.loads(lines[-1][len("RESULT "):])


def test_closing_the_engines_frees_every_device_allocation(report):
    assert report["allocations"] > 0 and report["held"] > 0
    assert report["after_close"] == 0


def test_every_failed_allocation_raises_and_leaks_nothing(report):
    bad = [f for f in report["failures"] if not f["fired"] or f["code"] is None or f["leaked"] != 0]
    assert len(report["failures"]) == report["allocations"]
    assert not bad, bad


if __name__ == "__main__":
    main()
