"""Host logic of the mirror's 2-D path (MPM(res=(r0, r1)) -> capi.Engine2D) with the device engine replaced by an in-memory
stand-in — no GPU: the 2-D lattice and the band rejection of add_particles, particles added between steps keeping their ids,
the level set's 2-vectors, frame dumps with zero third components, snapshots, and the MPM<3>-only verbs refused with
ValueError.  The 3-D mirror is left as it was (its refusals of the dampings included)."""
import numpy as np
import pytest

from taichi_mpm_b200 import async_mpm, bgeo, capi, mpm as mpm_mod, scenes, slab


class FakeEngine2D:
    """Stores what is uploaded; substep() advects x by v*dt*n; ids are upload positions, as the engine numbers them."""

    def __init__(self, res, dx, dt, gravity, particle_gravity, clean_boundary, device=0, capacity=0, apic_damping=0.0, rpic_damping=0.0):
        self.res, self.dt, self.gravity = tuple(res), dt, tuple(gravity)
        self.dampings = (apic_damping, rpic_damping)
        self.cfg = type("Cfg", (), {"dim": 2})()
        self.mats, self.p, self.updates = {}, None, 0
        self.levelset = None

    def set_material(self, g, kind, params):
        self.mats[g] = (kind, np.array(params, np.float32))

    def set_sdf(self, sdf, friction):
        self.levelset = ("sdf", sdf, friction)

    def set_planes(self, planes, friction):
        self.levelset = ("planes", np.asarray(planes), friction)

    def set_levelset_shapes(self, shapes, friction):
        self.levelset = ("shapes", shapes, friction)

    def set_id_base(self, base):
        assert base == 0

    def upload(self, x, v, mass, vol, F, b, ps, group):
        n = len(x)
        assert np.shape(x) == (n, 2) and np.shape(v) == (n, 2) and np.shape(F) == (n, 4) and np.shape(b) == (n, 4)
        self.p = dict(id=np.arange(n, dtype=np.uint32), x=np.array(x, np.float32), v=np.array(v, np.float32), F=np.array(F, np.float32),
                      b=np.array(b, np.float32), mass=np.array(mass, np.float32), vol=np.array(vol, np.float32), ps=np.array(ps, np.float32),
                      group=np.array(group, np.int32))

    def num_particles(self):
        return 0 if self.p is None else len(self.p["x"])

    def download(self):
        return {k: a.copy() for k, a in self.p.items()}

    def substep(self, n):
        self.p["x"] = (self.p["x"] + self.p["v"] * np.float32(self.dt * n)).astype(np.float32)
        self.updates += n * len(self.p["x"])

    def update_count(self):
        return self.updates

    def drop(self, engine_ids):
        keep = ~np.isin(self.p["id"], engine_ids)
        self.p = {k: a[keep] for k, a in self.p.items()}

    def download_bgeo_points(self, id_range):
        p = self.p
        n = len(p["x"])
        w = np.zeros((n, 12), ">u4")
        f = w.view(">f4")
        f[:, 0:2] = p["x"]
        f[:, 3] = 1.0
        w[:, 5] = p["id"]
        w[:, 6:9] = 1
        f[:, 9:11] = p["v"]
        return n, w.view(np.uint8).reshape(-1)


@pytest.fixture
def fake2d(monkeypatch):
    monkeypatch.setattr(capi, "Engine2D", FakeEngine2D)


def test_2d_solver_seeds_a_4_per_cell_lattice(fake2d):
    m = mpm_mod.MPM2D(res=(64, 48), base_delta_t=1e-4)
    assert m.dim == 2 and m.gravity == (0.0, -10.0) and m.engine.gravity == (0.0, -10.0)
    m.add_particles(type="sand", benchmark_block=((4, 10), (20, 20)), density=400)
    p = m.get_particles()
    dx = 1.0 / 64
    # cells whose particles lie within 7 cells of a face are rejected (src/mpm.cpp:129-132): x cells 4..6 go
    assert len(p["x"]) == 4 * (20 - 7) * 10
    assert p["x"].shape[1] == 2 and (p["x"].min(0) * 64 >= 7).all()
    assert np.allclose(p["vol"], dx * dx / 4) and np.allclose(p["mass"], dx * dx / 4 * 400)
    X = p["x"] * 64 - 0.5
    assert np.allclose(np.abs(X - np.round(X)), 0.25)       # cell centre +- 0.25 dx
    kind, params = m.engine.mats[0]
    assert kind == scenes.MAT_SAND and np.array_equal(params, scenes.material_params(scenes.MAT_SAND))


def test_positions_take_2_vectors_and_ids_survive_adds(fake2d):
    m = mpm_mod.MPM2D(res=(32, 32), base_delta_t=1e-4, gravity=(1.0, -5.0))
    m.add_particles(type="jelly", positions=np.array([[0.3, 0.3], [0.4, 0.4], [0.5, 0.5], [0.01, 0.5]]), initial_velocity=(1.0, 0.0))
    assert np.array_equal(m.get_particles()["id"], [0, 1, 2])         # the band particle is rejected, its id not handed out
    m.step(0.001)
    m.engine.drop([1])                                                # the engine deleted id 1
    m.add_particles(type="water", positions=np.array([[0.6, 0.6]]))
    p = m.get_particles()
    assert np.array_equal(p["id"], [0, 2, 3])
    assert np.array_equal(p["group"], [0, 0, 1])
    assert np.allclose(p["x"][0], [0.3 + m.substep_counter * 1e-4, 0.3], atol=1e-6)   # the state came back with the ids
    assert p["vol"][2] == np.float32((1 / 32) ** 2 / 4)


def test_level_set_takes_2_vectors(fake2d):
    m = mpm_mod.MPM2D(res=(32, 32))
    ls = m.create_levelset()
    ls.add_plane((0, 2), -0.25)
    ls.add_sphere((0.5, 0.3), 0.1)
    ls.add_cuboid((0.1, 0.1), (0.2, 0.4), inside_out=True)
    ls.set_friction(0.4)
    m.set_levelset(ls)
    kind, shapes, fr = m.engine.levelset
    assert kind == "shapes" and fr == 0.4
    assert shapes[0] == (capi.SHAPE_PLANE, False, [0.0, 1.0, 0.0, -8.0])
    assert shapes[1][2] == pytest.approx([16.0, 9.6, 0.0, 3.2])
    assert shapes[2][2] == pytest.approx([3.2, 3.2, 0.0, 6.4, 12.8, 0.0]) and shapes[2][1]
    phi = ls.node_phi()
    # at node (16, 4): the plane gives -4, the circle +2.4 and the rectangle container -(16 - 6.4)
    assert phi.shape == (33, 33) and phi[16, 4] == pytest.approx(-9.6, abs=1e-5)
    with pytest.raises(ValueError):
        ls.add_plane((0, 1, 0), 0.0)


def test_frames_have_zero_third_components_and_keep_ids(fake2d, tmp_path):
    m = mpm_mod.MPM2D(res=(32, 32), base_delta_t=1e-4, frame_directory=str(tmp_path))
    m.add_particles(type="snow", positions=np.array([[0.3, 0.4], [0.5, 0.5], [0.6, 0.3]]), initial_velocity=(0.5, -0.5))
    m.step(0.001)
    m.engine.drop([0])
    m.add_particles(type="snow", positions=np.array([[0.4, 0.6]]))
    fn = m.visualize()
    pos, attrs = bgeo.read_bgeo(fn)
    a = {name: arr.reshape(len(pos), -1) for name, _, arr in attrs}
    p = m.get_particles()
    assert np.array_equal(a["index"][:, 0], [1, 2, 3]) and np.array_equal(a["index"][:, 0], p["id"])
    assert np.array_equal(pos[:, :2], p["x"]) and (pos[:, 2] == 0).all()
    assert np.array_equal(a["v"][:, :2], p["v"]) and (a["v"][:, 2] == 0).all()
    m.verbose_bgeo = True
    pos2, attrs2 = bgeo.read_bgeo(m.visualize())
    a2 = {name: arr.reshape(len(pos2), -1) for name, _, arr in attrs2}
    assert np.array_equal(pos2, pos) and np.array_equal(a2["index"], a["index"]) and (a2["boundary_normal"] == 0).all()


def test_snapshot_round_trip_keeps_ids(fake2d, tmp_path):
    m = mpm_mod.MPM2D(res=(32, 32), base_delta_t=1e-4)
    m.add_particles(type="sand", benchmark_block=((8, 8), (12, 12)))
    m.step(0.002)
    m.engine.drop([0, 5])
    m.save(str(tmp_path / "s.npz"))
    m2 = mpm_mod.MPM2D(res=(32, 32), base_delta_t=1e-4)
    m2.load(str(tmp_path / "s.npz"))
    a, b = m.get_particles(), m2.get_particles()
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    assert m2.current_t == m.current_t
    m2.add_particles(type="sand", positions=np.array([[0.5, 0.5]]))
    assert m2.get_particles()["id"][-1] == 64


def test_mpm3_only_verbs_raise_value_error(fake2d):
    m = mpm_mod.MPM2D(res=(32, 32))
    with pytest.raises(ValueError):
        m.add_particles(type="rigid", codimensional=False, tris=np.zeros((1, 3, 3)), initial_position=(0.5, 0.5, 0.5))
    with pytest.raises(ValueError):
        m.set_levelset(m.create_levelset(), is_dynamic_levelset=True)
    with pytest.raises(ValueError):
        m.delete_particles_inside_level_set()
    with pytest.raises(ValueError):
        mpm_mod.MPM2D(res=(32, 32), affine_damping=0.1)
    with pytest.raises(ValueError):
        async_mpm.AsyncMPM(res=(32, 32))
    with pytest.raises(ValueError):
        slab.EngineAdapter(m.engine)
    with pytest.raises(ValueError):
        slab.append_particles(m.engine, {}, 0)
    with pytest.raises(ValueError):
        mpm_mod.MPM2D(res=(32, 32), gravity=(0.0, -10.0, 0.0))
    m = mpm_mod.MPM2D(res=(32, 32), apic_damping=0.25, rpic_damping=0.5)
    assert m.engine.dampings == (0.25, 0.5)


def test_2d_scenes_take_mpm2d_and_mpm_stays_3d(monkeypatch):
    """MPM keeps refusing a 2-D res (tests/test_mirror_host.py); MPM2D builds the 2-D engine and refuses a 3-D res."""
    made = []

    class Fake3D:
        def __init__(self, *a, **kw):
            made.append((a, kw))

    monkeypatch.setattr(capi, "Engine", Fake3D)
    monkeypatch.setattr(capi, "Engine2D", FakeEngine2D)
    with pytest.raises(ValueError, match="MPM2D"):
        mpm_mod.MPM(res=(64, 64))
    with pytest.raises(ValueError):
        mpm_mod.MPM2D(res=(32, 32, 32))
    m = mpm_mod.MPM(res=(32, 32, 32))
    assert m.dim == 3 and made[-1][0][0] == (32, 32, 32) and m.gravity == (0.0, -10.0, 0.0)
    m2 = mpm_mod.MPM2D(res=(64, 64), gravity=-5)
    assert m2.dim == 2 and isinstance(m2.engine, FakeEngine2D) and m2.gravity == (0.0, -5.0) and len(made) == 1
    for kw in (dict(optimized=False), dict(affine_damping=0.1)):
        with pytest.raises(ValueError):
            mpm_mod.MPM2D(res=(64, 64), **kw)
