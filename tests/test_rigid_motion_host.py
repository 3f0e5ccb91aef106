"""What the mirror asks of the engine for rigid scenes (MPM._rigid_substeps) with the engine replaced by an in-memory stand-in:
bodies uploaded once, one read-back per step, the state pushed only after a user edit, the script table evaluated at the
float32 clock sequence of step(), read-back poses landing in the HostRigidBody objects."""
import numpy as np
import pytest

from taichi_mpm_b200 import capi, mpm as mpm_mod, scenes
from tests.test_mirror_host import FakeEngine


class RigidFakeEngine(FakeEngine):
    """FakeEngine that records the rigid calls; get_rigid_state moves every free body by +0.001 in x per substep run."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.calls = []
        self.table = None
        self.pose = None

    def set_rigid(self, rec):
        self.calls.append("set_rigid")
        self.pose = np.array(rec["position"], np.float32)
        self.rot = np.array(rec["rot"], np.float32)
        self.vel = np.array(rec["velocity"], np.float32)

    def set_rigid_motion(self, motion, levelset_collision=False):
        self.calls.append("set_rigid_motion")
        self.motion = motion

    def set_rigid_state(self, rec):
        self.calls.append("set_rigid_state")
        self.pose = np.array(rec["position"], np.float32)

    def set_rigid_script(self, poses):
        self.calls.append("set_rigid_script")
        self.table = np.array(poses)

    def substep(self, n):
        self.calls.append(("substep", n))
        super().substep(n)
        for b, m in enumerate(self.motion):
            if b and not m["scripted_position"]:
                self.pose[b, 0] += np.float32(0.001 * n)

    def get_rigid_state(self, nb):
        self.calls.append("get_rigid_state")
        return dict(position=self.pose.copy(), velocity=np.full((nb, 3), 0.5, np.float32), angular_velocity=np.full((nb, 3), 0.25, np.float32),
                    rotation=np.array([np.reshape(r, (3, 3)).T for r in self.rot], np.float32))


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(capi, "Engine", RigidFakeEngine)
    made = []
    orig = scenes.rigid_boundary_samples

    def counting(*a, **kw):
        made.append(1)
        return orig(*a, **kw)
    monkeypatch.setattr(scenes, "rigid_boundary_samples", counting)
    return made


def _scene(clock):
    m = mpm_mod.MPM(res=(32, 32, 32), base_delta_t=3e-4)
    m.add_particles(type="sand", benchmark_block=((10, 10, 10), (13, 13, 13)))
    m.add_particles(type="rigid", tris=scenes.plate_mesh(0.03, 0.1, axis=0), codimensional=True,
                    scripted_position=lambda t: (clock.append(t), (0.4 + t, 0.4, 0.5))[1], scripted_rotation=lambda t: (0.0, 0.0, 10.0))
    m.add_particles(type="rigid", tris=scenes.box_mesh((0.04, 0.03, 0.04)), codimensional=False, initial_position=(0.6, 0.5, 0.5))
    return m


def test_bodies_uploaded_once_one_read_back_per_step(fake):
    clock = []
    m = _scene(clock)
    for _ in range(4):
        m.step(0.002)
    calls = m.engine.calls
    assert calls.count("set_rigid") == 1 and calls.count("set_rigid_motion") == 1
    assert len(fake) == 2                                           # the samples of each body built once, not per substep
    assert calls.count("get_rigid_state") == 4 and calls.count("set_rigid_state") == 0
    assert [c for c in calls if isinstance(c, tuple)] == [("substep", 6), ("substep", 7), ("substep", 7), ("substep", 6)]
    assert m.substep_counter == 26


def test_state_pushed_only_after_a_user_edit(fake):
    m = _scene([])
    m.step(0.002)
    m.step(0.002)
    assert m.engine.calls.count("set_rigid_state") == 0
    m.rigids[1].velocity = np.array([0.0, 3.0, 0.0])               # the user throws the box
    m.step(0.002)
    assert m.engine.calls.count("set_rigid_state") == 1
    assert m.engine.calls.index("set_rigid_state") > len(m.engine.calls) - 6
    m.step(0.002)
    assert m.engine.calls.count("set_rigid_state") == 1


def test_script_table_at_the_float32_clock_sequence(fake):
    clock = []
    m = _scene(clock)
    del clock[:]
    m.step(0.002)
    h = np.float32(3e-4)
    t, want = np.float32(0.0), []
    while np.float32(t + h) < np.float32(0.002):
        want.append(float(t) + float(h))
        t = np.float32(t + h)
    assert clock == want and len(want) == 6
    table = m.engine.table
    assert table.shape == (6, 3, capi.RIGID_SCRIPT_STRIDE)
    assert np.allclose(table[:, 1, 0], 0.4 + np.array(want)) and not table[:, 2].any()   # the free box has no entries
    assert np.allclose(table[1:, 1, 12], (np.diff(0.4 + np.array(want))) / float(h))   # velocity = finite difference of positions
    assert m.current_t == t


def test_read_back_poses_land_in_the_host_bodies(fake):
    m = _scene([])
    x0 = m.rigids[1].position.copy()
    m.step(0.002)
    box, paddle = m.rigids[1], m.rigids[0]
    assert np.allclose(box.position, x0 + [0.006, 0, 0], atol=1e-6) and box.position.dtype == np.float64
    assert np.array_equal(box.velocity, [0.5, 0.5, 0.5]) and np.array_equal(box.angular_velocity, [0.25, 0.25, 0.25])
    # the scripted paddle keeps the table's fp64 pose
    assert np.array_equal(paddle.position, m.engine.table[-1, 1, 0:3])
