"""Routing of MPM.add_particles / delete_particles_inside_level_set between the device edits (capi.Engine.append /
delete_inside_levelset) and the host concatenate-and-upload path, with the engine replaced by an in-memory stand-in."""
import numpy as np
import pytest

from taichi_mpm_b200 import async_mpm, capi, mpm as mpm_mod
from tests.test_mirror_host import FakeEngine


class EditingFakeEngine(FakeEngine):
    """FakeEngine with the two device edits: ids continue after every id handed out, survivors keep theirs."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = []
        self.span = 0

    def upload(self, x, *a):
        super().upload(x, *a)
        self.calls.append("upload")
        self.span = len(x)

    def append(self, x, v, mass, vol, F=None, b=None, scalar=None, group=None):
        self.calls.append("append")
        n = len(x)
        first = self.id_base + self.span
        new = dict(id=(first + np.arange(n)).astype(np.uint32), x=np.array(x, np.float32), v=np.array(v, np.float32),
                   F=np.array(F, np.float32).reshape(n, 9), b=np.array(b, np.float32).reshape(n, 9), mass=np.array(mass, np.float32),
                   vol=np.array(vol, np.float32), ps=np.array(scalar, np.float32), group=np.array(group, np.int32))
        self.p = new if self.p is None else {k: np.concatenate([self.p[k], new[k]]) for k in new}
        self.span += n
        return first

    def delete_inside_levelset(self):
        self.calls.append("delete")
        keep = self.p["x"][:, 1] >= 0.36          # the plane of the test below
        self.p = {k: a[keep] for k, a in self.p.items()}
        return int((~keep).sum())


@pytest.fixture
def editing_engine(monkeypatch):
    monkeypatch.setattr(capi, "Engine", EditingFakeEngine)


def _positions(n, y=0.5):
    return np.stack([np.linspace(0.4, 0.6, n), np.full(n, y), np.full(n, 0.5)], 1).astype(np.float32)


def test_device_append_only_when_particles_are_resident(tmp_path, editing_engine):
    m = mpm_mod.MPM(res=(32, 32, 32), base_delta_t=1e-4, frame_directory=str(tmp_path / "f"))
    m.add_particles(type="sand", benchmark_block=((10, 10, 10), (13, 13, 13)))
    m.add_particles(type="water", positions=_positions(5))      # nothing resident yet: both sets wait on the host
    assert m.engine.calls == []
    m.step(1e-3)
    n0 = m.num_particles()
    assert m.engine.calls == ["upload"] and n0 == 8 * 27 + 5
    m.add_particles(type="water", positions=_positions(4))      # resident, no host copy: on the device
    assert m.engine.calls == ["upload", "append"] and m._host is None
    assert m._id_range() == n0 + 4
    p = m.get_particles()
    assert np.array_equal(p["id"], np.arange(n0 + 4))
    m._pull_host()                                              # a pending host copy: the new particles join it
    m.add_particles(type="water", positions=_positions(3))
    assert m.engine.calls == ["upload", "append"] and len(m._host["x"]) == n0 + 7
    m.step(1e-3)
    assert m.engine.calls[-1] == "upload" and m._id_range() == n0 + 7
    m.visualize()


def test_device_delete_only_with_a_level_set_and_resident_particles(editing_engine):
    m = mpm_mod.MPM(res=(32, 32, 32), base_delta_t=1e-4)
    ls = m.create_levelset()
    ls.add_plane((0, 1, 0), -0.36)
    m.set_levelset(ls, False)
    m.add_particles(type="sand", benchmark_block=((10, 10, 10), (13, 14, 13)))
    m.delete_particles_inside_level_set()                       # still on the host: filtered there, then uploaded
    assert "delete" not in m.engine.calls
    m.step(1e-3)
    m.add_particles(type="sand", positions=_positions(6, y=0.3))
    m.delete_particles_inside_level_set()
    assert m.engine.calls[-2:] == ["append", "delete"]
    p = m.get_particles()
    assert (p["x"][:, 1] >= 0.36).all()
    assert m._id_range() > p["id"].max()                        # the survivors' ids stay inside the range visualize packs


def test_async_mpm_never_appends_on_the_device(monkeypatch):
    # AsyncMPM's pools own the particles and advance() uploads them: the device edits must never be reached
    from tests.test_async_host import OracleEngine

    class NoEdits(OracleEngine):
        def append(self, *a, **k):
            raise AssertionError("AsyncMPM appended on the device")

        def delete_inside_levelset(self):
            raise AssertionError("AsyncMPM deleted on the device")

    monkeypatch.setattr(capi, "Engine", NoEdits)
    m = async_mpm.AsyncMPM(res=(32, 32, 32), base_delta_t=2.5e-5, unit_delta_t=2.5e-5, max_units=64, cfl_dt_mul=0.1)
    m.add_particles(type="snow", benchmark_block=((12, 12, 12), (14, 14, 14)))
    m.step(2.5e-4)
    m.add_particles(type="snow", positions=_positions(4))
    m.step(2.5e-4)
    assert m._n_uploaded == 0 and len(m.pool["id"]) == 64 + 4
    assert m.num_particles() == 64 + 4
