"""AsyncMPM (scripts/async/*.py) on the mirror + device engine: a snow block whose one half moves fast, so that its blocks take
a finer time level than the rest:

    python examples/async_snow.py [steps]

The scheduler (per-block power-of-two time levels, neighbour masks) is host code; the particle and backup pools live on the
device, and every advance it schedules (gather, pool edits and one substep with the level's step) runs there without moving a
particle record across the bus."""
import sys

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
from taichi_mpm_b200 import AsyncMPM  # noqa: E402


def main(steps=2):
    unit = 2.5e-5
    mpm = AsyncMPM(res=(32, 32, 32), base_delta_t=unit, unit_delta_t=unit, max_units=64, cfl_dt_mul=0.1)
    mpm.add_particles(type="snow", benchmark_block=((12, 12, 12), (16, 20, 20)), jitter=0.2)
    mpm.add_particles(type="snow", benchmark_block=((16, 12, 12), (20, 20, 20)), jitter=0.2, initial_velocity=(10.0, 0.0, 0.0))
    for s in range(steps):
        mpm.step(80 * unit)
        st = mpm.scheduler_stats()
        print("step %d: t = %d units, time levels %d..%d units, %d particle updates so far, %d particles" %
              (s + 1, st["current_t_int"], st["min_level"], st["max_level"], st["update_counter"], mpm.num_particles()))
    return mpm


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:2]))
