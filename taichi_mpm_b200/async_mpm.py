"""AsyncMPM on the device engine: the reference's block scheduler (src/async/async_mpm.{h,cpp}) as host code above the C-ABI.

The reference's AsyncMPM<dim> derives from MPM<dim>; per 4x4x8-node block it keeps a time-step level (a power-of-two multiple of
`unit_delta_t`, from the block's strength and CFL limits), a pool of particle records and a backup pool of frozen copies, and for
every level whose turn it is it gathers a particle set, sets base_delta_t and calls MPM<dim>::substep().  That substep is the
engine's; the scheduler around it (time levels, neighbour masks, the step loop: work per block) is restated here with numpy,
vectorised over blocks.  The pools (work per particle) live on the device: the engine keeps both as record arrays labelled with
their block (mpmb_async_*), reduces the pool to per-block limits for update_dt_limits and runs each advance — gather, pool
edits, the substep — without moving a particle record across the bus (DESIGN.md §8 row 3).  Records added before the first
step() are staged in `pool` / `backup` and move into the engine then.  An engine without those calls (the CPU suite's
stand-in) gets the same pools as numpy record arrays here, gathered and uploaded per advance: the reference the device pools
are tested against bit for bit.

An engine that also offers mpmb_async_schedule / mpmb_async_advance_level keeps the block state (level, local_min,
particle_t, backup_t) too and makes the scheduler's decisions per block on the device, the same decisions bit for bit as the
numpy code here: update_dt_limits is then one call returning the two level bounds, advance one call returning the gathered
count, and only the step loop and the clock stay on the host.  The numpy scheduler remains the one for every other engine and
the reference the device scheduler is tested against.

Citations are lines of src/async/async_mpm.cpp unless a file is named.  What cannot be reproduced bit for bit: the reference
takes 1/sqrt(max |v|^2) with `_mm_rsqrt_ss` (:78-80), a 12-bit hardware approximation; the exact reciprocal square root is used
here, which can move a block's CFL limit across an integer — and so its level — only when the limit sits within 2e-4 of one."""
import numpy as np

from . import capi, scenes
from .mpm import MPM


def _morton(bx, by, bz):
    """The scheduler's block order: the page index of SPGrid's linear offset for 32-byte elements in 4 KB pages — bits of the
    block coordinates interleaved (y, x, z) from the least significant (external/SPGrid/Core/SPGrid_Mask.h:40-44)."""
    out = np.zeros(np.shape(bx), np.int64)
    bx, by, bz = (np.asarray(a, np.int64) for a in (bx, by, bz))
    for i in range(12):
        out |= ((by >> i) & 1) << (3 * i)
        out |= ((bx >> i) & 1) << (3 * i + 1)
        out |= ((bz >> i) & 1) << (3 * i + 2)
    return out


def allowed_dt(kind, prm, F, ps, mass, vol, v, dx):
    """MPMParticle::get_allowed_dt of the registered types (src/particles.cpp:136-153, 254-281, 480-494, 649-668, 734-753, 814-833)."""
    f = np.float32
    J = np.linalg.det(F.reshape(-1, 3, 3).astype(np.float64)).astype(f)
    u = np.sqrt((v.astype(f) ** 2).sum(1))
    rho0 = mass.astype(f) / vol.astype(f)
    if kind == scenes.MAT_SNOW:
        J = J * ps.astype(f)
        h = np.exp(f(prm[2]) * (f(1.0) - ps.astype(f)))              # get_lame_parameters (src/particles.cpp:244-252)
        mu, lam = f(prm[0]) * h, f(prm[1]) * h
        c = np.sqrt((lam + f(2.0) * mu) / (rho0 / J))
    elif kind == scenes.MAT_WATER:
        c = np.sqrt(f(prm[0]) * f(prm[1]) / np.power(ps.astype(f), f(prm[1]) - f(1.0)))   # c^2 = k gamma / j^(gamma-1) (src/particles.cpp:480-482)
    elif kind in (scenes.MAT_SAND, scenes.MAT_VON_MISES, scenes.MAT_ELASTIC, scenes.MAT_VISCO):
        mu, lam = f(prm[0]), f(prm[1])
        K = f(2.0) * mu / f(3.0) + lam
        c2 = f(4.0) * mu / (f(3.0) * (rho0 / J)) + K * (f(1.0) - np.log(J)) / rho0
        c = np.sqrt(np.maximum(c2, f(1e-20)))
    else:
        raise ValueError("particle type without a time-step limit (jelly / linear return 0: the reference stops, :112-124)")
    return f(dx) / (c + u)


class AsyncMPM(MPM):
    """`tc.dynamics.MPM(..., async=True)` / scripts/async/async_mpm.py: the same surface as MPM plus the scheduler's keys
    unit_delta_t (1e-6), max_units (8192), cfl_dt_mul (1.0), strength_dt_mul (1.0) (:21-24)."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        if self.rigids:
            raise ValueError("AsyncMPM with rigid bodies is not supported")
        self.unit_delta_t = float(np.float32(kwargs.get("unit_delta_t", 1e-6)))
        self.max_units = int(kwargs.get("max_units", 8192))
        self.cfl_dt_mul = float(kwargs.get("cfl_dt_mul", 1.0))
        self.strength_dt_mul = float(kwargs.get("strength_dt_mul", 1.0))
        spgrid = 4096                                                      # src/mpm.cpp:50-54
        while spgrid // 2 > max(self.res) + 1:
            spgrid //= 2
        self.nb = (spgrid // 4, spgrid // 4, spgrid // 8)                 # scheduler blocks = SPGrid pages (:16)
        shape = self.nb
        gx, gy, gz = np.meshgrid(*(np.arange(n) for n in shape), indexing="ij")
        self._offset = _morton(gx, gy, gz)                                 # [bx,by,bz] -> scheduler offset (gather order)
        self.level = np.ones(shape, np.int64)                              # continuous_dt_limit (:32)
        self.local_min = np.ones(shape, np.int64)
        self.particle_t = np.zeros(shape, np.int64)
        self.backup_t = np.zeros(shape, np.int64)
        self.current_t_int = 0
        self.min_delta_t_int = self.max_delta_t_int = 1
        self.pool = None       # particle_pool: dict of record arrays + "block" [n,3] (host pools, or staged before the first step)
        self.backup = None     # backup_pool
        self._next_id = 0
        self._device_pools = hasattr(self.engine, "async_advance")   # the engine keeps the pools (mpmb_async_*)
        # ... and the block state with the scheduler's decisions (mpmb_async_schedule / mpmb_async_advance_level)
        self._device_sched = self._device_pools and hasattr(self.engine, "async_schedule")
        self._on_device = False    # the staged records have moved into the engine's pools (first step)
        self.step_counter = 0
        self._async_updates = 0

    # ---- pools
    @staticmethod
    def _empty_like(rec):
        return {k: v[:0].copy() for k, v in rec.items()}

    @staticmethod
    def _cat(a, b):
        if a is None or len(a["id"]) == 0:
            return b
        if b is None or len(b["id"]) == 0:
            return a
        return {k: np.concatenate([a[k], b[k]]) for k in a}

    def _block_of(self, x):
        X = x.astype(np.float32) * np.float32(1.0 / self.delta_x)
        base = (X - np.float32(0.5)).astype(np.int32)                      # get_grid_base_pos (src/mpm.h:244-247)
        return np.stack([base[:, 0] >> 2, base[:, 1] >> 2, base[:, 2] >> 3], 1)

    def add_particles(self, **kwargs):
        """AsyncMPM::add_particles (:60-76): the new particles go to the pool of their block."""
        if kwargs.get("type") == "rigid":
            raise ValueError("AsyncMPM with rigid bodies is not supported")
        before = None if self._host is None else len(self._host["x"])
        # the pools own the particles and advance() uploads them itself, so _n_uploaded stays 0: MPM.add_particles never
        # appends on the device here, it always leaves the new particles in self._host
        ret = super().add_particles(**kwargs)
        h = self._host
        lo = 0 if before is None else before
        rec = {k: np.ascontiguousarray(h[k][lo:]) for k in ("x", "v", "F", "b", "mass", "vol", "ps", "group")}
        n0 = int(self._next_id)
        rec["id"] = np.arange(n0, n0 + len(rec["x"]), dtype=np.int64)
        self._next_id = n0 + len(rec["x"])
        rec["block"] = self._block_of(rec["x"])
        if self._on_device:
            self.engine.async_add(0, rec)                                  # the engine computes the same blocks from x
        else:
            self.pool = self._cat(self.pool, rec)
            if self.backup is None:
                self.backup = self._empty_like(rec)
        self._host, self._dirty = None, False                              # this->particles.clear() (:75): the pools own the particles
        return ret

    def _pools_to_device(self):
        """First step with an engine that keeps the pools: the records staged by add_particles move into them."""
        if not self._device_pools or self._on_device:
            return
        self.engine.async_init(self.nb, np.float32(1.0 / self.delta_x))
        for which, rec in ((0, self.pool), (1, self.backup)):
            if rec is not None and len(rec["id"]):
                self.engine.async_add(which, rec)
        self.pool = self.backup = None
        if self._device_sched:      # mpmb_async_init gave the engine's block state these arrays' initial values
            self.level = self.local_min = self.particle_t = self.backup_t = None
        self._on_device = True

    def block_state(self, fields=("level", "local_min", "particle_t", "backup_t")):
        """The scheduler's per-block state as int64 arrays of shape nb (read from the engine if it keeps them)."""
        if self._device_sched and self._on_device:
            return self.engine.async_block_state(fields)
        return {k: getattr(self, k).copy() for k in fields}

    def pools(self):
        """(particle_pool, backup_pool) as host record dicts in pool order (read from the device pools if the engine keeps them)."""
        if not self._on_device:
            return self.pool, self.backup
        out = []
        for which in (0, 1):
            d = self.engine.async_download(which)
            blk = np.stack(np.unravel_index(d.pop("block"), self.nb), 1).astype(np.int32)
            d["id"] = d["id"].astype(np.int64)
            d["block"] = blk
            out.append(d)
        return tuple(out)

    # ---- update_dt_limits (:90-254)
    def _neighbour_levels(self):
        """For every block the 26 neighbours' (level, particle_t + level), out-of-range neighbours masked (the scheduler's
        cached_neighbours, src/async/async_mpm.h:255-300)."""
        big = np.int64(1) << 62
        pad_l = np.pad(self.level, 1, constant_values=0)
        pad_e = np.pad(self.particle_t + self.level, 1, constant_values=big)
        nx, ny, nz = self.nb
        for i in (0, 1, 2):
            for j in (0, 1, 2):
                for k in (0, 1, 2):
                    if (i, j, k) != (1, 1, 1):
                        yield (i - 1, j - 1, k - 1), pad_l[i:i + nx, j:j + ny, k:k + nz], pad_e[i:i + nx, j:j + ny, k:k + nz]

    def _pool_scan(self, t):
        """The pass over the particle pool: its occupied blocks, and a function returning per block (flat) min(0.1, allowed_dt)
        and max |v|^2 (:100-112).  Device pools: one mpmb_async_block_limits call, with the limits whenever some block's level
        is aligned to the clock (only such a block can be due)."""
        nblk = int(np.prod(self.nb))
        if self._on_device:
            aligned = (t & (self.level - 1)) == 0
            try:
                blk, mn, mx = self.engine.async_block_limits(bool(aligned.any()))
            except capi.MpmbError as e:
                if e.code != -1:
                    raise
                blk, _, _ = self.engine.async_block_limits(False)      # a type without a limit matters only if a block is due
                if aligned.reshape(-1)[blk].any():
                    raise ValueError("particle type without a time-step limit (jelly / linear return 0: the reference stops, :112-124)") from e
                mn = mx = None
            nonempty = np.zeros(nblk, bool)
            nonempty[blk] = True

            def limits():
                min_adt = np.full(nblk, np.float32(0.1))
                max_v2 = np.full(nblk, np.float32(1e-16))
                min_adt[blk], max_v2[blk] = mn, mx
                return min_adt, max_v2
            return nonempty.reshape(self.nb), limits
        p = self.pool
        nonempty = np.zeros(self.nb, bool)
        if p is None or len(p["id"]) == 0:
            return nonempty, None
        blk = p["block"]
        nonempty[blk[:, 0], blk[:, 1], blk[:, 2]] = True

        def limits():
            lin = (blk[:, 0] * self.nb[1] + blk[:, 1]) * self.nb[2] + blk[:, 2]
            adt = np.full(len(lin), 0.1, np.float32)
            for g, (kind, prm) in enumerate(self._groups):
                m = p["group"] == g
                if m.any():
                    adt[m] = np.minimum(np.float32(0.1), allowed_dt(kind, prm, p["F"][m], p["ps"][m], p["mass"][m], p["vol"][m], p["v"][m], self.delta_x))
            v2 = (p["v"].astype(np.float32) ** 2).sum(1)
            min_adt = np.full(nblk, np.float32(0.1))
            max_v2 = np.full(nblk, np.float32(1e-16))
            np.minimum.at(min_adt, lin, adt)
            np.maximum.at(max_v2, lin, v2)
            return min_adt, max_v2
        return nonempty, limits

    def update_dt_limits(self):
        t = self.current_t_int
        inv_unit = np.float32(1.0) / np.float32(self.unit_delta_t)
        if self._device_sched:
            self._pools_to_device()
            try:
                self.min_delta_t_int, self.max_delta_t_int = self.engine.async_schedule(
                    t, np.float32(self.strength_dt_mul), np.float32(self.cfl_dt_mul), np.float32(self.delta_x), inv_unit, self.max_units)
            except capi.MpmbError as e:
                if e.code == capi.ERR_INVALID:
                    raise ValueError("particle type without a time-step limit (jelly / linear return 0: the reference stops, :112-124)") from e
                if e.code == capi.ERR_LIMIT:
                    raise RuntimeError("a block's time-step limit is below unit_delta_t (the reference stops here, :115-124)") from e
                raise
            return
        nonempty, limits = self._pool_scan(t)
        if nonempty.any():
            due = nonempty & ((t & (self.level - 1)) == 0)                  # :95-96
            if due.any():
                min_adt, max_v2 = limits()
                sdl = (np.float32(self.strength_dt_mul) * min_adt * inv_unit).astype(np.int64).reshape(self.nb)          # :110
                cdl = (np.float32(self.cfl_dt_mul) * np.float32(self.delta_x) * inv_unit * (np.float32(1.0) / np.sqrt(max_v2))).astype(np.int64).reshape(self.nb)   # :111-112
                tmp = np.minimum(np.minimum(cdl, sdl), self.max_units)
                if (tmp[due] < 1).any():
                    raise RuntimeError("a block's time-step limit is below unit_delta_t (the reference stops here, :115-124)")
                lv = self.level.copy()
                for _ in range(64):                                         # while (tmp_limit < limit) limit >>= 1  (:125-127)
                    m = due & (tmp < lv)
                    if not m.any():
                        break
                    lv[m] >>= 1
                for _ in range(64):                                         # grow while allowed and aligned (:128-131)
                    m = due & (tmp >= (lv << 1)) & ((t & ((lv << 1) - 1)) == 0)
                    if not m.any():
                        break
                    lv[m] <<= 1
                self.level = lv
        if nonempty.any():                                                  # update_dt_limit_boundary(true)
            self.min_delta_t_int, self.max_delta_t_int = int(self.level[nonempty].min()), int(self.level[nonempty].max())
        else:
            self.min_delta_t_int, self.max_delta_t_int = 1 << 31, 1
        due = (~nonempty) & ((t & (self.level - 1)) == 0)                   # empty blocks (:138-152)
        lv = self.level.copy()
        for _ in range(64):
            m = due & (self.max_delta_t_int < lv)
            if not m.any():
                break
            lv[m] >>= 1
        for _ in range(64):
            m = due & (self.max_delta_t_int >= (lv << 1)) & ((t & ((lv << 1) - 1)) == 0)
            if not m.any():
                break
            lv[m] <<= 1
        self.level = lv
        self.min_delta_t_int, self.max_delta_t_int = int(self.level.min()), int(self.level.max())   # update_dt_limit_boundary(false)
        # local_min_dt_limit (:165-181): the earliest time a neighbour will be stepped next
        lm = np.full(self.nb, np.int64(1) << 31)
        for _, _, nb_next in self._neighbour_levels():
            lm = np.minimum(lm, nb_next)
        keep = self.level == self.min_delta_t_int
        self.local_min = np.where(keep, self.local_min, lm)
        # larger / smaller neighbours per level (:183-250), as boolean block masks per log2 level
        self._larger, self._smaller = {}, {}
        for off, nl, _ in self._neighbour_levels():
            has = nl > 0
            mine_smaller = has & (self.level < nl)                           # this block is finer than that neighbour
            if not mine_smaller.any():
                continue
            idx = np.argwhere(mine_smaller)
            nbr = idx + np.asarray(off)
            for lg in np.unique(np.log2(self.level[mine_smaller]).astype(int)):
                sel = np.log2(self.level[idx[:, 0], idx[:, 1], idx[:, 2]]).astype(int) == lg
                m = self._larger.setdefault(int(lg), np.zeros(self.nb, bool))
                m[nbr[sel, 0], nbr[sel, 1], nbr[sel, 2]] = True              # larger_neighbours[log2(level[offset])] gets the neighbour
            nl_here = self.level[nbr[:, 0], nbr[:, 1], nbr[:, 2]]
            for lg in np.unique(np.log2(nl_here).astype(int)):
                sel = np.log2(nl_here).astype(int) == lg
                m = self._smaller.setdefault(int(lg), np.zeros(self.nb, bool))
                m[idx[sel, 0], idx[sel, 1], idx[sel, 2]] = True              # smaller_neighbours[log2(level[neighbour])] gets this block

    # ---- advance (:256-373)
    def _select(self, rec, mask3):
        if rec is None or len(rec["id"]) == 0:
            return None
        b = rec["block"]
        m = mask3[b[:, 0], b[:, 1], b[:, 2]]
        return {k: v[m] for k, v in rec.items()} if m.any() else None

    def advance(self, limit):
        t = self.current_t_int
        if self._device_sched:
            self._pools_to_device()
            self._async_updates += self.engine.async_advance_level(t, limit, float(np.float32(self.unit_delta_t) * np.float32(limit)))
            return
        lg = int(np.log2(limit))
        smaller = self._smaller.get(lg, np.zeros(self.nb, bool))
        larger = self._larger.get(lg, np.zeros(self.nb, bool))
        equal = self.level == limit
        has_copied = smaller | larger                                       # :262-268, :300-310
        swap = equal & (self.particle_t == t)                               # backup_current_dt_limit (:318-326)
        drop = has_copied & (self.level > limit) & (self.local_min == t + limit)
        clear_b = drop & ~equal                                             # :331-343
        dt = float(np.float32(self.unit_delta_t) * np.float32(limit))       # :407-409
        if self._on_device:
            flags = (smaller * capi.ASYNC_SMALLER | equal * capi.ASYNC_EQUAL | larger * capi.ASYNC_LARGER | swap * capi.ASYNC_SWAP |
                     clear_b * capi.ASYNC_CLEAR).astype(np.uint8)
            n = self.engine.async_advance(flags, dt)                        # gather, pool edits and the substep, on the device
        else:
            n = self._advance_host(smaller, equal, larger, swap, clear_b, dt)
        self._async_updates += n                                            # update_counter += particles.size() (:328)
        # update backup_t and particle_t (:318-343)
        self.backup_t = np.where(swap, t, self.backup_t)
        self.particle_t = np.where(equal, t + limit, self.particle_t)
        self.backup_t = np.where(clear_b, t + limit, self.backup_t)

    def _advance_host(self, smaller, equal, larger, swap, clear_b, dt):
        """The pool work of one advance on host pools; returns the size of the gathered set."""
        parts = [self._select(self.pool, smaller), self._select(self.pool, equal), self._select(self.backup, larger)]
        g = None
        for q in parts:                                                     # gather order: smaller neighbours, this level, larger neighbours' backups
            if q is not None:
                o = np.argsort(self._offset[q["block"][:, 0], q["block"][:, 1], q["block"][:, 2]], kind="stable")
                g = self._cat(g, {k: v[o] for k, v in q.items()})
        if g is not None:                                                   # particles_cnt / global_cnt: the first copy of an id wins
            _, first = np.unique(g["id"], return_index=True)
            g = {k: v[np.sort(first)] for k, v in g.items()}
        # backup_current_dt_limit (:318-326): the level's pools become their blocks' backups
        if self.pool is not None and len(self.pool["id"]):
            pb = self.pool["block"]
            mv = swap[pb[:, 0], pb[:, 1], pb[:, 2]]
            bb = self.backup["block"]
            keep_b = ~swap[bb[:, 0], bb[:, 1], bb[:, 2]] if len(bb) else np.zeros(0, bool)
            self.backup = self._cat({k: v[keep_b] for k, v in self.backup.items()}, {k: v[mv] for k, v in self.pool.items()})
            self.pool = {k: v[~mv] for k, v in self.pool.items()}
        n = 0 if g is None else len(g["id"])
        out = None
        if n:
            self.engine.set_delta_t(dt)
            self.engine.upload(g["x"], g["v"], g["mass"], g["vol"], g["F"], g["b"], g["ps"], g["group"].astype(np.int32))
            self.engine.substep(1)                                          # MPM<dim>::substep() (:329)
            d = self.engine.download()
            k = d["id"].astype(np.int64)                                    # upload index of the survivors
            out = dict(x=d["x"], v=d["v"], F=d["F"], b=d["b"], mass=d["mass"], vol=d["vol"], ps=d["ps"], group=g["group"][k], id=g["id"][k])
            out["block"] = self._block_of(out["x"])
        if len(self.backup["id"]):                                          # blocks whose backups were consumed (:331-343)
            bb = self.backup["block"]
            self.backup = {k: v[~clear_b[bb[:, 0], bb[:, 1], bb[:, 2]]] for k, v in self.backup.items()}
        # update backup_pool and particle_pool (:345-370)
        if out is not None and len(out["id"]):
            ob = out["block"]
            to_pool = equal[ob[:, 0], ob[:, 1], ob[:, 2]]
            to_backup = (~to_pool) & clear_b[ob[:, 0], ob[:, 1], ob[:, 2]]
            self.pool = self._cat(self.pool, {k: v[to_pool] for k, v in out.items()})
            self.backup = self._cat(self.backup, {k: v[to_backup] for k, v in out.items()})
        return n

    # ---- step (:375-421)
    def step(self, dt):
        if dt < 0:
            raise ValueError("AsyncMPM.step needs dt >= 0 here")
        self.request_t = np.float32(self.request_t + np.float32(dt))
        self._pools_to_device()
        while True:
            self.update_dt_limits()
            delta = self.max_delta_t_int
            while delta >= self.min_delta_t_int:
                if self.current_t_int % delta == 0:
                    self.current_t = np.float32(np.float32(self.unit_delta_t) * np.float32(self.current_t_int))
                    self.advance(delta)
                delta >>= 1
            self.current_t_int += self.min_delta_t_int - self.current_t_int % self.min_delta_t_int
            self.current_t = np.float32(np.float32(self.unit_delta_t) * np.float32(self.current_t_int))
            if not (self.current_t < self.request_t):
                break
        self.step_counter += 1

    @property
    def update_counter(self):
        return self._async_updates

    @update_counter.setter
    def update_counter(self, value):
        self._async_updates = int(value)

    def get_particles(self):
        """The particles of the pools by id (every live particle's current record is the LAST one a pool received for its id)."""
        p = self.pools()[0]
        if p is None or len(p["id"]) == 0:
            return {k: np.zeros((0,) + s, np.float32) for k, s in (("x", (3,)), ("v", (3,)), ("F", (9,)), ("b", (9,)), ("mass", ()), ("vol", ()), ("ps", ()))}
        o = np.argsort(self._offset[p["block"][:, 0], p["block"][:, 1], p["block"][:, 2]], kind="stable")
        q = {k: v[o] for k, v in p.items()}
        _, last = np.unique(q["id"][::-1], return_index=True)
        sel = np.sort(len(q["id"]) - 1 - last)
        sel = sel[np.argsort(q["id"][sel], kind="stable")]
        return {k: v[sel] for k, v in q.items() if k != "block"}

    def num_particles(self):
        p = self.pool if not self._on_device else self.engine.async_download(0, ("id",))
        return 0 if p is None else len(np.unique(p["id"]))

    def visualize(self):
        """The frame dump of MPM.visualize from the pools (the engine only ever holds the particle set of the last advance)."""
        import os
        from . import bgeo
        from .mpm import frame_attributes
        if not self.frame_directory:
            raise ValueError("frame_directory was not given to AsyncMPM(...)")
        self.frame_count += 1
        os.makedirs(self.frame_directory, exist_ok=True)
        fn = os.path.join(self.frame_directory, "%04d.bgeo" % self.frame_count)
        p = self.get_particles()
        p = dict(p, id=p["id"].astype(np.uint32))
        bgeo.write_bgeo(fn, p["x"], frame_attributes(p, [k for k, _ in self._groups], self.verbose_bgeo))
        return fn

    def general_action(self, **kwargs):
        if kwargs.get("action") in ("save", "load", "delete_particles_inside_level_set"):
            raise ValueError("AsyncMPM: %s is not supported (the reference's AsyncMPM::io is a stub too, src/async/async_mpm.h:126-129)" % kwargs["action"])
        return super().general_action(**kwargs)

    def scheduler_stats(self):
        p = self.pools()[0]
        ne = np.zeros(self.nb, bool)
        if p is not None and len(p["id"]):
            ne[p["block"][:, 0], p["block"][:, 1], p["block"][:, 2]] = True
        level = self.block_state(("level",))["level"]
        return dict(pool_entries=0 if p is None else len(p["id"]), update_counter=self._async_updates, current_t_int=self.current_t_int,
                    min_level=int(level[ne].min()) if ne.any() else 0, max_level=int(level[ne].max()) if ne.any() else 0)
