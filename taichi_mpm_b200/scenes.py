"""Synthetic inputs for the BASELINE.json configs (numpy, host side).

Generator = the reference's deterministic `benchmark` lattice (src/mpm.cpp:149-186): 8 particles
per cell at cell-centre +- 0.25 dx, with the physically consistent volume vol = dx^3/8
(texture-seeding convention vol = dx^dim / maximum, src/mpm.cpp:134-135) and mass = vol*density.
Material parameter vectors follow include/mpmb.h; defaults are the reference's
(src/particles.cpp:192-205,383-389,448-449,570-597).
"""
import math

import numpy as np

MAT_LINEAR, MAT_JELLY, MAT_SNOW, MAT_WATER, MAT_SAND, MAT_ELASTIC, MAT_VON_MISES, MAT_VISCO = range(8)
N_MAT_PARAMS = 8


def lame(E, nu):
    mu = E / (2 * (1 + nu))
    lam = E * nu / ((1 + nu) * (1 - 2 * nu))
    return mu, lam


def material_params(kind, **kw):
    """Parameter vector of a reference particle type, with the reference's defaults."""
    p = np.zeros(N_MAT_PARAMS, np.float32)
    if kind in (MAT_LINEAR, MAT_JELLY):  # src/particles.cpp:317-323,383-389
        mu, lam = lame(kw.get("E", 1e5), kw.get("nu", 0.3))
        p[0], p[1] = mu, lam
    elif kind == MAT_SNOW:  # src/particles.cpp:192-205
        E, nu = kw.get("youngs_modulus", 1.4e5), kw.get("poisson_ratio", 0.2)
        mu, lam = lame(E, nu)
        p[0], p[1] = kw.get("mu_0", mu), kw.get("lambda_0", lam)
        p[2] = kw.get("hardening", 10.0)
        p[3], p[4] = kw.get("theta_c", 2.5e-2), kw.get("theta_s", 7.5e-3)
        p[5], p[6] = kw.get("min_Jp", 0.6), kw.get("max_Jp", 20.0)
    elif kind == MAT_WATER:  # src/particles.cpp:448-461
        p[0], p[1] = kw.get("k", 1e4), kw.get("gamma", 7.0)
    elif kind == MAT_SAND:  # src/particles.cpp:570-597
        p[0], p[1] = kw.get("mu_0", 136038.0), kw.get("lambda_0", 204057.0)
        phi = kw.get("friction_angle", 30.0)
        s = math.sin(np.float32(phi) / np.float32(180.0) * np.float32(3.141592653))
        p[2] = math.sqrt(2.0 / 3.0) * 2.0 * s / (3.0 - s)
        p[3], p[4] = kw.get("cohesion", 0.0), kw.get("beta", 1.0)
    elif kind == MAT_ELASTIC:  # src/particles.cpp:775-781 (keys "E", "nu")
        p[0], p[1] = lame(kw.get("E", 5e3), kw.get("nu", 0.4))
    elif kind == MAT_VON_MISES:  # src/particles.cpp:691-700
        p[0], p[1] = lame(kw.get("youngs_modulus", 5e3), kw.get("poisson_ratio", 0.4))
        p[2] = kw.get("yield_stress", 1.0)
    elif kind == MAT_VISCO:  # src/particles.cpp:55-67; [4] is the particle's own copy of base_delta_t (default 1e-4)
        p[0], p[1] = lame(kw.get("youngs_modulus", 4e4), kw.get("poisson_ratio", 0.4))
        p[2], p[3], p[4] = kw.get("nu", 10000.0), kw.get("kappa", 0.0), kw.get("base_delta_t", 1e-4)
    else:
        raise ValueError("unknown material kind %r" % (kind,))
    return p


def default_scalar(kind):
    if kind == MAT_VISCO:
        return 1000.0  # visco_tau (src/particles.cpp:62)
    return 1.0 if kind in (MAT_SNOW, MAT_WATER) else 0.0  # Jp=1, j=1, logJp=0


def lattice_block(res, lo_cell, hi_cell, density=400.0, jitter=0.0, seed=20260922, dtype=np.float32, dx=None):
    """8 particles per cell over cells [lo_cell, hi_cell) (3-vectors) of cell size dx (default 1/res): positions
    (cell + 0.5 +- 0.25) * dx, where add_particles(benchmark=...) puts them with its delta_x (src/mpm.cpp:168-178);
    vol = dx^3 / 8 and mass = vol * density (see above)."""
    dx = 1.0 / res if dx is None else float(dx)
    lo = np.asarray(lo_cell, np.int64)
    hi = np.asarray(hi_cell, np.int64)
    ii, jj, kk = np.meshgrid(np.arange(lo[0], hi[0]), np.arange(lo[1], hi[1]), np.arange(lo[2], hi[2]), indexing="ij")
    centre = (np.stack([ii, jj, kk], -1).reshape(-1, 1, 3) + 0.5)  # cell centre, grid units
    sign = np.array([[(-1 if (i % 2 == 0) else 1), (-1 if (i // 2 % 2 == 0) else 1), (-1 if (i // 4 % 2 == 0) else 1)] for i in range(8)],
                    np.float64)
    X = (centre + 0.25 * sign[None]).reshape(-1, 3)
    if jitter > 0:
        rng = np.random.default_rng(seed)
        X = X + rng.uniform(-jitter, jitter, X.shape)
    x = (X * dx).astype(dtype)
    n = len(x)
    vol = np.full(n, dx ** 3 / 8.0, dtype)
    mass = (vol * density).astype(dtype)
    return x, mass, vol


def seed_hash(idx, axis, seed):
    """Counter-based hash of (lattice index, axis, seed) -> uint32; the numpy twin of seed_hash in csrc/mpmb_engine.cu."""
    with np.errstate(over="ignore"):
        h = (idx.astype(np.uint32) * np.uint32(3) + np.uint32(axis)) ^ np.uint32(seed)
        h = h * np.uint32(0x9E3779B1)
        h ^= h >> np.uint32(16)
        h = h * np.uint32(0x85EBCA6B)
        h ^= h >> np.uint32(13)
        h = h * np.uint32(0xC2B2AE35)
        h ^= h >> np.uint32(16)
    return h


def lattice_block_hashed(res, lo_cell, hi_cell, density=400.0, jitter=0.0, seed=20260922, z_cells=None, dx=None):
    """The `benchmark` lattice of MPM<3>::add_particles (src/mpm.cpp:149-186) with a jitter that is a hash of the
    particle's lattice index — the host twin of mpmb_seed_lattice (device-side seeding), float32 operation for float32
    operation, so both produce the same bits whatever the z-slab partition.  Returns (ids, x, mass, vol); particles in
    the 7-cell boundary band are dropped as add_particles drops them (src/mpm.cpp:129-132).
    z_cells = (k0, k1): only the cell layers lo[2]+k0 .. lo[2]+k1-1 (a slab's share), ids unchanged.
    dx: the engine's cell size (default 1/res[0]), rounded to float32 as the engine stores it; vol = dx^3 / 8."""
    if np.isscalar(res):
        res = (res, res, res)
    f32 = np.float32
    cell = 1.0 / res[0] if dx is None else float(dx)
    dx = f32(cell)
    lo = np.asarray(lo_cell, np.int64)
    n = np.asarray(hi_cell, np.int64) - lo
    k0, k1 = (0, int(n[2])) if z_cells is None else z_cells
    kx, ky, kz, c = np.meshgrid(np.arange(n[0]), np.arange(n[1]), np.arange(k0, k1), np.arange(8), indexing="ij")
    kx, ky, kz, c = (a.reshape(-1) for a in (kx, ky, kz, c))
    lattice = (((kx * n[1] + ky) * n[2] + kz) * 8 + c).astype(np.uint32)
    X = np.empty((len(lattice), 3), f32)
    for a, k in enumerate((kx, ky, kz)):
        off = np.where((c >> a) & 1, f32(0.75), f32(0.25)).astype(f32)
        u = (seed_hash(lattice, a, seed) >> np.uint32(8)).astype(f32) * f32(1.0 / 8388608.0) - f32(1.0)
        X[:, a] = ((lo[a] + k).astype(f32) + off) + f32(jitter) * u
    x = X * dx
    keep = (X.min(1) >= f32(7.0)) & ((X - np.asarray(res, f32)).max(1) <= f32(-7.0))
    vol = np.full(int(keep.sum()), cell ** 3 / 8.0, f32)
    mass = (vol * f32(density)).astype(f32)
    return lattice[keep], x[keep], mass, vol


def make_state(x, mass, vol, kind, group=0, v0=(0.0, 0.0, 0.0)):
    n = len(x)
    F = np.zeros((n, 9), np.float32)
    F[:, 0] = F[:, 4] = F[:, 8] = 1.0
    return dict(x=x.astype(np.float32), v=np.tile(np.asarray(v0, np.float32), (n, 1)), F=F, b=np.zeros((n, 9), np.float32),
                mass=mass.astype(np.float32), vol=vol.astype(np.float32), ps=np.full(n, default_scalar(kind), np.float32),
                group=np.full(n, group, np.int32), alive=np.ones(n, np.uint8))


def floor_sdf(res, floor_cells, dtype=np.float32):
    """Dense node level set of one floor plane y >= floor_cells (grid units): (n, phi)."""
    n = res + 1
    sdf = np.zeros((n, n, n, 4), dtype)
    sdf[..., 1] = 1.0
    sdf[..., 3] = (np.arange(n, dtype=np.float64) - floor_cells)[None, :, None]
    return sdf


def planes_sdf(res, planes, dtype=np.float32):
    """Dense node level set of an intersection of half-spaces phi_i = n_i.X + d_i (grid units)."""
    if np.isscalar(res):
        res = (res, res, res)
    nn = [r + 1 for r in res]
    I, J, K = np.meshgrid(np.arange(nn[0], dtype=np.float32), np.arange(nn[1], dtype=np.float32), np.arange(nn[2], dtype=np.float32),
                          indexing="ij")
    best = np.full(nn, 1e30, np.float32)
    out = np.zeros(tuple(nn) + (4,), np.float32)
    out[..., 0] = 1.0
    out[..., 3] = 1e30
    for pl in np.asarray(planes, np.float32).reshape(-1, 4):
        phi = pl[0] * I + pl[1] * J + pl[2] * K + pl[3]
        m = phi < best
        best = np.where(m, phi, best)
        out[m, 0], out[m, 1], out[m, 2] = pl[0], pl[1], pl[2]
        out[..., 3] = np.where(m, phi, out[..., 3])
    return out.astype(dtype)


def shapes_sdf(res, shapes, dtype=np.float32):
    """Numpy twin of mpmb_set_levelset_shapes (include/mpmb.h): dense node level set (n, phi) in grid units from
    [(kind, inside_out, params)], kind 0 plane / 1 sphere / 2 cuboid; phi = min over shapes."""
    if np.isscalar(res):
        res = (res, res, res)
    nn = [r + 1 for r in res]
    X = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float32) for n in nn], indexing="ij"), -1)
    best = np.full(nn, 1e30, np.float32)
    out = np.zeros(tuple(nn) + (4,), np.float32)
    out[..., 0] = 1.0
    out[..., 3] = 1e30
    f32 = np.float32
    for kind, io, prm in shapes:
        p = np.asarray(list(prm) + [0.0] * (6 - len(prm)), np.float32)
        if kind == 0:
            n = np.broadcast_to(p[:3], X.shape).copy()
            phi = p[0] * X[..., 0] + p[1] * X[..., 1] + p[2] * X[..., 2] + p[3]
        elif kind == 1:
            d = X - p[:3]
            r = np.sqrt((d * d).sum(-1, dtype=np.float32))
            with np.errstate(divide="ignore", invalid="ignore"):
                n = np.where(r[..., None] > 1e-20, d * (f32(1.0) / r)[..., None], np.array([1.0, 0.0, 0.0], np.float32))
            phi = r - p[3]
        else:
            c, hw = f32(0.5) * (p[:3] + p[3:6]), f32(0.5) * (p[3:6] - p[:3])
            d = X - c
            sgn = np.where(d < 0, f32(-1), f32(1))
            q = np.abs(d) - hw
            qp = np.where(q > 0, q, f32(0))
            out2 = (qp * qp).sum(-1, dtype=np.float32)
            r = np.sqrt(out2)
            with np.errstate(divide="ignore", invalid="ignore"):
                n_out = sgn * qp * (f32(1.0) / r)[..., None]
            amax = np.argmin(-q, -1)            # first axis of least depth
            n_in = np.zeros_like(d)
            np.put_along_axis(n_in, amax[..., None], np.take_along_axis(sgn, amax[..., None], -1), -1)
            outside = out2 > 0
            n = np.where(outside[..., None], n_out, n_in)
            phi = np.where(outside, r, -(-q).min(-1))
        if io:
            n, phi = -n, -phi
        m = phi < best
        best = np.where(m, phi, best)
        out[..., :3] = np.where(m[..., None], n, out[..., :3])
        out[..., 3] = best
    return out.astype(dtype)


# ---------------------------------------------------------------------------------------------------- 2-D (MPM<2>)
def lattice_block2d(res, lo_cell, hi_cell, density=400.0, jitter=0.0, seed=20260922, dx=None, maximum=4):
    """The 2-D lattice of this project (the reference's `benchmark` branch is 3-D only, src/mpm.cpp:152): 4 particles
    per cell over cells [lo_cell, hi_cell) at (cell + 0.5 +- 0.25) * dx, vol = dx^2 / maximum (the texture-seeding
    convention vol = dx^dim / maximum, src/mpm.cpp:134-135), mass = vol * density."""
    dx = 1.0 / res[0] if dx is None else float(dx)
    lo, hi = np.asarray(lo_cell, np.int64), np.asarray(hi_cell, np.int64)
    ii, jj = np.meshgrid(np.arange(lo[0], hi[0]), np.arange(lo[1], hi[1]), indexing="ij")
    centre = np.stack([ii, jj], -1).reshape(-1, 1, 2) + 0.5
    sign = np.array([[-1, -1], [-1, 1], [1, -1], [1, 1]], np.float64)
    X = (centre + 0.25 * sign[None]).reshape(-1, 2)
    if jitter > 0:
        X = X + np.random.default_rng(seed).uniform(-jitter, jitter, X.shape)
    x = (X * dx).astype(np.float32)
    vol = np.full(len(x), dx * dx / maximum, np.float32)
    return x, (vol * density).astype(np.float32), vol


def make_state2d(x, mass, vol, kind, group=0, v0=(0.0, 0.0)):
    n = len(x)
    F = np.zeros((n, 4), np.float32)
    F[:, 0] = F[:, 3] = 1.0
    return dict(x=np.asarray(x, np.float32), v=np.tile(np.asarray(v0, np.float32), (n, 1)), F=F, b=np.zeros((n, 4), np.float32),
                mass=np.asarray(mass, np.float32), vol=np.asarray(vol, np.float32), ps=np.full(n, default_scalar(kind), np.float32),
                group=np.full(n, group, np.int32), alive=np.ones(n, np.uint8))


def flat_shapes2d(shapes):
    """2-D solids as the engine rasterises them (include/mpmb.h, dim = 2): plane (n_x, n_y, 0, d), circle (c_x, c_y, 0, r)
    and rectangle (lo_x, lo_y, 0, hi_x, hi_y, 0); a rectangle is the cuboid that is unbounded along z."""
    out = []
    for kind, io, prm in shapes:
        p = [float(v) for v in prm] + [0.0] * (6 - len(prm))
        if (p[2] != 0.0) or (kind == 2 and p[5] != 0.0):
            raise ValueError("a 2-D shape has no z part: %r" % (prm,))
        if kind == 2:
            p[2], p[5] = -1e30, 1e30
        out.append((kind, io, p))
    return out


def shapes_sdf2d(res, shapes, dtype=np.float32):
    """Numpy twin of mpmb_set_levelset_shapes on a 2-D handle: (r0+1, r1+1, 4) = (n_x, n_y, 0, phi), grid units."""
    return shapes_sdf((int(res[0]), int(res[1]), 0), flat_shapes2d(shapes), dtype)[:, :, 0].copy()


def planes_sdf2d(res, planes, dtype=np.float32):
    """Numpy twin of mpmb_set_planes on a 2-D handle: planes (n_x, n_y, 0, d)."""
    return shapes_sdf2d(res, [(0, 0, p) for p in np.asarray(planes, np.float32).reshape(-1, 4)], dtype)


def config(name, scale=1.0, state=True):
    """The BASELINE.json configs as dict(scene=..., state=..., meta=...).

    `scale` < 1 shrinks grid and block together (parity-test sizes); 1.0 is the quoted size.
    state=False: no host particle arrays (meta carries the block for device-side seeding, mpmb_seed_lattice).
    scene: res, dx, dt, gravity, particle_gravity, mat_kind, mat_params, planes, friction
    """
    if name == "jelly128":      # config 2: 3D fixed-corotated block, 128^3 grid, 1M particles
        res, cells, kind, dt = 128, 50, MAT_JELLY, 1e-4
        kw, floor, friction = dict(E=1e5, nu=0.3), 0.1, -1.0
    elif name == "sand256":     # config 3 (north star): 256^3 grid, 8M Drucker-Prager sand
        res, cells, kind, dt = 256, 100, MAT_SAND, 2e-5
        kw, floor, friction = dict(), None, 0.4
    elif name == "snow256":     # config 4: 256^3 grid, 16M snow, block 100x100x200
        res, cells, kind, dt = 256, 100, MAT_SNOW, 1e-4
        kw, floor, friction = dict(), None, 0.4
    elif name == "water512":    # config 5: 512^3 grid, 64M water
        res, cells, kind, dt = 512, 200, MAT_WATER, 5e-5
        kw, floor, friction = dict(), None, 0.4
    elif name == "linear125":   # the reference's own benchmark (scripts/benchmark/benchmark_3d.py)
        res, cells, kind, dt = 125, 100, MAT_LINEAR, 1e-2
        kw, floor, friction = dict(E=1e2, nu=0.3), None, None
    else:
        raise ValueError(name)
    res = int(round(res * scale))
    cells = int(round(cells * scale))
    dx = 1.0 / res
    if name == "jelly128":
        lo = np.array([(res - cells) // 2] * 3)
        hi = lo + cells
        floor_cells = floor * res
        gravity = (0.0, -10.0, 0.0)
    elif name == "linear125":
        lo = np.array([int(round(res * 0.1))] * 3)
        hi = lo + int(round(res * 0.8))
        floor_cells = None
        gravity = (0.0, 0.0, 0.0)
    else:
        floor_cells = 10.0
        lo = np.array([(res - cells) // 2, 10, (res - cells) // 2])
        hi = lo + cells
        if name == "snow256":
            lo[2] = (res - 2 * cells) // 2
            hi[2] = lo[2] + 2 * cells
        gravity = (0.0, -10.0, 0.0)
    n_block = int(np.prod(hi - lo)) * 8
    st = None
    if state:
        x, mass, vol = lattice_block(res, lo, hi, jitter=0.05, seed=20260922)
        st = make_state(x, mass, vol, kind)
        n_block = len(x)
    planes = None if floor_cells is None else np.array([[0.0, 1.0, 0.0, -floor_cells]], np.float32)
    scene = dict(res=(res, res, res), dx=dx, dt=dt, gravity=gravity, particle_gravity=1, mat_kind=np.array([kind], np.int32),
                 mat_params=material_params(kind, **kw)[None], planes=planes, friction=friction if planes is not None else 0.0)
    vol1 = np.float32((1.0 / res) ** 3 / 8.0)
    meta = dict(name=name, res=res, n=n_block, kind=kind, lo=tuple(int(v) for v in lo), hi=tuple(int(v) for v in hi), density=400.0,
                vol=float(vol1), mass=float(np.float32(vol1 * np.float32(400.0))), jitter=0.05, seed=20260922)
    return dict(scene=scene, state=st, meta=meta)


# --------------------------------------------------------------------------- rigid bodies (CPIC, SURVEY §8f row 2)
def rigid_boundary_samples(tris, dx, eps=1e-6):
    """The RigidBoundaryParticles MPM<3>::add_rigid_particle seeds on a triangle mesh (src/mpm_rigid_body.cpp:227-250):
    per element a lattice of spacing dx along its two edges from v0, starting at min(len/3, dx/2), points past an edge pulled
    back by dx/2, kept while x/|e1| + y/|e2| <= 1 - eps.  tris: [m,3,3] in the centroid frame.  Returns (offset[ns,3],
    tri[ns,9], element index[ns])."""
    tris = np.asarray(tris, np.float64).reshape(-1, 3, 3)
    off, tri, idx = [], [], []
    for e, (v0, v1, v2) in enumerate(tris):
        lx, ly = np.linalg.norm(v1 - v0), np.linalg.norm(v2 - v0)
        xn, yn = (v1 - v0) / lx, (v2 - v0) / ly
        _x = min(lx / 3.0, dx / 2.0)
        while _x < lx + dx:
            _y = min(ly / 3.0, dx / 2.0)
            while _y < ly + dx:
                x = _x if _x < lx else _x - dx / 2.0
                y = _y if _y < ly else _y - dx / 2.0
                if not (x / lx + y / ly > 1.0 - eps):
                    off.append(v0 + xn * x + yn * y)
                    tri.append(np.concatenate([v0, v1, v2]))
                    idx.append(e)
                _y += dx
            _x += dx
    return np.asarray(off, np.float32).reshape(-1, 3), np.asarray(tri, np.float32).reshape(-1, 9), np.asarray(idx, np.int32)


def box_mesh(half):
    """Triangles [12,3,3] of an axis-aligned box centred at the origin, outward normals."""
    hx, hy, hz = half
    c = np.array([[sx * hx, sy * hy, sz * hz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], np.float64)   # index = 4 sx + 2 sy + sz
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]   # -x +x -y +y -z +z, counter-clockwise from outside
    tris = []
    for a, b, cc, d in quads:
        tris += [[c[a], c[b], c[cc]], [c[a], c[cc], c[d]]]
    return np.asarray(tris)


def plate_mesh(half_u, half_v, axis=1):
    """Two triangles [2,3,3] of a thin (codimensional) rectangular plate through the origin, normal along +axis."""
    u, v = [a for a in range(3) if a != axis]
    p = np.zeros((4, 3))
    p[0, [u, v]] = [-half_u, -half_v]; p[1, [u, v]] = [half_u, -half_v]; p[2, [u, v]] = [half_u, half_v]; p[3, [u, v]] = [-half_u, half_v]
    t = np.array([[p[0], p[1], p[2]], [p[0], p[2], p[3]]])
    n = np.cross(t[0, 1] - t[0, 0], t[0, 2] - t[0, 0])
    return t if n[axis] > 0 else t[:, ::-1]


def euler_rotation(euler_deg):
    """Rotation matrix of create_rigid_body's `initial_rotation` (degrees; Rx(a) Ry(b) Rz(c), src/mpm_rigid_body.cpp:118-128)."""
    a, b, c = np.radians(np.asarray(euler_deg, np.float64))
    rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    rz = np.array([[np.cos(c), -np.sin(c), 0], [np.sin(c), np.cos(c), 0], [0, 0, 1]])
    return rx @ ry @ rz


def make_rigid(bodies, dx, penalty=0.0, pushing_force=20000.0):
    """Assembles the rigid-body description the engine and the oracle take.  bodies: list of dicts(tris[m,3,3] in the centroid
    frame, position[3], rotation (3x3 matrix, default I), velocity, angular_velocity, inv_mass (0 = scripted / infinite mass),
    inv_inertia (3x3 world-space, default 0), friction or frictions (2,)).  Body k of the list gets the reference's rigid id k+1
    (id 0 is MPM::rigids[0], the background body, src/mpm.cpp:72-74); at most 11 bodies (GridState::max_num_rigid_bodies = 12)."""
    nr = len(bodies) + 1
    if nr > 12:
        raise ValueError("at most 11 rigid bodies (GridState::max_num_rigid_bodies, src/mpm_fwd.h:79)")
    r = dict(position=np.zeros((nr, 3), np.float32), rot=np.tile(np.eye(3, dtype=np.float32).reshape(9), (nr, 1)), velocity=np.zeros((nr, 3), np.float32),
             angular_velocity=np.zeros((nr, 3), np.float32), inv_mass=np.zeros(nr, np.float32), inv_inertia=np.zeros((nr, 9), np.float32),
             frictions=np.zeros((nr, 2), np.float32), penalty=float(penalty), pushing_force=float(pushing_force))
    offs, tris, rid = [], [], []
    for k, b in enumerate(bodies):
        i = k + 1
        r["position"][i] = b["position"]
        r["rot"][i] = np.asarray(b.get("rotation", np.eye(3)), np.float32).T.reshape(9)      # column-major
        r["velocity"][i] = b.get("velocity", (0, 0, 0))
        r["angular_velocity"][i] = b.get("angular_velocity", (0, 0, 0))
        r["inv_mass"][i] = b.get("inv_mass", 0.0)
        r["inv_inertia"][i] = np.asarray(b.get("inv_inertia", np.zeros((3, 3))), np.float32).T.reshape(9)
        r["frictions"][i] = b["frictions"] if "frictions" in b else (b.get("friction", 0.0),) * 2
        o, t, _ = rigid_boundary_samples(b["tris"], dx)
        offs.append(o); tris.append(t); rid.append(np.full(len(o), i, np.int32))
    r["sample_offset"] = np.concatenate(offs) if offs else np.zeros((0, 3), np.float32)
    r["sample_tri"] = np.concatenate(tris) if tris else np.zeros((0, 9), np.float32)
    r["sample_rigid"] = np.concatenate(rid) if rid else np.zeros(0, np.int32)
    return r
