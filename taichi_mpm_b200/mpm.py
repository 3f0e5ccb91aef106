"""Host-side mirror of the reference's solver surface for the accelerated path.

Same verbs and keyword names as the reference's Python driver (`tc.dynamics.MPM`, mirrored in the
reference tree by scripts/async/async_mpm.py:17-300) and the `MPM<3>` plugin behind it
(src/mpm.cpp:27-75 initialize, 77-270 add_particles, 428-450 step, 452-575 substep):

    mpm = MPM(res=(256,256,256), base_delta_t=2e-5, gravity=(0,-10,0))
    ls = mpm.create_levelset(); ls.add_plane((0,1,0), -0.1); ls.set_friction(0.4); mpm.set_levelset(ls)
    mpm.add_particles(type='sand', benchmark_block=(lo, hi), density=400)
    mpm.step(frame_dt)            # runs substeps on the GPU engine through the C-ABI
    mpm.visualize()               # frame_directory/0001.bgeo, the reference's bytes (src/visualize.cpp:16-100)
    mpm.general_action(action='save', file_name='snap.npz')   # and action='load'
    p = mpm.get_particles()       # the same data as numpy arrays

Everything numerical happens in libmpmb.so (capi.Engine); this file is glue: kwargs -> MpmbConfig,
registered particle type names -> material groups, level-set planes -> the engine's dense SDF.
Only the fast path of the reference is mirrored (optimized=True, static level set); rigid bodies are advanced on the device.

MPM2D(res=(r0, r1), ...) is the same surface on the MPM<2> engine (capi.Engine2D; MPM itself keeps refusing a 2-D res): positions and velocities are 2-vectors, gravity defaults to
(0, -10), add_particles(benchmark_block=...) seeds 4 particles per cell, apic_damping / rpic_damping are honoured, and level
sets take planes, circles (add_sphere) and rectangles (add_cuboid) with 2-vectors.  Rigid bodies, AsyncMPM, z-slabs, dynamic
level sets and delete_particles_inside_level_set are MPM<3> only and raise ValueError.  Particles added between steps take a
host round trip; their ids are kept.
"""
import os

import numpy as np

from . import bgeo, capi, rigid as rigid_mod, scenes

# MPMParticle::get_debug_info().y per registered type (src/particles.cpp:288-290,347-349,422-424,
# 496-498,669-671,156-158,754-756,838-840); water also reports (j, 5, sticky); elastic reports its Young's modulus in .x,
# which this mirror does not carry per particle (0 is written)
_DEBUG_CODE = {scenes.MAT_SNOW: 2.0, scenes.MAT_LINEAR: 3.0, scenes.MAT_JELLY: 4.0, scenes.MAT_WATER: 5.0, scenes.MAT_SAND: 6.0,
               scenes.MAT_VISCO: 1.0, scenes.MAT_VON_MISES: 7.0, scenes.MAT_ELASTIC: 8.0}


def frame_attributes(p, group_kinds, verbose=False):
    """Point attributes of one frame dump from a `download()` dict sorted by id — pure host code, so
    the file layer is testable without a GPU.  group_kinds[g] = material kind of group g."""
    debug = None
    if verbose:
        kinds = np.asarray(group_kinds, np.int64)[np.asarray(p["group"], np.int64)] if len(p["group"]) else np.zeros(0, np.int64)
        debug = np.zeros((len(kinds), 3), np.float32)
        for k, code in _DEBUG_CODE.items():
            debug[kinds == k, 1] = code
        water = kinds == scenes.MAT_WATER
        debug[water, 0] = np.asarray(p["ps"], np.float32)[water]
    return bgeo.reference_attributes(p, verbose=verbose, debug_code=debug)


def _pad3(a):
    """[n, 2] -> [n, 3] with a zero third column."""
    a = np.asarray(a, np.float32)
    return np.concatenate([a, np.zeros((len(a), 1), np.float32)], 1)


def _pad3x3(b):
    """[n, 4] column-major 2x2 -> [n, 9] column-major 3x3, zero third row and column."""
    b = np.asarray(b, np.float32).reshape(-1, 2, 2)
    out = np.zeros((len(b), 3, 3), np.float32)
    out[:, :2, :2] = b
    return out.reshape(-1, 9)


class LevelSet:
    """Static level set made of half-spaces (tc.core LevelSet3D.add_plane / set_friction as used by
    scripts/mls-cpic/sand_sweep.py:13-19).  World units: phi(x) = n.x + d, inside is phi>0."""

    def __init__(self, res, delta_x):
        self.res = tuple(res)
        self.delta_x = delta_x
        self.planes = []
        self.shapes = []      # (kind, inside_out, params) in WORLD units, in the order they were added
        self.friction = 0.0
        self.dense = None

    def _vec(self, v):
        """A point or direction of this level set's dimension, as the 3-vector the engine takes (z = 0 in 2-D)."""
        v = [float(c) for c in v]
        if len(v) != len(self.res):
            raise ValueError("a %d-D level set takes %d-vectors, got %r" % (len(self.res), len(self.res), v))
        return v + [0.0] * (3 - len(v))

    def add_plane(self, normal, d):
        n = np.asarray(self._vec(normal), np.float64)
        n = n / np.linalg.norm(n)
        self.planes.append((n[0], n[1], n[2], float(d)))

    def add_sphere(self, center, radius, inside_out=False):
        """tc LevelSet3D.add_sphere (scripts/mls-cpic/sand_stir.py:9); a circle in 2-D."""
        self.shapes.append((capi.SHAPE_SPHERE, bool(inside_out), self._vec(center) + [float(radius)]))

    def add_cuboid(self, lower, upper, inside_out=False):
        """tc LevelSet3D.add_cuboid (scripts/async/sand.py:35); a rectangle in 2-D."""
        self.shapes.append((capi.SHAPE_CUBOID, bool(inside_out), self._vec(lower) + self._vec(upper)))

    def set_friction(self, f):
        self.friction = float(f)

    def shapes_grid_units(self):
        """Planes and solids as the engine takes them: lengths divided by dx (plane normals are unit)."""
        out = [(capi.SHAPE_PLANE, False, [p[0], p[1], p[2], p[3] / self.delta_x]) for p in self.planes]
        out += [(k, io, [v / self.delta_x for v in prm]) for k, io, prm in self.shapes]
        return out

    def set_dense(self, sdf4):
        """Arbitrary static level set sampled at the nodes: [nx][ny][nz][4] = (n, phi in grid units)."""
        self.dense = np.ascontiguousarray(sdf4, np.float32)

    def planes_grid_units(self):
        # phi_grid(X) = phi(x)/dx with X = x/dx  ->  n.X + d/dx
        return np.array([[p[0], p[1], p[2], p[3] / self.delta_x] for p in self.planes], np.float32)

    def node_phi(self):
        """phi at the nodes, grid units (what the engine's level set holds)."""
        if self.dense is not None:
            return np.asarray(self.dense[..., 3], np.float32)
        sh = self.shapes_grid_units()
        if not sh:
            return np.full(tuple(r + 1 for r in self.res), 1e30, np.float32)
        return (scenes.shapes_sdf2d if len(self.res) == 2 else scenes.shapes_sdf)(self.res, sh)[..., 3]

    def sample(self, X):
        """phi at positions X (grid units), trilinear in the node values — LevelSet::sample as
        delete_particles_inside_level_set uses it (src/mpm.cpp:960-961; the interpolation itself is core code: assumed)."""
        phi = self.node_phi()
        X = np.asarray(X, np.float64)
        hi = np.asarray(phi.shape) - 1
        Xc = np.clip(X, 0, hi - 1e-9)
        i0 = np.floor(Xc).astype(np.int64)
        f = Xc - i0
        out = np.zeros(len(X))
        for a in (0, 1):
            for b in (0, 1):
                for c in (0, 1):
                    w = (f[:, 0] if a else 1 - f[:, 0]) * (f[:, 1] if b else 1 - f[:, 1]) * (f[:, 2] if c else 1 - f[:, 2])
                    out += w * np.minimum(phi[i0[:, 0] + a, i0[:, 1] + b, i0[:, 2] + c], np.float32(1e20))
        return out


class MPM:
    """Mirror of `tc.dynamics.MPM(**kwargs)` for 3D scenes (MPM<3>) on the accelerated path; MPM2D is the same surface for 2D
    scenes (MPM<2>)."""

    DIM = 3

    PARTICLE_TYPES = capi.MATERIAL_BY_NAME  # registered names, src/particles.cpp:845-856

    def __init__(self, **kwargs):
        res = kwargs["res"]
        if len(res) != self.DIM:
            raise ValueError("%s takes a %d-D res; %s" % (type(self).__name__, self.DIM, "2-D scenes run with MPM2D(res=(r0, r1), ...)"
                                                                  if len(res) == 2 else "3-D scenes run with MPM(res=(r0, r1, r2), ...)"))
        self.res = tuple(int(r) for r in res)
        self.dim = len(self.res)
        self.delta_x = float(kwargs.get("delta_x", 1.0 / self.res[0]))          # async_mpm.py:40-41
        # the reference's clocks are `real` = float (src/mpm.h:100, src/mpm.cpp:42-43,428-450,573): carried as float32 so
        # that a frame runs exactly the reference's number of substeps
        self.base_delta_t = float(np.float32(np.float32(kwargs.get("base_delta_t", 1e-4)) * np.float32(kwargs.get("dt_multiplier", 1.0))))
        g = kwargs.get("gravity", (0.0, -10.0, 0.0)[: self.dim])               # mpm.cpp:38: Vector::axis(1) * -10
        if np.isscalar(g):
            g = (0.0, float(g), 0.0)[: self.dim]
        self.gravity = tuple(float(x) for x in g)
        if len(self.gravity) != self.dim:
            raise ValueError("gravity must have %d components" % self.dim)
        self.frame_dt = float(kwargs.get("frame_dt", 0.01))
        self.particle_gravity = bool(kwargs.get("particle_gravity", True))      # mpm.cpp:47
        self.clean_boundary = bool(kwargs.get("clean_boundary", True))          # mpm.cpp:563
        if not kwargs.get("optimized", True):
            raise ValueError("optimized=False (the scalar transfers) is not accelerated")
        # MPM<2>'s resample damps apic_b with apic_damping / rpic_damping (src/mpm.h:465-469); MPM<3>'s optimized resample
        # does not damp the matrix (it passes a block index), and affine_damping is not read by either transfer
        for key in (("apic_damping", "rpic_damping", "affine_damping") if self.dim == 3 else ("affine_damping",)):
            if float(kwargs.get(key, 0.0)) != 0.0:
                raise ValueError("%s != 0 is outside the accelerated fast path" % key)
        self.penalty = float(kwargs.get("penalty", 0.0))                        # mpm.cpp:35: rigid-coupled scenes only
        self.pushing_force = float(kwargs.get("pushing_force", 20000.0))        # mpm.cpp:40
        self.rigid_body_levelset_collision = bool(kwargs.get("rigid_body_levelset_collision", False))   # mpm.cpp:535-538
        self.rigids = []          # HostRigidBody per add_particles(type='rigid'); engine body id = index + 1 (rigids[0] of the
        self._rigid_dirty = False  # reference is the background body, mpm.cpp:72-74)
        self._rigid_seen = None   # body states at the last read-back (a difference is a user edit, pushed before the next step)
        if self.dim == 2:
            self.engine = capi.Engine2D(self.res, self.delta_x, self.base_delta_t, self.gravity, self.particle_gravity, self.clean_boundary,
                                        device=int(kwargs.get("device", 0)), capacity=int(kwargs.get("capacity", 0)),
                                        apic_damping=float(kwargs.get("apic_damping", 0.0)), rpic_damping=float(kwargs.get("rpic_damping", 0.0)))
        else:
            self.engine = capi.Engine(self.res, self.delta_x, self.base_delta_t, self.gravity, self.particle_gravity,
                                      self.clean_boundary, device=int(kwargs.get("device", 0)), capacity=int(kwargs.get("capacity", 0)))
        self.current_t = np.float32(0.0)
        self.request_t = np.float32(0.0)
        self._update_counter = 0   # "Times of particle updating" (mpm.cpp:436,449): summed on the device, read lazily
        self._update_seen = 0
        self.substep_counter = 0
        self._groups = []         # (kind, params) per material group
        self.frame_directory = kwargs.get("frame_directory")                    # async_mpm.py:49, mpm.h:335
        self.verbose_bgeo = bool(kwargs.get("verbose_bgeo", False))             # visualize.cpp:22
        self.frame_count = 0                                                    # mpm.h:105
        self._host = None         # pending host-side particle set (dict of arrays)
        self._dirty = False
        self._n_uploaded = 0
        self._id_base = 0         # the engine's id base (set by 'load')
        self._id_span = 0         # ids handed out since the last upload: [id_base, id_base + _id_span)
        # 2-D: the engine numbers an upload 0..n-1, so the ids a user sees are kept here: _ids[engine id], increasing
        self._ids = np.zeros(0, np.int64)
        self._host_ids = None     # ids of the pending host set
        self._next_id = 0

    # ---- level set
    def create_levelset(self):
        return LevelSet(self.res, self.delta_x)

    def set_levelset(self, levelset, is_dynamic_levelset=False):
        if is_dynamic_levelset:
            raise ValueError("dynamic level sets are outside the accelerated fast path")
        self._levelset = levelset
        if levelset.dense is not None:
            self.engine.set_sdf(levelset.dense, levelset.friction)
        elif levelset.shapes:
            self.engine.set_levelset_shapes(levelset.shapes_grid_units(), levelset.friction)
        elif levelset.planes:
            self.engine.set_planes(levelset.planes_grid_units(), levelset.friction)
        else:
            self.engine.set_sdf(None, 0.0)

    # ---- particles
    def _group_of(self, kind, params):
        for g, (k, p) in enumerate(self._groups):
            if k == kind and np.array_equal(p, params):
                return g
        if len(self._groups) >= capi.MPMB_MAX_GROUPS:
            raise ValueError("more than %d distinct materials" % capi.MPMB_MAX_GROUPS)
        self._groups.append((kind, params))
        self.engine.set_material(len(self._groups) - 1, kind, params)
        return len(self._groups) - 1

    def add_particles(self, **kwargs):
        """type=<registered name>, plus either positions=[n,3] (world units) or
        benchmark_block=(lo_cell, hi_cell) for the reference's 8-per-cell lattice
        (src/mpm.cpp:164-180).  density (400), initial_velocity, and the material keys of the
        reference type (E, nu, youngs_modulus, friction_angle, ...) are honoured."""
        name = kwargs["type"]
        if name == "rigid":
            if self.dim == 2:
                raise ValueError("2-D rigid bodies (segment meshes, CPIC) are not accelerated")
            return self.add_rigid_particle(**kwargs)
        if name not in self.PARTICLE_TYPES:
            raise ValueError("unknown particle type %r" % name)
        kind = self.PARTICLE_TYPES[name]
        params = scenes.material_params(kind, **kwargs)
        group = self._group_of(kind, params)
        density = float(kwargs.get("density", 400.0))                           # mpm.cpp:135
        if "benchmark_block" in kwargs:
            lo, hi = kwargs["benchmark_block"]
            if self.dim == 2:   # this project's 2-D lattice: the reference's benchmark branch is 3-D only (mpm.cpp:152)
                x, mass, vol = scenes.lattice_block2d(self.res, lo, hi, density, kwargs.get("jitter", 0.0), dx=self.delta_x,
                                                      maximum=float(kwargs.get("maximum", 4.0)))
            else:
                x, mass, vol = scenes.lattice_block(self.res[0], lo, hi, density, kwargs.get("jitter", 0.0), dx=self.delta_x)
        else:
            x = np.ascontiguousarray(kwargs["positions"], np.float32).reshape(-1, self.dim)
            ppc = float(kwargs.get("maximum", 8.0 if self.dim == 3 else 4.0))
            vol = np.full(len(x), self.delta_x ** self.dim / ppc, np.float32)   # mpm.cpp:134
            mass = (vol * density).astype(np.float32)
        # near_boundary particles are ignored (mpm.cpp:129-132)
        X = x / np.float32(self.delta_x)
        keep = (X.min(1) >= 7.0) & ((X - np.asarray(self.res, np.float32)).max(1) <= -7.0)
        x, mass, vol = x[keep], mass[keep], vol[keep]
        if self.dim == 2:
            st = scenes.make_state2d(x, mass, vol, kind, group, kwargs.get("initial_velocity", (0.0, 0.0)))
        else:
            st = scenes.make_state(x, mass, vol, kind, group, kwargs.get("initial_velocity", (0.0, 0.0, 0.0)))
        if kind == scenes.MAT_VISCO and "tau" in kwargs:                         # visco_tau, src/particles.cpp:62
            st["ps"][:] = np.float32(kwargs["tau"])
        if self.dim == 2:   # a host round trip that keeps every id: the new particles are numbered after all ids so far
            cur = self._pull_host()
            new_ids = np.arange(self._next_id, self._next_id + len(x), dtype=np.int64)
            self._next_id += len(x)
            st.pop("alive")
            self._host = st if cur is None else {k: np.concatenate([cur[k], st[k]]) for k in st}
            self._host_ids = new_ids if cur is None else np.concatenate([self._host_ids, new_ids])
            self._dirty = True
            return ""
        if self._host is None and self._n_uploaded > 0 and hasattr(self.engine, "append"):
            # particles are resident and no host copy is pending: append on the device (mpm.cpp:147), the resident
            # particles keep their ids and state, the new ones are numbered after every id handed out so far
            first = self.engine.append(st["x"], st["v"], st["mass"], st["vol"], st["F"], st["b"], st["ps"], st["group"])
            self._id_span = max(self._id_span, int(first) - self._id_base + len(st["x"]))
            return ""
        cur = self._pull_host()
        if cur is None:
            self._host = st
        else:
            self._host = {k: np.concatenate([cur[k], st[k]]) for k in st if k != "alive"}
        self._dirty = True
        return ""

    def add_rigid_particle(self, **kwargs):
        """MPM<3>::add_rigid_particle (src/mpm_rigid_body.cpp:57-250): the keys of create_rigid_body — initial_position |
        scripted_position, initial_rotation (Euler degrees) | scripted_rotation, initial_velocity, initial_angular_velocity,
        friction | friction0 + friction1, density (40 codimensional / 400), codimensional (required, as in the reference), scale,
        recenter, rotation_axis, linear_damping, angular_damping — with the mesh given as `mesh_fn` (.obj) or `tris` [m,3,3].
        Scripted functions are Python callables t -> 3 numbers (the reference wraps them with tc.function13).  Returns the
        body's id as the reference does (a string)."""
        if "scripted" in kwargs or "position" in kwargs or "rotation" in kwargs:                # check_scripting_parameters, :16-22
            raise ValueError("use initial_position / scripted_position and initial_rotation / scripted_rotation")
        if ("scripted_position" in kwargs) == ("initial_position" in kwargs):
            raise ValueError("specify one (and only one) of 'scripted_position' and 'initial_position'")
        if "friction" in kwargs and ("friction0" in kwargs or "friction1" in kwargs):
            raise ValueError("friction and friction0/friction1 cannot coexist")
        if ("friction0" in kwargs) != ("friction1" in kwargs):
            raise ValueError("friction0 and friction1 must be specified simultaneously")
        if len(self.rigids) >= 11:
            raise ValueError("at most 11 rigid bodies (GridState::max_num_rigid_bodies)")
        codim = bool(kwargs["codimensional"])
        tris = rigid_mod.load_obj(kwargs["mesh_fn"]) if "mesh_fn" in kwargs else np.asarray(kwargs["tris"], np.float64).reshape(-1, 3, 3)
        tris = tris * np.asarray(kwargs.get("scale", (1.0, 1.0, 1.0)), np.float64)              # :183-189
        fr = (kwargs["friction0"], kwargs["friction1"]) if "friction0" in kwargs else (kwargs.get("friction", 0.0),) * 2
        body = rigid_mod.HostRigidBody(
            tris, density=float(kwargs.get("density", 40.0 if codim else 400.0)), codimensional=codim,
            position=kwargs.get("initial_position", (0, 0, 0)), euler_deg=kwargs.get("initial_rotation", (0, 0, 0)),
            velocity=kwargs.get("initial_velocity", (0, 0, 0)), angular_velocity=kwargs.get("initial_angular_velocity", (0, 0, 0)), frictions=fr,
            scripted_position=kwargs.get("scripted_position"), scripted_rotation=kwargs.get("scripted_rotation"),
            recenter=bool(kwargs.get("recenter", True)), rotation_axis=kwargs.get("rotation_axis", (0, 0, 0)),
            linear_damping=float(kwargs.get("linear_damping", 0.0)), angular_damping=float(kwargs.get("angular_damping", 0.0)), t0=float(self.current_t),
            restitution=float(kwargs.get("restitution", 0.0)))
        self.rigids.append(body)
        self._rigid_dirty = True
        return str(len(self.rigids))

    def _rigid_records(self):
        return rigid_mod.engine_records(self.rigids, self.delta_x, self.penalty, self.pushing_force)

    def _rigid_substeps(self, n):
        """n substeps of the reference's substep() with bodies (src/mpm.cpp:452-575) in one engine call: the transfers at the
        current pose, then on the device the level-set collision (if enabled) and advect_rigid_bodies.  Scripted parts follow a
        table evaluated here in fp64 at the float32 clock sequence of step().  The bodies are uploaded when the set changed and
        their state only after a user edit (the device keeps an fp64 master state); one read-back per call puts the advanced
        state into the HostRigidBody objects.  The level-set collision follows the transfers of a substep, where in the reference
        it sits between the grid normalisation and the boundary condition (src/mpm.cpp:535-538).  Returns the clock after."""
        h = np.float32(self.base_delta_t)
        t = np.float32(self.current_t)
        if self._rigid_dirty:
            self.engine.set_rigid(self._rigid_records())            # boundary samples of every body + coupling constants + state
            self.engine.set_rigid_motion([{}] + [b.motion_record() for b in self.rigids], self.rigid_body_levelset_collision)
            self._rigid_dirty = False
        elif self._rigid_edited():
            self.engine.set_rigid_state(rigid_mod.state_records(self.rigids))
        clocks = []
        for _ in range(n):
            clocks.append(float(t) + float(h))                      # HostRigidBody.advect(t, h) evaluates its functions at t + h
            t = np.float32(t + h)
        scripted = [b.pos_func is not None or b.rot_func is not None for b in self.rigids]
        table = None
        if any(scripted):
            table = np.zeros((n, len(self.rigids) + 1, capi.RIGID_SCRIPT_STRIDE))
            for k, b in enumerate(self.rigids):
                if scripted[k]:
                    table[:, k + 1] = b.script_poses(clocks, float(h))
            self.engine.set_rigid_script(table)
        self.engine.substep(n)
        rs = self.engine.get_rigid_state(len(self.rigids) + 1)
        for k, b in enumerate(self.rigids):
            b.velocity = rs["velocity"][k + 1].astype(np.float64)
            b.angular_velocity = rs["angular_velocity"][k + 1].astype(np.float64)
            # scripted parts keep the table's fp64 pose (the device holds the same): the next table differences against it
            b.position = table[-1, k + 1, 0:3].copy() if b.pos_func else rs["position"][k + 1].astype(np.float64)
            b.rotation = table[-1, k + 1, 3:12].reshape(3, 3).T.copy() if b.rot_func else rs["rotation"][k + 1].astype(np.float64)
        self._rigid_seen = [(b.position.copy(), b.rotation.copy(), b.velocity.copy(), b.angular_velocity.copy()) for b in self.rigids]
        return t

    def _rigid_edited(self):
        """Whether the user changed a body's pose or velocities since the last read-back."""
        seen = self._rigid_seen
        if seen is None or len(seen) != len(self.rigids):
            return True
        return any(not (np.array_equal(b.position, p) and np.array_equal(b.rotation, r) and np.array_equal(b.velocity, v) and
                        np.array_equal(b.angular_velocity, w)) for b, (p, r, v, w) in zip(self.rigids, seen))

    def _pull_host(self):
        """Host copy of the resident particles (download -> mutate -> upload contract, SURVEY §8b)."""
        if self._host is not None:
            return self._host
        if self._n_uploaded == 0:
            return None
        d = self.engine.download()
        self._host = dict(x=d["x"], v=d["v"], F=d["F"], b=d["b"], mass=d["mass"], vol=d["vol"], ps=d["ps"], group=d["group"])
        if self.dim == 2:
            self._host_ids = self._ids[d["id"].astype(np.int64)]
        return self._host

    def _push(self):
        if self._dirty and self._host is not None:
            h = self._host
            self.engine.upload(h["x"], h["v"], h["mass"], h["vol"], h["F"], h["b"], h["ps"], h["group"])
            if self.dim == 2:
                self._ids = self._host_ids
                self._host_ids = None
            self._n_uploaded = len(h["x"])
            self._id_span = len(h["x"])     # an upload numbers its particles id_base + 0..n-1
            self._dirty = False
            self._host = None

    # ---- time stepping
    def substep(self):
        self._push()
        if self.rigids:
            self.current_t = self._rigid_substeps(1)
        else:
            self.engine.substep(1)
            self.current_t = np.float32(self.current_t + np.float32(self.base_delta_t))   # src/mpm.cpp:573, float
        self.substep_counter += 1

    def step(self, dt):
        """MPM<dim>::step (src/mpm.cpp:428-450): dt<0 runs exactly one substep."""
        self._push()
        if dt < 0:
            self.substep()
            self.request_t = self.current_t
            return
        # float32 compare-and-accumulate, as the reference's `real` members do (29996 substeps for 60 frames of
        # 0.01 at base_delta_t = 2e-5, not 30000: pinned against MPM<3>::step itself, tests/test_mirror_host.py)
        h = np.float32(self.base_delta_t)
        self.request_t = np.float32(self.request_t + np.float32(dt))
        n = 0
        t = np.float32(self.current_t)
        while np.float32(t + h) < self.request_t:
            t = np.float32(t + h)
            n += 1
        if n:
            # "Times of particle updating" (src/mpm.cpp:436,449) = particles.size() per substep: the engine sums the
            # particles every ordering bins (exact when particles are deleted inside the frame); see update_counter
            if self.rigids:
                self._rigid_substeps(n)
            else:
                self.engine.substep(n)
            self.current_t = t
            self.substep_counter += n
        self._host = None

    @property
    def update_counter(self):
        """MPM::update_counter (src/mpm.cpp:436,449), read from the device counter on demand (no sync inside step())."""
        seen = self.engine.update_count()
        self._update_counter += seen - self._update_seen
        self._update_seen = seen
        return self._update_counter

    @update_counter.setter
    def update_counter(self, value):
        self._update_seen = self.engine.update_count()
        self._update_counter = int(value)

    def get_current_time(self):
        return self.current_t

    def get_particles(self):
        """Live particles as numpy arrays (the data visualize() writes: src/visualize.cpp:16-100)."""
        self._push()
        p = self.engine.download()
        if self.dim == 2:
            p["id"] = self._ids[p["id"].astype(np.int64)].astype(np.uint32)
        return p

    def num_particles(self):
        self._push()
        return self.engine.num_particles()

    def get_debug_information(self):
        """MPM<dim>::get_debug_information (src/mpm.cpp:635-639): the reference returns an empty string."""
        return ""

    def test(self):
        """MPM<dim>::test (src/mpm.cpp:577-580)."""
        return True

    def get_name(self):
        return "mpm"                                                            # src/mpm.h:487, TC_IMPLEMENTATION(..., "mpm")

    # ---- frame output and snapshots (SURVEY §8f row 1)
    def visualize(self):
        """MPM<3>::visualize -> write_bgeo (src/visualize.cpp:156-159, src/mpm.h:333-343): the frame
        counter is incremented first, the file is `<frame_directory>/<count:04>.bgeo`, particles in
        id order with the attributes of write_partio.  Returns the file name."""
        if not self.frame_directory:
            raise ValueError("frame_directory was not given to MPM(...)")
        self.frame_count += 1
        os.makedirs(self.frame_directory, exist_ok=True)
        fn = os.path.join(self.frame_directory, "%04d.bgeo" % self.frame_count)
        if not self.verbose_bgeo and hasattr(self.engine, "download_bgeo_points"):
            # non-verbose dump: the point records are packed on the device in id order (48 B per particle cross the bus
            # instead of the full state, and no host pass over the particles)
            self._push()
            n, block = self.engine.download_bgeo_points(self._id_range())
            if self.dim == 2 and n:   # the index word carries the engine id: the kept ids are increasing in it, the order holds
                w = block.view(">u4").reshape(n, 12)
                w[:, 5] = self._ids[w[:, 5].astype(np.int64)]
            bgeo.write_bgeo_packed(fn, n, block)
            return fn
        p = self.get_particles()
        if self.dim == 2:   # write_partio leaves the third components 0 (src/visualize.cpp:62,78,90)
            p = dict(p, x=_pad3(p["x"]), v=_pad3(p["v"]), b=_pad3x3(p["b"]))
        bgeo.write_bgeo(fn, p["x"], frame_attributes(p, [k for k, _ in self._groups], self.verbose_bgeo))
        return fn

    def _id_range(self):
        # ids lie in [id_base, id_base + id span): the last upload plus every device append since
        return max(int(self._id_span), 1)

    def _refuse_2d(self, what):
        if self.dim == 2:
            raise ValueError("%s is MPM<3> only" % what)

    def general_action(self, **kwargs):
        """The actions of MPM<dim>::general_action (src/mpm.cpp:920-976) that concern the accelerated
        state: 'save' / 'load' of a snapshot (the reference serialises itself with the taichi core's
        binary format, which is not available here — this is a numpy .npz of the same state:
        particles, material groups, clocks and counters; level sets are re-attached by the scene
        script, as scripted rigid motion is in the reference, mpm.cpp:943-958)."""
        action = kwargs["action"]
        if action == "save":
            p = self.get_particles()
            kinds = np.array([k for k, _ in self._groups], np.int32)
            params = np.stack([q for _, q in self._groups]).astype(np.float32) if self._groups else np.zeros((0, scenes.N_MAT_PARAMS), np.float32)
            with open(kwargs["file_name"], "wb") as f:
                np.savez(f, format=np.array("mpmb-snapshot-1"), res=np.array(self.res), delta_x=self.delta_x, base_delta_t=self.base_delta_t,
                         gravity=np.array(self.gravity), current_t=self.current_t, request_t=self.request_t,
                         counters=np.array([self.update_counter, self.substep_counter, self.frame_count], np.int64),
                         mat_kind=kinds, mat_params=params, **{"p_" + k: v for k, v in p.items()})
            return ""
        if action == "load":
            with np.load(kwargs["file_name"]) as z:
                if str(z["format"]) != "mpmb-snapshot-1":
                    raise ValueError("not an mpmb snapshot")
                if tuple(int(r) for r in z["res"]) != self.res or abs(float(z["delta_x"]) - self.delta_x) > 0:
                    raise ValueError("snapshot grid %s does not match this solver %s" % (tuple(z["res"]), self.res))
                self._groups = []
                for g, (k, q) in enumerate(zip(z["mat_kind"], z["mat_params"])):
                    self._groups.append((int(k), np.asarray(q, np.float32)))
                    self.engine.set_material(g, int(k), self._groups[-1][1])
                self.current_t, self.request_t = np.float32(z["current_t"]), np.float32(z["request_t"])
                self.update_counter, self.substep_counter, self.frame_count = (int(c) for c in z["counters"])
                self._host = {k: np.ascontiguousarray(z["p_" + k]) for k in ("x", "v", "F", "b", "mass", "vol", "ps", "group")}
                ids = np.ascontiguousarray(z["p_id"])
            # ids are positions in the upload: keep the snapshot's ids by uploading in id order with the base id
            self._dirty = True
            self._push_with_ids(ids)
            return ""
        if action == "delete_particles_inside_level_set":                      # mpm.cpp:958-972
            self._refuse_2d("delete_particles_inside_level_set")
            ls = getattr(self, "_levelset", None)
            if ls is not None and self._host is None and self._n_uploaded > 0 and hasattr(self.engine, "delete_inside_levelset"):
                self.engine.delete_inside_levelset()     # on the device: the survivors keep their ids and state
                return ""
            p = self.get_particles()
            if ls is None or len(p["x"]) == 0:
                return ""
            keep = ~(ls.sample(p["x"].astype(np.float64) / self.delta_x) < 0)
            if keep.all():
                return ""
            self._host = {k: np.ascontiguousarray(p[k][keep]) for k in ("x", "v", "F", "b", "mass", "vol", "ps", "group")}
            self._dirty = True
            self._push_with_ids(p["id"][keep].astype(np.int64))
            return ""
        raise ValueError("Unknown action: %s" % action)  # TC_ERROR("Unknown action") mpm.cpp:974

    # ---- the verbs of the reference's Python driver around general_action and the frame loop (scripts/async/async_mpm.py:217-299)
    def action(self, **kwargs):
        return self.general_action(**kwargs)

    def save(self, fn):
        return self.general_action(action="save", file_name=fn)

    def load(self, fn):
        return self.general_action(action="load", file_name=fn)

    def delete_particles_inside_level_set(self):
        return self.general_action(action="delete_particles_inside_level_set")

    def simulate(self, num_frames=None, frame_update=None, update_frequency=1, snapshot_interval=0, snapshot_directory=None):
        """The driver's main cycle (scripts/async/async_mpm.py:236-248): per frame `update_frequency` calls of
        frame_update(t, dt) + step(dt), then visualize(); a snapshot every `snapshot_interval` frames."""
        n = int(num_frames if num_frames is not None else getattr(self, "num_frames", 1000))
        frame = 0
        while frame < n:
            for _ in range(update_frequency):
                if frame_update:
                    frame_update(float(self.get_current_time()), self.frame_dt / update_frequency)
                self.step(self.frame_dt / update_frequency)
            if self.frame_directory:
                self.visualize()
            frame += 1
            if snapshot_interval and snapshot_directory and frame % snapshot_interval == 0:
                os.makedirs(snapshot_directory, exist_ok=True)
                self.save(os.path.join(snapshot_directory, "%04d.npz" % frame))
        return frame

    def _push_with_ids(self, ids):
        """Upload after 'load': the engine numbers particles id_base + position, so a snapshot whose
        ids are not 0..n-1 (deleted particles) keeps them only if they are contiguous; otherwise the
        particles are renumbered 0..n-1 in id order (the reference reloads its own ids)."""
        h = self._host
        order = np.argsort(ids, kind="stable")
        h = {k: v[order] for k, v in h.items()}
        ids = ids[order]
        if self.dim == 2:   # the snapshot's ids are kept as they are
            self._host = h
            self._host_ids = ids.astype(np.int64)
            self._next_id = int(ids[-1]) + 1 if len(ids) else 0
            self._push()
            return
        base = int(ids[0]) if len(ids) and np.array_equal(ids - ids[0], np.arange(len(ids), dtype=ids.dtype)) else 0
        self.engine.set_id_base(base)
        self._id_base = base
        self._host = h
        self._push()


class MPM2D(MPM):
    """Mirror of `tc.dynamics.MPM(res=(r0, r1), ...)`: the same surface as MPM on the 2-D engine (capi.Engine2D, MPM<2>).
    Positions and velocities are 2-vectors, gravity defaults to (0, -10), add_particles(benchmark_block=...) seeds 4 particles per
    cell, apic_damping / rpic_damping are honoured and level sets take 2-vectors (planes, circles, rectangles)."""

    DIM = 2
