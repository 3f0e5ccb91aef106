"""Host-side rigid bodies for the mirror (`MPM.add_particles(type='rigid', ...)`).

In the reference the bodies are objects of its un-vendored core (`taichi/dynamics/rigid_body.h`): the solver only *uses* them
— `create_rigid_body` / `add_rigid_particle` / `advect_rigid_bodies` (src/mpm_rigid_body.cpp:57-135, 137-250, 252-284) call
`initialize_mass_and_inertia`, `advance`, `apply_impulse`, `enforce_angular_velocity_parallel_to`.  The device engine needs
poses and velocities per substep and returns velocities (include/mpmb.h, "rigid bodies"); this module is the small host class
in between.  What the core does inside those calls cannot be read here, so the definitions below are the textbook ones and are
ASSUMPTIONS (SURVEY appendix C): mass properties of a closed triangle mesh at uniform density (codimensional: a shell of
surface density `density`), explicit Euler for the position, the exponential map for the rotation, scripted bodies follow
their functions exactly with infinite mass / inertia (set_infinity_mass / set_infinity_inertia, src/mpm_rigid_body.cpp:198-203).
Rigid-rigid collisions (`rigidify`, src/mpm_rigid_body.cpp:286-330) and articulation are not restated."""
import math

import numpy as np

from . import scenes


def load_obj(path):
    """Triangles [m,3,3] of a Wavefront .obj (v / f records; polygons are fanned)."""
    verts, tris = [], []
    with open(path) as f:
        for line in f:
            t = line.split()
            if not t:
                continue
            if t[0] == "v":
                verts.append([float(x) for x in t[1:4]])
            elif t[0] == "f":
                idx = [int(w.split("/")[0]) for w in t[1:]]
                idx = [i - 1 if i > 0 else len(verts) + i for i in idx]
                for k in range(1, len(idx) - 1):
                    tris.append([verts[idx[0]], verts[idx[k]], verts[idx[k + 1]]])
    return np.asarray(tris, np.float64).reshape(-1, 3, 3)


def mass_properties(tris, density, codimensional):
    """(mass, centre of mass, inertia tensor about the centre of mass) of a closed mesh of uniform density, or of a thin shell of
    surface density `density` when codimensional."""
    t = np.asarray(tris, np.float64).reshape(-1, 3, 3)
    if codimensional:
        n = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
        area = 0.5 * np.linalg.norm(n, axis=1)
        m = density * area
        mass = m.sum()
        com = (m[:, None] * t.mean(1)).sum(0) / mass
        s = t.sum(1)
        cov = (m[:, None, None] / 12.0 * (np.einsum("ni,nj->nij", s, s) + np.einsum("nki,nkj->nij", t, t))).sum(0)   # int x x^T dm
    else:
        det = np.einsum("ni,ni->n", t[:, 0], np.cross(t[:, 1], t[:, 2]))
        vol = det.sum() / 6.0
        sign = 1.0 if vol >= 0 else -1.0
        mass = density * abs(vol)
        com = sign * density * (det[:, None] * t.sum(1)).sum(0) / 24.0 / mass
        canon = (np.ones((3, 3)) + np.eye(3)) / 120.0
        A = np.transpose(t, (0, 2, 1))                       # columns v0 v1 v2
        cov = sign * density * np.einsum("n,nij->ij", det, A @ canon @ np.transpose(A, (0, 2, 1)))
    cov = cov - mass * np.outer(com, com)                    # about the centre of mass
    inertia = np.trace(cov) * np.eye(3) - cov
    return float(mass), com, inertia


def _incremental_angular_velocity(new, old, dt):
    """Angular velocity that turns `old` into `new` over dt (axis-angle of the incremental rotation new old^T)."""
    d = new @ old.T
    ang = math.acos(max(-1.0, min(1.0, (np.trace(d) - 1) / 2)))
    axis = np.array([d[2, 1] - d[1, 2], d[0, 2] - d[2, 0], d[1, 0] - d[0, 1]])
    nrm = np.linalg.norm(axis)
    return (axis / nrm * ang / dt) if nrm > 1e-12 else np.zeros(3)


def _expmap(w):
    """Rotation matrix exp([w]x)."""
    a = float(np.linalg.norm(w))
    if a < 1e-12:
        return np.eye(3)
    k = np.asarray(w, np.float64) / a
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(a) * K + (1 - math.cos(a)) * (K @ K)


class HostRigidBody:
    """One body: mesh in the centroid frame, pose, velocities, mass properties, optional scripted motion."""

    def __init__(self, tris, density=400.0, codimensional=False, position=(0, 0, 0), euler_deg=(0, 0, 0), velocity=(0, 0, 0),
                 angular_velocity=(0, 0, 0), frictions=(0.0, 0.0), scripted_position=None, scripted_rotation=None, recenter=True,
                 rotation_axis=(0, 0, 0), linear_damping=0.0, angular_damping=0.0, t0=0.0, restitution=0.0):
        tris = np.asarray(tris, np.float64).reshape(-1, 3, 3)
        self.mass, com, self.inertia_body = mass_properties(tris, density, codimensional)     # src/mpm_rigid_body.cpp:190
        if not recenter:                                                                       # :191-195 (needs both scripts)
            if scripted_position is None or scripted_rotation is None:
                raise ValueError("recenter=False needs scripted_position and scripted_rotation")
            com = np.zeros(3)
        self.tris = tris - com                                                                 # :205-209
        self.pos_func, self.rot_func = scripted_position, scripted_rotation
        self.position = np.asarray(scripted_position(t0) if scripted_position else position, np.float64)
        self.rotation = scenes.euler_rotation(scripted_rotation(t0) if scripted_rotation else euler_deg)
        self.velocity = np.asarray(velocity, np.float64).copy()
        self.angular_velocity = np.asarray(angular_velocity, np.float64).copy()
        self.frictions = tuple(float(f) for f in frictions)
        self.inv_mass = 0.0 if scripted_position else 1.0 / self.mass                          # set_infinity_mass, :198-200
        self.inv_inertia_body = np.zeros((3, 3)) if scripted_rotation else np.linalg.inv(self.inertia_body)   # :201-203
        self.rotation_axis = np.asarray(rotation_axis, np.float64)
        self.linear_damping, self.angular_damping = float(linear_damping), float(angular_damping)
        self.restitution = float(restitution)                                                  # src/mpm_rigid_body.cpp:74

    def inv_inertia_world(self):
        return self.rotation @ self.inv_inertia_body @ self.rotation.T

    def _enforce_axis(self):                                                                   # enforce_angular_velocity_parallel_to
        if np.abs(self.rotation_axis).max() > 0.1:                                             # src/mpm_rigid_body.cpp:256-258
            a = self.rotation_axis / np.linalg.norm(self.rotation_axis)
            self.angular_velocity = a * float(a @ self.angular_velocity)

    # ---- what the solver calls of the core's RigidBody for collisions with the level set (standard rigid-body impulse algebra)
    def velocity_at(self, p):
        return self.velocity + np.cross(self.angular_velocity, np.asarray(p, np.float64) - self.position)

    def impulse_contribution(self, r0, n):
        """Velocity change along n at the contact point per unit impulse along n: 1/m + n . ((I^-1 (r0 x n)) x r0)."""
        return self.inv_mass + float(np.dot(n, np.cross(self.inv_inertia_world() @ np.cross(r0, n), r0)))

    def apply_impulse(self, j, p):
        self.velocity = self.velocity + self.inv_mass * np.asarray(j, np.float64)
        self.angular_velocity = self.angular_velocity + self.inv_inertia_world() @ np.cross(np.asarray(p, np.float64) - self.position, j)

    def levelset_collision(self, sample_world, phi, gradient):
        """MPM<dim>::rigid_body_levelset_collision for this body (src/mpm_rigid_body.cpp:346-381): every boundary sample inside
        the level set (phi < 0) takes a normal impulse that removes the approach velocity (restitution e) and a Coulomb friction
        impulse bounded by frictions[0] times it; the impulses are applied one sample after the other, as the reference loops."""
        if self.inv_mass == 0.0 and not self.inv_inertia_body.any():
            return 0
        hits = 0
        for p, ph, g in zip(sample_world, phi, gradient):
            if not ph < 0:
                continue
            r0 = p - self.position
            v0 = float(np.dot(g, self.velocity_at(p)))
            J = -((1.0 + self.restitution) * v0) / self.impulse_contribution(r0, g)
            if J < 0:
                continue
            self.apply_impulse(J * g, p)
            v10 = self.velocity_at(p)
            tao = v10 - g * float(np.dot(g, v10))
            if np.abs(tao).max() > 1e-7:
                tao = tao / np.linalg.norm(tao)
                j = -float(np.dot(v10, tao)) / self.impulse_contribution(r0, tao)
                j = min(max(j, -self.frictions[0] * J), self.frictions[0] * J)
                self.apply_impulse(j * tao, p)
            hits += 1
        return hits

    def motion_record(self):
        """This body's capi.Engine.set_rigid_motion record (device advection)."""
        return dict(mass=self.mass, inv_inertia_body=self.inv_inertia_body, rotation_axis=self.rotation_axis, linear_damping=self.linear_damping,
                    angular_damping=self.angular_damping, restitution=self.restitution, scripted_position=self.pos_func is not None,
                    scripted_rotation=self.rot_func is not None)

    def script_poses(self, clocks, dt):
        """Script entries [n, 18] (position, rotation column-major, velocity, angular velocity) of the substeps whose scripted
        functions are evaluated at `clocks` (each substep's start time + dt), in fp64 as advect computes them: the velocity is the
        finite difference of positions, the angular velocity that of the incremental rotation.  Free parts are 0; the body is not
        changed."""
        out = np.zeros((len(clocks), 18))
        pos, rot = self.position, self.rotation
        for k, tc in enumerate(clocks):
            if self.pos_func:
                new = np.asarray(self.pos_func(tc), np.float64)
                out[k, 12:15] = (new - pos) / dt
                out[k, 0:3] = pos = new
            if self.rot_func:
                new = scenes.euler_rotation(self.rot_func(tc))
                out[k, 15:18] = _incremental_angular_velocity(new, rot, dt)
                out[k, 3:12] = new.T.reshape(9)
                rot = new
        return out

    def advect(self, t, dt, gravity):
        """advect_rigid_bodies for this body (src/mpm_rigid_body.cpp:254-267): axis constraint, advance, gravity impulse."""
        self._enforce_axis()
        if self.pos_func:
            new = np.asarray(self.pos_func(t + dt), np.float64)
            self.velocity = (new - self.position) / dt
            self.position = new
        else:
            self.velocity *= math.exp(-self.linear_damping * dt)
            self.position = self.position + self.velocity * dt
        if self.rot_func:
            new = scenes.euler_rotation(self.rot_func(t + dt))
            self.angular_velocity = _incremental_angular_velocity(new, self.rotation, dt)
            self.rotation = new
        else:
            self.angular_velocity *= math.exp(-self.angular_damping * dt)
            self.rotation = _expmap(self.angular_velocity * dt) @ self.rotation
        self.velocity = self.velocity + np.asarray(gravity, np.float64) * (self.mass * dt) * self.inv_mass   # apply_impulse(g m dt, position)
        self._enforce_axis()


def state_records(bodies):
    """The state rows of engine_records without the boundary samples (capi.Engine.set_rigid_state; row 0 = the background body)."""
    nr = len(bodies) + 1
    r = dict(position=np.zeros((nr, 3), np.float32), rot=np.tile(np.eye(3, dtype=np.float32).reshape(9), (nr, 1)), velocity=np.zeros((nr, 3), np.float32),
             angular_velocity=np.zeros((nr, 3), np.float32), inv_mass=np.zeros(nr, np.float32), inv_inertia=np.zeros((nr, 9), np.float32),
             frictions=np.zeros((nr, 2), np.float32))
    for k, b in enumerate(bodies):
        i = k + 1
        r["position"][i], r["velocity"][i], r["angular_velocity"][i] = b.position, b.velocity, b.angular_velocity
        r["rot"][i] = np.asarray(b.rotation, np.float32).T.reshape(9)
        r["inv_mass"][i] = b.inv_mass
        r["inv_inertia"][i] = np.asarray(b.inv_inertia_world(), np.float32).T.reshape(9)
        r["frictions"][i] = b.frictions
    return r


def engine_records(bodies, dx, penalty, pushing_force):
    """The dict capi.Engine.set_rigid / set_rigid_state take (row 0 = the background body)."""
    desc = [dict(tris=b.tris, position=b.position, rotation=b.rotation, velocity=b.velocity, angular_velocity=b.angular_velocity, inv_mass=b.inv_mass,
                 inv_inertia=b.inv_inertia_world(), frictions=b.frictions) for b in bodies]
    return scenes.make_rigid(desc, dx, penalty=penalty, pushing_force=pushing_force)
