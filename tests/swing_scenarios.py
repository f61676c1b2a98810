"""Deterministic swing-leg / terrain scenarios for B robots (test helper).  Every robot stands still for a few ticks and then trots
over a sloped plane; per robot: gait_counter_speed, slope (both signs, steep enough for the +-0.5 clip), body height (with spans
below 0.1 m), and whether late swing feet meet the ground early (force > FOOT_FORCE_LOW past 1.5 counter_per_swing).

Scenario.tick() returns one control tick's inputs, batch-major [F, B]: what update_plan reads (movement_mode, lin_vel, lin_vel_d,
rot_z, rot, root_pos) plus foot_pos_abs and foot_force, together with update_plan's own outputs (gait_counter, plan_contacts,
foot_pos_target_rel) computed here with the reference's arithmetic (fmod of the counters, Raibert heuristic)."""
import numpy as np

CPG, CPS, CONTROL_DT = 240.0, 120.0, 0.0025
DEFAULT_FOOT = np.array([[0.17, 0.17, -0.17, -0.17], [0.15, -0.15, 0.15, -0.15], [-0.35, -0.35, -0.35, -0.35]])   # A1CtrlStates.h:45-47
KP_RESET, KD_RESET = np.tile([300.0, 400.0, 400.0], 4), np.tile([8.0, 8.0, 8.0], 4)      # A1CtrlStates.h:105-120
KP_ROS, KD_ROS = np.tile([150.0, 150.0, 200.0], 4), np.tile([0.0, 0.0, 0.0], 4)          # A1CtrlStates.h:247-253
SPEEDS = np.array([2.0, 3.0, 1.5, 4.0, 2.5, 2.0])


def _rz(yaw):
    c, s = np.cos(yaw), np.sin(yaw)
    z, o = np.zeros_like(yaw), np.ones_like(yaw)
    return np.stack([c, -s, z, s, c, z, z, z, o])            # [9, B] row-major


def _rot(yaw, pitch, roll):
    cy, sy, cp, sp, cr, sr = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    return np.stack([cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr,
                     sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr,
                     -sp, cp * sr, cp * cr])                   # Rz(yaw) Ry(pitch) Rx(roll), [9, B] row-major


TOL_FKIN = 1e-10     # relative to max(1, |f_kin|_inf), N
TOL_PITCH = 1e-7     # rad absolute: acos near 1 (flat ground) turns rounding of 1e-16 in the cosine into ~1e-8 in the angle


def check_tick(got, want, what=""):
    """got / want: (f_kin [12,B], contacts [B], foot_pos_recent_contact [12,B], terrain_pitch [B], ref row 1 [B]).  contacts exact,
    recent-contact points bit-identical (additions in a fixed order and one IEEE division), f_kin and the angles to the tolerances above.
    Returns the worst relative f_kin and absolute angle errors."""
    fk, con, rc, pitch, e1 = got
    fk0, con0, rc0, pitch0, e10 = want
    assert np.array_equal(con, con0), (what, np.nonzero(con != con0)[0][:8])
    assert np.array_equal(rc, rc0), (what, np.abs(rc - rc0).max())
    ef = float((np.abs(fk - fk0) / np.maximum(1.0, np.abs(fk0).max(axis=0))).max())
    ea = float(max(np.abs(pitch - pitch0).max(), np.abs(e1 - e10).max()))
    assert ef <= TOL_FKIN and ea <= TOL_PITCH, (what, ef, ea)
    return ef, ea


class Scenario:
    def __init__(self, B, seed, slopes=None, early=None, low=None, speeds=None):
        rng = np.random.default_rng(seed)
        self.rng, self.B, self.t = rng, B, 0
        self.n_stand = rng.integers(5, 40, B)
        self.speed = np.asarray(speeds, dtype=np.float64) if speeds is not None else SPEEDS[rng.integers(0, len(SPEEDS), B)]
        sl = rng.uniform(-1.0, 1.0, (2, B)) * np.array([[0.9], [0.3]])
        self.slope = np.asarray(slopes, dtype=np.float64).T if slopes is not None else sl            # [2, B]: dz/dx, dz/dy
        self.early = np.asarray(early, dtype=bool) if early is not None else rng.random(B) < 0.5
        lo = rng.random(B) < 0.3
        self.low = np.asarray(low, dtype=bool) if low is not None else lo                            # spans with root z <= 0.1
        self.yaw0, self.yaw_rate = rng.uniform(-np.pi, np.pi, B), rng.uniform(-0.5, 0.5, B) * CONTROL_DT
        self.vd = np.stack([rng.uniform(-0.2, 0.5, B), rng.uniform(-0.2, 0.2, B), np.zeros(B)])
        self.gc = np.zeros((4, B))

    def tick(self):
        B, rng, t = self.B, self.rng, self.t
        self.t += 1
        mode = (t >= self.n_stand).astype(np.uint32)
        # update_plan's counters (A1RobotControl.cpp:150-165)
        walk = mode != 0
        gc = np.where(walk[None, :], np.fmod(self.gc + self.speed[None, :], CPG), np.array([[0.0], [120.0], [120.0], [0.0]]))
        self.gc = gc
        plan = ((gc <= CPS) * (1 << np.arange(4))[:, None]).sum(axis=0).astype(np.uint32)
        yaw = self.yaw0 + self.yaw_rate * t
        pitch, roll = 0.03 * np.sin(0.01 * t + self.yaw0), 0.02 * np.cos(0.013 * t + self.yaw0)
        rz, rot = _rz(yaw), _rot(yaw, pitch, roll)
        z = 0.3 + 0.01 * np.sin(0.05 * t + self.yaw0)
        z = np.where(self.low & (t % 120 >= 90), 0.08, z)
        root_pos = np.stack([0.001 * t * np.cos(yaw), 0.001 * t * np.sin(yaw), z])
        lin_vel = self.vd + 0.05 * rng.standard_normal((3, B))
        # Raibert foothold target in the body frame (:168-197)
        vrel = np.stack([rz[0] * lin_vel[0] + rz[3] * lin_vel[1] + rz[6] * lin_vel[2], rz[1] * lin_vel[0] + rz[4] * lin_vel[1] + rz[7] * lin_vel[2]])
        k = np.sqrt(abs(DEFAULT_FOOT[2, 0]) / 9.8)
        trel = np.zeros((12, B))
        for i in range(4):
            for a in range(2):
                d = k * (vrel[a] - self.vd[a]) + ((CPS / self.speed) * CONTROL_DT) / 2.0 * self.vd[a]
                trel[3 * i + a] = DEFAULT_FOOT[a, i] + np.clip(d, -0.1, 0.1)
            trel[3 * i + 2] = DEFAULT_FOOT[2, i]
        # feet: nominal stance under the body, on the plane z = slope . (x, y) below the hips; swing feet lifted
        fabs = np.zeros((12, B))
        force = np.zeros((4, B))
        for i in range(4):
            rel = DEFAULT_FOOT[:, i][:, None] + 0.01 * rng.standard_normal((3, B))
            ab = np.stack([rot[3 * a] * rel[0] + rot[3 * a + 1] * rel[1] + rot[3 * a + 2] * rel[2] for a in range(3)])
            ab[2] += self.slope[0] * ab[0] + self.slope[1] * ab[1]
            swing = gc[i] > CPS
            ab[2] += np.where(swing, 0.08 * np.sin(np.pi * np.clip(gc[i] - CPS, 0.0, CPS) / CPS), 0.0)
            fabs[3 * i:3 * i + 3] = ab
            late = swing & (gc[i] > 1.5 * CPS + 10.0) & self.early
            force[i] = np.where(swing, np.where(late, 45.0 + 10.0 * rng.random(B), 5.0 * rng.random(B)), 40.0 + 40.0 * rng.random(B))
        return dict(movement_mode=mode, lin_vel=lin_vel, lin_vel_d=self.vd.copy(), root_pos=root_pos, rot_z=rz, rot=rot, foot_pos_abs=fabs,
                    foot_force=force, gait_counter=gc.copy(), plan_contacts=plan, foot_pos_target_rel=trel)
