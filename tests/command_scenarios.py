"""Sensor and command sequences for the orientation / command stages (a1mpc_orientation_batch, a1mpc_command_batch), shared by the
fixture generator (tests/golden/make_command_golden.py), the emulator test and the GPU tests, and the tolerances they are held to.

Tolerances (device or emulator against the oracle):
  rot                 <= 4e-16 absolute (the products and sums of Eigen's toRotationMatrix, rounded alike: in practice bit-identical)
  euler               <= 1e-15 rad; yaw compared modulo 2 pi, so that +-pi on either side of the atan2 branch cut agree.  The atan2 /
                      asin arguments are rounded alike, so the only difference is the last bits of the device's atan2 / asin.
  rot_z               <= 4e-16 + |yaw - yaw_oracle|: the cos / sin of the yaw each side computed
  filters, ang_vel    <= 1e-15 relative (to max(1, |x|))
  discrete outputs    exact (movement_mode); kp_linear, ref, des <= 1e-15 relative (sums of the same terms in the same order)
"""
import numpy as np

VARIANTS = (0, 1, 2)                    # Gazebo, hardware, Isaac (A1MPC_VARIANT_*)
HEIGHT0 = {0: 0.3, 1: 0.12, 2: 0.32}   # GazeboA1ROS.h:130, HardwareA1ROS.h:107, IsaacA1ROS.h:80
HMIN, HMAX = 0.1, 0.32                  # A1Params.h:16-17
KP_LINEAR, KP_LOCK = (120.0, 120.0, 500.0), (120.0, 120.0)   # A1CtrlStates.h:270-301 defaults
DT = 0.0025
SPEEDS = np.array([0.0, 0.02, 0.049, 0.051, 0.08, 0.3, 0.6])  # |v_xy| both sides of 0.05, never within 1e-9 of it


def quat_from_euler(r, p, y):
    """unit (w, x, y, z) of R = Rz(y) Ry(p) Rx(r), arrays broadcast"""
    cr, sr, cp, sp, cy, sy = np.cos(r / 2), np.sin(r / 2), np.cos(p / 2), np.sin(p / 2), np.cos(y / 2), np.sin(y / 2)
    return np.stack([cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy])


def imu_sequence(B, T, seed, gimbal_share=0.1, gentle=False):
    """quat [T,4,B]: a yaw sweep across +-pi with roll / pitch wobble, scaled off unit length by up to 1e-3; a share of the robots
    pitched to +-pi/2 (|t2| >= 1 for the scaled-up ones).  gyro / acc [T,3,B] raw IMU readings.  gentle: a walking robot's rates
    (yaw sweeps from near +-pi at up to 8 rad/s, smaller wobble and sensor noise) for the closed-loop tick."""
    rng = np.random.default_rng(seed)
    t = np.arange(T)[:, None]
    if gentle:
        yaw0 = np.pi + rng.uniform(-0.3, 0.3, B)
        yaw_rate = rng.choice([-1.0, 1.0], B) * rng.uniform(0.01, 0.02, B)
    else:
        yaw0 = rng.uniform(-np.pi, np.pi, B)
        yaw_rate = rng.choice([-1.0, 1.0], B) * rng.uniform(0.02, 0.08, B)     # rad per tick: crosses +-pi within a few dozen ticks
    yaw = np.mod(yaw0 + yaw_rate * t + np.pi, 2 * np.pi) - np.pi
    wob, noise = (0.06, 0.005) if gentle else (0.15, 0.02)
    roll = wob * np.sin(0.3 * t + rng.uniform(0, 6, B)) + noise * rng.standard_normal((T, B))
    pitch = wob * np.sin(0.21 * t + rng.uniform(0, 6, B)) + noise * rng.standard_normal((T, B))
    g = rng.random(B) < gimbal_share
    pitch[:, g] = np.sign(rng.standard_normal(g.sum())) * (np.pi / 2 - np.abs(1e-9 * rng.standard_normal((T, g.sum()))))
    scale = 1.0 + rng.uniform(-1e-3, 1e-3, (T, B))
    quat = np.transpose(quat_from_euler(roll, pitch, yaw), (1, 0, 2)) * scale[:, None, :]
    gyro = (0.1 if gentle else 0.5) * rng.standard_normal((T, 3, B))
    acc = np.array([0.0, 0.0, 9.8])[None, :, None] + (0.2 if gentle else 0.8) * rng.standard_normal((T, 3, B))
    return np.ascontiguousarray(quat), np.ascontiguousarray(gyro), np.ascontiguousarray(acc)


def command_sequence(B, T, seed):
    """cmd [T,7,B]: velx, vely (|v_xy| from SPEEDS, held for stretches), velz (pushes the height into both clamps), roll / pitch / yaw
    rates, toggle requests (walking toggles in and out).  root_pos [T,3,B]: the previous estimate the lock copies."""
    rng = np.random.default_rng(seed)
    cmd = np.zeros((T, 7, B))
    seg = 10
    for s in range(0, T, seg):
        sp = rng.choice(SPEEDS, B)
        ang = rng.uniform(-np.pi, np.pi, B)
        cmd[s:s + seg, 0] = sp * np.cos(ang)
        cmd[s:s + seg, 1] = sp * np.sin(ang)
        cmd[s:s + seg, 2] = rng.choice([-4.0, -0.04, 0.0, 0.04, 4.0], B)
        cmd[s:s + seg, 3:6] = rng.uniform(-0.4, 0.4, (3, B))
    cmd[:, 6] = (rng.random((T, B)) < 0.12).astype(np.float64)
    cmd[0, 6] = 1.0                                                       # every robot starts walking on tick 0
    root_pos = np.ascontiguousarray(np.array([0.0, 0.0, 0.28])[None, :, None] + 0.05 * rng.standard_normal((T, 3, B)).cumsum(axis=0))
    return np.ascontiguousarray(cmd), root_pos


def pitch_overrides(B, T, seed):
    """[T,B] values compute_grf's terrain adaptation leaves in root_euler_d[1] before the next command tick (NaN: no adaptation)"""
    rng = np.random.default_rng(seed)
    ov = np.where(rng.random((T, B)) < 0.3, rng.uniform(-0.5, 0.5, (T, B)), np.nan)
    ov[0] = np.nan
    return ov


def _rel(a, b):
    return float((np.abs(a - b) / np.maximum(1.0, np.abs(b))).max()) if np.size(b) else 0.0


def check_orientation(o, o0, what):
    """o, o0: dicts rot, rot_z, euler, ang_vel, imu_acc, imu_ang_vel (device / emulator vs oracle).  Returns the worst errors."""
    er = float(np.abs(o["rot"] - o0["rot"]).max())
    assert er <= 4e-16, (what, "rot", er)
    d = o["euler"] - o0["euler"]
    d[2] = np.mod(d[2] + np.pi, 2 * np.pi) - np.pi
    ee = float(np.abs(d).max())
    assert ee <= 1e-15, (what, "euler", ee)
    ez = float((np.abs(o["rot_z"] - o0["rot_z"]) - (4e-16 + np.abs(d[2]))[None, :]).max())
    assert ez <= 0.0, (what, "rot_z", ez)
    ef = max(_rel(o["imu_ang_vel"], o0["imu_ang_vel"]), _rel(o["imu_acc"], o0["imu_acc"]) if o0.get("imu_acc") is not None else 0.0)
    ea = _rel(o["ang_vel"], o0["ang_vel"])
    assert ef <= 1e-15 and ea <= 1e-15, (what, "filters / ang_vel", ef, ea)
    return max(er, ee, ef, ea)


def check_command(got, want, what):
    """got, want: (movement_mode [B], kp_linear [3,B], ref [9,B], des [12,B])"""
    assert np.array_equal(got[0], want[0]), (what, "movement_mode")
    e = max(_rel(g, w) for g, w in zip(got[1:], want[1:]))
    assert e <= 1e-15, (what, "kp_linear / ref / des", e)
    return e
