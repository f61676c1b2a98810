"""Generates tests/golden/command_v1.npz: sequences of quaternions, IMU samples and joystick commands for the three adapter variants and
the outputs of the orientation and command stages over them.  The parts the reference lets us pin come from its own compiled code
(oracle/_ref/libref_command.so: Utils::quat_to_euler and MovingWindowFilter, `make -C oracle -f command.mk ref`), and the generator
checks that the oracle (oracle/command_oracle.cpp) reproduces them bit for bit before it records the oracle's chain.  The command
stage is the oracle's restatement of main_update (its adapter bodies need ROS message types and cannot be compiled here).  The file
carries all of it to the GPU box, which has no /root/reference.

Contents, variant-major [V = 3 (Gazebo, hardware, Isaac), T ticks, fields, R robots], float64 unless noted:
  inputs   quat [4] (w, x, y, z, non-unit by up to 1e-3, some at the pitch singularity), gyro [3], acc [3], cmd [7], root_pos [3],
           pitch_override [V,T,R] (NaN: none) -- what compute_grf's terrain adaptation leaves in root_euler_d[1] before that tick
  records  rot, rot_z [9], euler (= the reference's quat_to_euler), ang_vel, imu_acc, imu_ang_vel [3] (filtered on Gazebo / Isaac,
           raw on hardware); movement_mode (uint32), kp_linear [3], ref [9] (a1mpc_inputs layout), des [12] (stance layout)
  pins     win_x [K,T] samples and win_y [K,T] the reference's MovingWindowFilter(5) averages
Run:  python tests/golden/make_command_golden.py        (CPU only, seconds; needs oracle/_ref/libref_command.so)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import command_oracle_py as CO  # noqa: E402
from oracle import ref_command_py as RC  # noqa: E402
from command_scenarios import DT, HEIGHT0, HMAX, HMIN, KP_LINEAR, KP_LOCK, VARIANTS, command_sequence, imu_sequence, pitch_overrides  # noqa: E402

R, T = 8, 120


def run_chain(v, quat, gyro, acc, cmd, root_pos, ov):
    """the oracle's orientation + command stages over T ticks; ov: terrain overrides of root_euler_d[1] between ticks"""
    ori = CO.Orientation(R, filtered=(v != 1))
    com = CO.Command(R, v, HEIGHT0[v], HMIN, HMAX, KP_LINEAR, KP_LOCK)
    rec = {k: [] for k in ("rot", "rot_z", "euler", "ang_vel", "imu_acc", "imu_ang_vel", "movement_mode", "kp_linear", "ref", "des")}
    row1 = np.zeros(R)                                    # a1mpc_command_init_batch's ref rows
    for t in range(T):
        o = ori(quat[t], gyro[t], acc[t])
        row1 = np.where(np.isnan(ov[t]), row1, ov[t])
        mode, kp, ref, des = com(DT, cmd[t], root_pos[t], row1)
        row1 = ref[1].copy()
        for k in ("rot", "rot_z", "euler", "ang_vel", "imu_acc", "imu_ang_vel"):
            rec[k].append(o[k])
        for k, x in zip(("movement_mode", "kp_linear", "ref", "des"), (mode, kp, ref, des)):
            rec[k].append(x)
    return {k: np.stack(x) for k, x in rec.items()}


def main():
    assert RC.available(), "oracle/_ref/libref_command.so is missing: make -C oracle -f command.mk ref"
    out = {k: [] for k in ("quat", "gyro", "acc", "cmd", "root_pos", "pitch_override")}
    recs = []
    for v in VARIANTS:
        quat, gyro, acc = imu_sequence(R, T, 100 + v)
        cmd, root_pos = command_sequence(R, T, 200 + v)
        ov = pitch_overrides(R, T, 300 + v)
        rec = run_chain(v, quat, gyro, acc, cmd, root_pos, ov)
        # the pinned part: the reference's own quat_to_euler, bit for bit
        for t in range(T):
            e = RC.quat_to_euler(quat[t])
            assert np.array_equal(e, rec["euler"][t]), (v, t)
        for k, x in zip(out, (quat, gyro, acc, cmd, root_pos, ov)):
            out[k].append(x)
        recs.append(rec)
        mm = rec["movement_mode"]
        h = rec["des"][:, 5]
        print("variant %d: walking share %.2f, toggles %d, height at min %d / max %d ticks, |t2| >= 1 quats %d" % (
            v, mm.mean(), int((np.diff(mm.astype(int), axis=0) != 0).sum()), int((h == HMIN).sum()), int((h == HMAX).sum()),
            int((np.abs(2 * (quat[:, 0] * quat[:, 2] - quat[:, 3] * quat[:, 1])) >= 1).sum())))
    rng = np.random.default_rng(7)
    win_x = np.concatenate([rng.standard_normal((4, T)), 1e8 + rng.standard_normal((2, T)), rng.standard_normal((2, T)) * 1e-12])
    win_y = np.stack([RC.window(5, x) for x in win_x])
    for x, y in zip(win_x, win_y):
        assert np.array_equal(CO.window(5, x), y)
    G = {k: np.stack(x) for k, x in out.items()}
    for k in recs[0]:
        G[k] = np.stack([r[k] for r in recs])
    G["win_x"], G["win_y"] = win_x, win_y
    path = os.path.join(ROOT, "tests", "golden", "command_v1.npz")
    np.savez_compressed(path, **G)
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))


if __name__ == "__main__":
    main()
