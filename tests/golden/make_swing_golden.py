"""Generates tests/golden/swing_v1.npz from the REFERENCE'S OWN code: oracle/_ref/libref_swing.so (A1RobotControl.cpp and utils/Utils.cpp
compiled unmodified against the header stand-ins of oracle/ref_shim/, `make -C oracle -f swing.mk ref`), driven by ref_swing_ticks: update_plan ->
generate_swing_legs_ctrl -> compute_grf (MPC branch) for 300 ticks on one controller per robot, so that its filters carry over.  The
solve inside compute_grf is answered by zeros; only what comes before it (terrain adaptation) is recorded.  The file carries the
reference to the GPU box, which has no /root/reference.

Contents, robot-major [R, T, ...] (R = 6 robots, T = 300 ticks), float64 unless noted:
  inputs   movement_mode (int32), lin_vel, lin_vel_d, root_pos [3], rot_z, rot [9] row-major, foot_pos_abs [12], foot_force [4];
           per robot kp, kd [12] (robots 0-2: A1CtrlStates::reset() gains, 3-5: the ROS-parameter defaults), gait_counter_speed [4]
  records  gait_counter [4], plan_contacts, contacts (uint32 masks), foot_pos_target_rel, f_kin, foot_pos_cur, foot_pos_recent_contact [12],
           root_euler_d1, terrain_pitch -- every tick, as the reference's state holds them after compute_grf (use_terrain_adapt = 1)
Run:  python tests/golden/make_swing_golden.py        (CPU only, a few seconds; needs /root/reference)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_swing_py as R
from swing_scenarios import KD_RESET, KD_ROS, KP_RESET, KP_ROS, Scenario

T = 300
# robot: slope (dz/dx, dz/dy), early touchdown, spans with root z <= 0.1, gait_counter_speed
ROBOTS = [((0.0, 0.0), False, False, 2.0),      # flat ground: acos near 1
          ((0.9, 0.0), True, False, 3.0),       # steep, front feet high: F_R_diff > 0.05, clip at 0.5
          ((-0.9, 0.1), False, False, 2.0),     # steep the other way
          ((0.15, -0.05), True, False, 1.5),
          ((-0.3, 0.2), True, True, 2.5),
          ((0.5, 0.0), False, True, 4.0)]
INPUTS = ("movement_mode", "lin_vel", "lin_vel_d", "root_pos", "rot_z", "rot", "foot_pos_abs", "foot_force")


def scenario(seed, robots, T):
    """tick-major inputs of len(robots) robots: dict name -> [R, T, ...]"""
    sc = Scenario(len(robots), seed, slopes=[r[0] for r in robots], early=[r[1] for r in robots], low=[r[2] for r in robots],
                  speeds=[r[3] for r in robots])
    ticks = [sc.tick() for _ in range(T)]
    out = {k: np.stack([np.asarray(tk[k]).T for tk in ticks], axis=1) for k in INPUTS + ("gait_counter", "plan_contacts", "foot_pos_target_rel")}
    out["speed"] = sc.speed
    return out


def run_reference(inp, kp, kd, use_terrain_adapt=1):
    R_ = inp["movement_mode"].shape[0]
    recs = []
    for r in range(R_):
        recs.append(R.swing_ticks(kp[r], kd[r], np.full(4, inp["speed"][r]), *[inp[k][r] for k in INPUTS], use_terrain_adapt=use_terrain_adapt))
    return {k: np.stack([rc[k] for rc in recs]) for k in recs[0]}


def main():
    assert R.available(), "oracle/_ref/libref_swing.so missing: run `make -C oracle -f swing.mk ref` where /root/reference is mounted"
    inp = scenario(20261015, ROBOTS, T)
    kp = np.stack([KP_RESET] * 3 + [KP_ROS] * 3)
    kd = np.stack([KD_RESET] * 3 + [KD_ROS] * 3)
    rec = run_reference(inp, kp, kd)
    # update_plan inside the reference and the scenario's own counters agree (the scenario drives its forces and lifts by them)
    assert np.array_equal(rec["gait_counter"], inp["gait_counter"]) and np.array_equal(rec["plan_contacts"], inp["plan_contacts"])
    out = {k: inp[k] for k in INPUTS}
    out["movement_mode"] = out["movement_mode"].astype(np.int32)
    out.update(kp=kp, kd=kd, gait_counter_speed=np.repeat(inp["speed"][:, None], 4, axis=1))
    out.update(rec)
    path = os.path.join(ROOT, "tests", "golden", "swing_v1.npz")
    np.savez_compressed(path, **out)
    early = ((rec["contacts"] & ~rec["plan_contacts"]) != 0).sum()
    print("wrote %s (%.2f MB): %d early-contact ticks, |terrain_pitch| max %.3f, euler_d1 range [%.3f, %.3f], low-body ticks %d"
          % (path, os.path.getsize(path) / 1e6, early, np.abs(rec["terrain_pitch"]).max(), rec["root_euler_d1"].min(), rec["root_euler_d1"].max(),
             (inp["root_pos"][:, :, 2] <= 0.1).sum()))


if __name__ == "__main__":
    main()
