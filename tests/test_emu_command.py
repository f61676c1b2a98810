"""CPU: the unchanged device code of a1mpc_command.cuh (orientation_kernel, command_kernel) on the block emulator against the oracle over
the fixture's sequences (tests/golden/command_v1.npz), each side carrying its own filter and command state, with the tolerances of the
GPU suite (tests/command_scenarios.py)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import emu_command_py as E  # noqa: E402
from command_scenarios import DT, HEIGHT0, HMAX, HMIN, KP_LINEAR, KP_LOCK, VARIANTS, check_command, check_orientation  # noqa: E402
from oracle import command_oracle_py as CO  # noqa: E402


def test_emulator_matches_oracle_over_fixture():
    with np.load(os.path.join(ROOT, "tests", "golden", "command_v1.npz")) as z:
        G = {k: z[k] for k in z.files}
    _, T, _, R = G["quat"].shape
    worst = 0.0
    for v in VARIANTS:
        filt = v != 1
        imu = E.imu_init(R) if filt else None
        ref = np.full((9, R), np.nan)
        cst = E.command_init(R, v, HEIGHT0[v], HMIN, HMAX, KP_LINEAR, KP_LOCK, ref=ref)
        assert (ref == 0.0).all()
        ori = CO.Orientation(R, filtered=filt)
        com = CO.Command(R, v, HEIGHT0[v], HMIN, HMAX, KP_LINEAR, KP_LOCK)
        row1 = np.zeros(R)
        for t in range(T):
            args = (G["quat"][v, t], G["gyro"][v, t], G["acc"][v, t])
            worst = max(worst, check_orientation(E.orientation(*args, imu=imu), ori(*args), "variant %d tick %d" % (v, t)))
            ov = G["pitch_override"][v, t]
            ref[1] = np.where(np.isnan(ov), ref[1], ov)          # what the terrain stage leaves in row 1
            row1 = np.where(np.isnan(ov), row1, ov)
            mode, kp, des = E.command(cst, DT, G["cmd"][v, t], G["root_pos"][v, t], ref=ref)
            want = com(DT, G["cmd"][v, t], G["root_pos"][v, t], row1)
            row1 = want[2][1].copy()
            worst = max(worst, check_command((mode, kp, ref, des), want, "variant %d tick %d" % (v, t)))
            for k, got in zip(("movement_mode", "kp_linear", "ref", "des"), (mode, kp, ref, des)):
                assert np.array_equal(got, G[k][v, t]), (v, t, k)
    print("emulator vs oracle: worst %.2e" % worst)


def test_command_without_ref_keeps_its_own_pitch():
    """without ref, root_euler_d[1] integrates from the state; the 'des' rows match the ref-carrying run when nothing overrides row 1"""
    R, T = 64, 40
    rng = np.random.default_rng(5)
    cmd = np.zeros((7, R)); cmd[4] = 0.3; cmd[6, :] = 1.0
    pos = rng.standard_normal((3, R))
    a = E.command_init(R, 0)
    ref = np.zeros((9, R))
    b = E.command_init(R, 0, ref=ref)
    for t in range(T):
        _, _, d0 = E.command(a, DT, cmd, pos)
        _, _, d1 = E.command(b, DT, cmd, pos, ref=ref)
        cmd[6] = 0.0
        assert np.array_equal(d0, d1) and np.array_equal(ref[1], d1[1])
    assert np.abs(d0[1] - T * 0.3 * DT).max() < 1e-15
