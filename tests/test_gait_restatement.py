"""CPU: the staged gait kernels (update_plan_gait_kernel, swing_legs_gait_kernel on the block emulator) against two independent checks.
  * A numpy restatement of the generalised expressions, for rows with cpg != 2 cps (the walk 240 / 180, and 300 / 200 and 240 / 90) at
    non-integer leg speeds: counters, planned contacts, the Raibert foothold targets with the robot's own cps, the spline time
    (g - cps) / (cpg - cps) in single precision, the Bezier targets, f_kin, early contact past the middle of the swing, contacts, the
    swing state (foot_pos_start, last positions, early mask) and the recent-contact points, over 300 ticks of tests/swing_scenarios.py's
    stand-then-walk robots with early contacts.  Tolerances of tests/test_swing_ref_pin.py for f_kin, exact for the masks and counters.
  * Where oracle/_ref/libref_gait.so exists: the REFERENCE'S OWN update_plan and generate_swing_legs_ctrl (oracle/ref_gait_wrap.cpp:
    gait_type 0, counters preset to the row's offsets on standstill ticks, per-robot counter_per_gait / counter_per_swing) for the rows
    with cpg = 2 cps: trot, pace, bound, pronk, a phase-shifted trot and 200 / 100."""
import os
import sys
from collections import deque

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import emu_gait_py as EG  # noqa: E402
from oracle import ref_gait_py as RG  # noqa: E402
from swing_scenarios import TOL_FKIN  # noqa: E402

DT = 0.0025
KP, KD = np.tile([150.0, 150.0, 200.0], 4), np.tile([5.0, 5.0, 3.0], 4)
SW_START, SW_RLAST, SW_TLAST, SW_RC, SW_EARLY = 0, 12, 24, 36, 48
CLEAR2 = float(np.float32(0.4))


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


def inputs(rows, seed, T=300):
    """tick-major inputs of swing_scenarios for one robot per row, at non-integer speeds"""
    import make_swing_golden as M
    rng = np.random.default_rng(seed)
    robots = [((rng.uniform(-0.9, 0.9), rng.uniform(-0.3, 0.3)), True, bool(i % 3 == 2), float(rng.uniform(1.5, 4.5))) for i in range(len(rows))]
    return M.scenario(seed, robots, T)


class Restated:
    """the generalised update_plan + generate_swing_legs_ctrl of one robot with gait row `row`"""

    def __init__(self, row, gp, speed, wrong=None):
        self.off, self.cpg, self.cps = np.array(row[:4]), float(row[4]), float(row[5])
        self.wrong = wrong     # test only: one expression in the reference's cpg = 2 cps form (see the test below)
        self.dfp = np.array(gp.default_foot_pos).reshape(3, 4)
        self.cdt, self.dxl, self.dyl = gp.control_dt, gp.foot_delta_x_limit, gp.foot_delta_y_limit
        self.sp = float(speed)
        self.gc = np.zeros(4)
        self.start, self.rlast, self.tlast, self.rc = np.zeros((4, 3)), np.zeros((4, 3)), np.zeros((4, 3)), np.zeros((4, 3))
        self.early = 0
        self.win = [[deque() for _ in range(3)] for _ in range(4)]

    def tick(self, mode, lv, lvd, rz, fpa, ff):
        cps, cpg = self.cps, self.cpg
        if mode:
            self.gc = np.fmod(self.gc + self.sp, cpg)
            plan = sum(1 << i for i in range(4) if self.gc[i] <= cps)
        else:
            self.gc = self.off.copy()
            plan = 15
        Rz = rz.reshape(3, 3)
        vr = Rz.T @ lv
        kf = np.sqrt(abs(self.dfp[2, 0]) / 9.8)
        raibert = (((120.0 if self.wrong == "foothold" else cps) / self.sp) * self.cdt) / 2.0
        dx = np.clip(kf * (vr[0] - lvd[0]) + raibert * lvd[0], -self.dxl, self.dxl)
        dy = np.clip(kf * (vr[1] - lvd[1]) + raibert * lvd[1], -self.dyl, self.dyl)
        tgt = np.stack([self.dfp[0] + dx, self.dfp[1] + dy, self.dfp[2]], axis=1)      # [4 legs][3]
        fk, con, cur_all = np.zeros((4, 3)), 0, np.zeros((4, 3))
        for i in range(4):
            p = fpa.reshape(4, 3)[i]
            cur = Rz.T @ p
            cur_all[i] = cur
            g = self.gc[i]
            if g <= cps:
                t = 0.0
                self.start[i] = cur
            else:
                swing_len = cps if self.wrong == "spline" else cpg - cps
                t = float(np.float32(np.float32(g - cps) / np.float32(swing_len)))
            st, fin = self.start[i], tgt[i]
            P = [[st[a], st[a], fin[a], fin[a], fin[a]] for a in range(3)]
            P[2] = [st[2], st[2] + 0.0, fin[2] + CLEAR2, fin[2], fin[2]]
            c = [1.0, 4.0, 6.0, 4.0, 1.0]
            target = np.array([sum(c[k] * t ** k * (1.0 - t) ** (4 - k) * P[a][k] for k in range(5)) for a in range(3)])
            vcur, vtgt = (cur - self.rlast[i]) / DT, (target - self.tlast[i]) / DT
            self.rlast[i], self.tlast[i] = cur, target
            fk[i] = (target - cur) * KP[3 * i:3 * i + 3] + (vtgt - vcur) * KD[3 * i:3 * i + 3]
            planned = (plan >> i) & 1
            mid = cps * 1.5 if self.wrong == "mid" else cps + 0.5 * (cpg - cps)
            if g <= mid:
                self.early &= ~(1 << i)
            if not planned and g > mid and ff[i] > 30.0:
                self.early |= 1 << i
            if planned or (self.early >> i) & 1:
                con |= 1 << i
                for a in range(3):
                    w = self.win[i][a]
                    w.append(p[a])
                    if len(w) > 60:
                        w.popleft()
                    self.rc[i, a] = sum(w) / 60.0
        return dict(gc=self.gc.copy(), plan=plan, tgt=tgt.reshape(12), fk=fk.reshape(12), con=con, cur=cur_all.reshape(12),
                    start=self.start.reshape(12).copy(), rlast=self.rlast.reshape(12).copy(), tlast=self.tlast.reshape(12).copy(),
                    rc=self.rc.reshape(12).copy(), early=self.early)


def kernels(gp, rows, inp, T):
    """the staged gait kernels on the emulator over T ticks; per tick a dict of [R, ...] records (swing state fields included)"""
    R = rows.shape[1]
    speed = np.ascontiguousarray(np.repeat(inp["speed"][None, :], 4, axis=0))
    gc, swing = np.zeros((4, R)), np.zeros((EG.swing_fields(), R))
    g = lambda k, t: np.ascontiguousarray(inp[k][:, t].T)
    out = []
    for t in range(T):
        plan, tr = np.zeros(R, np.uint32), np.zeros((12, R))
        mode = np.ascontiguousarray(inp["movement_mode"][:, t].astype(np.uint32))
        EG.update_plan(gp, rows, gc, speed, mode, g("lin_vel", t), g("lin_vel_d", t), g("rot_z", t), g("rot", t), g("root_pos", t), plan, None, tr,
                       None, None)
        fk, con, cur, rc = np.zeros((12, R)), np.zeros(R, np.uint32), np.zeros((12, R)), np.zeros((12, R))
        EG.swing_legs(gp, KP, KD, DT, rows, swing, np.ascontiguousarray(gc), plan, g("rot_z", t), g("foot_pos_abs", t), tr, g("foot_force", t), fk,
                      con, cur, rc)
        out.append(dict(gc=gc.T.copy(), plan=plan.copy(), tgt=tr.T.copy(), fk=fk.T.copy(), con=con.copy(), cur=cur.T.copy(), rc=rc.T.copy(),
                        start=swing[SW_START:SW_START + 12].T.copy(), rlast=swing[SW_RLAST:SW_RLAST + 12].T.copy(),
                        tlast=swing[SW_TLAST:SW_TLAST + 12].T.copy(), early=swing[SW_EARLY].astype(np.uint32)))
    return out


def _fk_err(a, b):
    return float((np.abs(a - b) / np.maximum(1.0, np.abs(b).max())).max())


ROWS_GENERAL = [[120, 0, 180, 60, 240, 180], [0, 150, 150, 0, 300, 200], [0, 120, 120, 0, 240, 90], [30, 200, 100, 230, 240, 180],
                [0, 0, 0, 0, 300, 200], [50, 260, 50, 260, 300, 100]]


def test_general_rows_match_the_restatement(a1):
    gp = a1.default_tick_params(0, a1.TICK_MPC).gait
    rows = np.ascontiguousarray(np.array(ROWS_GENERAL, dtype=np.float64).T)
    R, T = rows.shape[1], 300
    inp = inputs(ROWS_GENERAL, 515, T)
    got = kernels(gp, rows, inp, T)
    ref = [Restated(rows[:, r], gp, inp["speed"][r]) for r in range(R)]
    worst = dict(fk=0.0, tgt=0.0, rc=0.0, state=0.0)
    swings = early = 0
    for t in range(T):
        for r in range(R):
            w = ref[r].tick(int(inp["movement_mode"][r, t]), inp["lin_vel"][r, t], inp["lin_vel_d"][r, t], inp["rot_z"][r, t],
                            inp["foot_pos_abs"][r, t], inp["foot_force"][r, t])
            k = {key: v[r] for key, v in got[t].items()}
            what = (t, r)
            assert np.array_equal(k["gc"], w["gc"]) and int(k["plan"]) == w["plan"], what
            assert int(k["con"]) == w["con"] and int(k["early"]) == w["early"], what
            assert np.abs(k["cur"] - w["cur"]).max() <= 1e-15, what
            worst["tgt"] = max(worst["tgt"], float(np.abs(k["tgt"] - w["tgt"]).max()))
            worst["fk"] = max(worst["fk"], _fk_err(k["fk"], w["fk"]))
            worst["rc"] = max(worst["rc"], float(np.abs(k["rc"] - w["rc"]).max()))
            worst["state"] = max(worst["state"], max(float(np.abs(k[f] - w[f]).max()) for f in ("start", "rlast", "tlast")))
            swings += int(w["plan"] != 15)
            early += int((w["con"] & ~w["plan"]) != 0)
    print("general rows vs restatement: %s; swing ticks %d, early-contact ticks %d" % (worst, swings, early))
    assert worst["tgt"] <= 1e-14 and worst["fk"] <= TOL_FKIN and worst["rc"] <= 1e-12 and worst["state"] <= 1e-12
    assert swings > 0 and early > 0


def test_the_restatement_tells_the_generalised_forms_apart(a1):
    """each generalised expression put back in its cpg = 2 cps form -- spline time over cps, early contact past 1.5 cps, the batch's
    cps = 120 in the foothold -- makes the restatement disagree with the kernels on the walk and the other rows: the test above would
    catch a kernel that used it"""
    gp = a1.default_tick_params(0, a1.TICK_MPC).gait
    rows = np.ascontiguousarray(np.array(ROWS_GENERAL, dtype=np.float64).T)
    R, T = rows.shape[1], 300
    inp = inputs(ROWS_GENERAL, 515, T)
    got = kernels(gp, rows, inp, T)
    for wrong in ("spline", "mid", "foothold"):
        ref = [Restated(rows[:, r], gp, inp["speed"][r], wrong) for r in range(R)]
        differs = False
        for t in range(T):
            for r in range(R):
                w = ref[r].tick(int(inp["movement_mode"][r, t]), inp["lin_vel"][r, t], inp["lin_vel_d"][r, t], inp["rot_z"][r, t],
                                inp["foot_pos_abs"][r, t], inp["foot_force"][r, t])
                k = {key: v[r] for key, v in got[t].items()}
                differs = differs or int(k["con"]) != w["con"] or float(np.abs(k["tgt"] - w["tgt"]).max()) > 1e-12 or \
                    _fk_err(k["fk"], w["fk"]) > TOL_FKIN
        assert differs, wrong


needs_ref = pytest.mark.skipif(not RG.available(), reason="oracle/_ref/libref_gait.so absent (no reference sources on this machine)")

ROWS_PINNED = [[0, 120, 120, 0, 240, 120], [0, 120, 0, 120, 240, 120], [0, 0, 120, 120, 240, 120], [0, 0, 0, 0, 240, 120],
               [60, 180, 180, 60, 240, 120], [0, 100, 100, 0, 200, 100], [150, 30, 90, 210, 240, 120]]


@needs_ref
def test_duty_half_rows_match_the_reference_build(a1):
    gp = a1.default_tick_params(0, a1.TICK_MPC).gait
    rows = np.ascontiguousarray(np.array(ROWS_PINNED, dtype=np.float64).T)
    R, T = rows.shape[1], 300
    inp = inputs(ROWS_PINNED, 616, T)
    got = kernels(gp, rows, inp, T)
    worst = dict(fk=0.0, tgt=0.0, rc=0.0)
    for r in range(R):
        rec = RG.gait_ticks(rows[:, r], KP, KD, np.full(4, inp["speed"][r]), *[inp[k][r] for k in ("movement_mode", "lin_vel", "lin_vel_d",
                                                                                                    "root_pos", "rot_z", "rot", "foot_pos_abs",
                                                                                                    "foot_force")])
        for t in range(T):
            k = {key: v[r] for key, v in got[t].items()}
            assert np.array_equal(k["gc"], rec["gait_counter"][t]) and int(k["plan"]) == rec["plan_contacts"][t], (r, t)
            assert int(k["con"]) == rec["contacts"][t], (r, t)
            assert np.abs(k["cur"] - rec["foot_pos_cur"][t]).max() <= 1e-15, (r, t)
            worst["tgt"] = max(worst["tgt"], float(np.abs(k["tgt"] - rec["foot_pos_target_rel"][t]).max()))
            worst["fk"] = max(worst["fk"], _fk_err(k["fk"], rec["f_kin"][t]))
            worst["rc"] = max(worst["rc"], float(np.abs(k["rc"] - rec["foot_pos_recent_contact"][t]).max()))
    print("duty-0.5 rows vs the reference build: %s" % worst)
    assert worst["tgt"] <= 1e-14 and worst["fk"] <= TOL_FKIN and worst["rc"] <= 1e-12
