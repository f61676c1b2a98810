"""Generates tests/golden/stance_v1.npz from the REFERENCE'S OWN code: oracle/_ref/libref_mpc.so (A1RobotControl.cpp compiled unmodified
against the header stand-ins of oracle/ref_shim/), driven through oracle/ref_py.py::compute_grf with stance_leg_control_type = 0 -- the QP
branch, PD law included (A1RobotControl.cpp:321-333, 377-445).  The QP it hands to OsqpEigen is solved by the oracle's OSQP-algorithm
restatement at eps 1e-11 (solver="tight").  The file carries the reference to the GPU box, which has no reference sources.

Contents: 96 states, 32 for each QP configuration (config/{gazebo,hardware,isaac}_a1_qp.yaml: gains and masses 12, 15, 12 kg), all 16
contact masks in each, kp_linear x, y = 0 on every third state, tilts up to 0.3 rad, yaw errors on both sides of +-1.5 * 3.1415926.
  yaml [S] (int32, index into stance_scenarios.NAMES); x0 [S,12]; rot, rot_z [S,9] row-major; foot [S,12]; contact [S] (uint32);
  des [S,12] (root_euler_d, root_pos_d, root_lin_vel_d body, root_ang_vel_d); kp_linear [S,3]; kd_linear, kp_angular, kd_angular [S,3];
  mass [S]; q [S,12] the gradient exactly as handed to OsqpEigen; f_body [S,12] what compute_grf returned.
Run:  python tests/golden/make_stance_golden.py        (CPU only, a few seconds; needs the reference sources for `make -C oracle ref`)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import oracle_py as O
from oracle import ref_py as R
from stance_scenarios import NAMES, PI_REF, YAMLS, robots, to_ref9

PER_YAML = 32


def main():
    assert R.available(), "oracle/_ref/libref_mpc.so missing: run `make -C oracle ref` where the reference sources are present"
    out = {k: [] for k in ("yaml", "x0", "rot", "rot_z", "foot", "contact", "des", "kp_linear", "kd_linear", "kp_angular", "kd_angular", "mass",
                           "q", "f_body")}
    for y, name in enumerate(NAMES):
        mass, _, kdl, kpa, kda = YAMLS[name]
        st = robots(PER_YAML, 20261015 + y, name, contact=np.arange(PER_YAML) % 16)
        cfg = O.make_config(mass=mass)
        for b in range(PER_YAML):
            ref9, yaw_d, pdxy = to_ref9(st["des"][:, b])
            g12 = np.concatenate([st["kp_linear"][:, b], kdl, kpa, kda])
            r = R.compute_grf(cfg, st["x0"][:, b], st["rot"][:, b], st["foot"][:, b], ref9, int(st["contact"][b]), control_type=0, solver="tight",
                              rot_z=st["rot_z"][:, b], root_pos_d_xy=pdxy, yaw_d=yaw_d, gains=g12)
            for k in ("x0", "rot", "rot_z", "foot", "des", "kp_linear"):
                out[k].append(st[k][:, b])
            out["contact"].append(st["contact"][b]); out["yaml"].append(y); out["mass"].append(mass)
            out["kd_linear"].append(kdl); out["kp_angular"].append(kpa); out["kd_angular"].append(kda)
            out["q"].append(r["qp"][1]); out["f_body"].append(r["f_body"])
    arr = {k: np.array(v, dtype=np.float64) for k, v in out.items()}
    arr["contact"] = arr["contact"].astype(np.uint32); arr["yaml"] = arr["yaml"].astype(np.int32)
    err = arr["des"][:, 2] - arr["x0"][:, 2]
    path = os.path.join(ROOT, "tests", "golden", "stance_v1.npz")
    np.savez_compressed(path, **arr)
    print("wrote %s (%.1f kB): %d states, yaw wraps +%d / -%d, locked kp %d, masks %d, |f|max %.1f N"
          % (path, os.path.getsize(path) / 1e3, len(arr["yaml"]), (err > 1.5 * PI_REF).sum(), (err < -1.5 * PI_REF).sum(),
             (arr["kp_linear"][:, 0] == 0).sum(), len(set(arr["contact"].tolist())), np.abs(arr["f_body"]).max()))


if __name__ == "__main__":
    main()
