"""Robot states and gains for the QP-branch stance controller (a1mpc_stance_qp_batch): the gains and masses of the reference's three
QP configurations, a seeded state generator in the batch-major layout of the call, and the PD law of A1RobotControl.cpp:325-333,
379-391 vectorised over a batch (tests/test_ref_pin.py::_root_acc is the one-robot statement it is checked against)."""
import numpy as np

# config/{gazebo,hardware,isaac}_a1_qp.yaml: robot mass, kp_linear, kd_linear, kp_angular, kd_angular
YAMLS = {
    "gazebo": (12.0, (100.0, 100.0, 300.0), (70.0, 70.0, 120.0), (150.0, 150.0, 1.0), (4.5, 4.5, 30.0)),
    "hardware": (15.0, (400.0, 400.0, 1500.0), (300.0, 200.0, 120.0), (40.0, 40.0, 10.0), (1.0, 1.0, 0.5)),
    "isaac": (12.0, (1450.0, 1450.0, 3800.0), (2600.0, 2600.0, 0.0), (420.0, 420.0, 150.0), (0.0, 0.0, 560.0)),
}
NAMES = ("gazebo", "hardware", "isaac")
PI_REF = 3.1415926          # the literal of A1RobotControl.cpp:328-332
NOMINAL_FOOT = np.array([[0.17, 0.15, -0.3], [0.17, -0.15, -0.3], [-0.17, 0.15, -0.3], [-0.17, -0.15, -0.3]])


def gains(name):
    """(mass, kd_linear[3], kp_angular[3], kd_angular[3]) -- the batch-uniform part"""
    m, _, kdl, kpa, kda = YAMLS[name]
    return m, np.array(kdl), np.array(kpa), np.array(kda)


def rot_rows(roll, pitch, yaw):
    """root_rot_mat = Rz(yaw) Ry(pitch) Rx(roll), row-major [9,B]"""
    cr, sr, cp, sp, cy, sy = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    return np.stack([cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr,
                     sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr,
                     -sp, cp * sr, cp * cr])


def rz_rows(yaw):
    c, s = np.cos(yaw), np.sin(yaw)
    z, o = np.zeros_like(yaw), np.ones_like(yaw)
    return np.stack([c, -s, z, s, c, z, z, z, o])


def robots(B, seed, name="gazebo", contact=None, lock_every=3, tilt=0.3):
    """B robots, batch-major: x0 [12,B], rot, rot_z [9,B], foot [12,B], contact [B], des [12,B], kp_linear [3,B].
    Tilts up to `tilt` rad; a quarter of the robots face near +-pi with a desired yaw across it, so that the euler-error wrap of
    :328-332 fires both ways (no error within 1e-9 of +-1.5 * 3.1415926); every `lock_every`-th robot has kp_linear x, y = 0 (the
    walking lock of GazeboA1ROS.cpp:183)."""
    rng = np.random.default_rng(seed)
    roll, pitch = rng.uniform(-tilt, tilt, (2, B))
    yaw = rng.uniform(-np.pi, np.pi, B)
    near = rng.random(B) < 0.25
    yaw = np.where(near, np.sign(yaw) * (np.pi - rng.uniform(0.0, 0.3, B)), yaw)
    yaw_d = yaw + rng.normal(0.0, 0.3, B)
    yaw_d = (yaw_d + np.pi) % (2 * np.pi) - np.pi
    err = yaw_d - yaw
    bad = np.minimum(np.abs(err - 1.5 * PI_REF), np.abs(err + 1.5 * PI_REF)) < 1e-9
    yaw_d[bad] += 1e-6
    x0 = np.zeros((12, B))
    x0[0], x0[1], x0[2] = roll, pitch, yaw
    x0[3:5] = rng.normal(0.0, 0.5, (2, B)); x0[5] = rng.uniform(0.15, 0.35, B)
    x0[6:9] = rng.normal(0.0, 0.5, (3, B)); x0[9:12] = rng.normal(0.0, 0.5, (3, B))
    rot = rot_rows(roll, pitch, yaw)
    rel = NOMINAL_FOOT[None] + rng.normal(0.0, 0.03, (B, 4, 3))
    foot = np.einsum("bij,blj->bli", rot.T.reshape(B, 3, 3), rel).reshape(B, 12).T.copy()
    if contact is None:
        contact = rng.integers(0, 16, B)
    des = np.zeros((12, B))
    des[0:2] = rng.normal(0.0, 0.1, (2, B)); des[2] = yaw_d
    des[3:5] = x0[3:5] + rng.normal(0.0, 0.05, (2, B)); des[5] = rng.uniform(0.25, 0.32, B)
    des[6:9] = rng.normal(0.0, 0.5, (3, B)); des[9:12] = rng.normal(0.0, 0.5, (3, B))
    kpl = np.repeat(np.array(YAMLS[name][1])[:, None], B, axis=1)
    kpl[0:2, ::lock_every] = 0.0
    return dict(x0=x0, rot=rot, rot_z=rz_rows(yaw), foot=foot, contact=np.asarray(contact, dtype=np.uint32), des=des, kp_linear=kpl)


def root_acc_batch(x0, rot, des, kp_linear, kd_linear, kp_angular, kd_angular, mass):
    """A1RobotControl.cpp:325-333, 379-391 over a batch: [6,B]"""
    B = x0.shape[1]
    R = rot.T.reshape(B, 3, 3)
    e, p, w, v = x0[0:3], x0[3:6], x0[6:9], x0[9:12]
    ed, pd, vd, wd = des[0:3], des[3:6], des[6:9], des[9:12]
    err = ed - e
    err[2] = np.where(err[2] > PI_REF * 1.5, ed[2] - PI_REF * 2 - e[2], np.where(err[2] < -PI_REF * 1.5, ed[2] + PI_REF * 2 - e[2], err[2]))
    kdl, kpa, kda = (np.asarray(g, dtype=np.float64)[:, None] for g in (kd_linear, kp_angular, kd_angular))
    acc = np.zeros((6, B))
    acc[0:3] = kp_linear * (pd - p) + np.einsum("bik,kb->ib", R, kdl * (vd - np.einsum("bki,kb->ib", R, v)))
    acc[3:6] = kpa * err + kda * (wd - np.einsum("bki,kb->ib", R, w))
    acc[2] += mass * 9.8
    return acc


def inertia_inv(rot_z, foot):
    """inertia_inv of A1RobotControl.cpp:394-399 for one robot: [6,12]"""
    rz = np.asarray(rot_z).reshape(3, 3)
    ft = np.asarray(foot).reshape(4, 3)
    M = np.zeros((6, 12))
    for i in range(4):
        r = ft[i]
        S = np.array([[0, -r[2], r[1]], [r[2], 0, -r[0]], [-r[1], r[0], 0]])
        M[0:3, 3 * i:3 * i + 3] = np.eye(3)
        M[3:6, 3 * i:3 * i + 3] = rz.T @ S
    return M


Q = np.diag([1.0, 1.0, 1.0, 400.0, 400.0, 100.0])   # A1RobotControl.cpp:11


def qp_gradient(rot_z, foot, acc):
    """-M^T Q root_acc: the gradient compute_grf hands to OsqpEigen (:406)"""
    return -inertia_inv(rot_z, foot).T @ Q @ acc


def oracle_forces(O, acc, rot_z, rot, foot, contact):
    """O.grf_qp_single per robot: f_body [12,B], status [B] in the engine's codes (NO_CONTACT for mask 0)"""
    B = acc.shape[1]
    f = np.zeros((12, B)); ok = np.zeros(B, dtype=bool)
    for b in range(B):
        if int(contact[b]) & 15 == 0:
            ok[b] = True
            continue
        fb, info = O.grf_qp_single(acc[:, b], rot_z[:, b], rot[:, b], foot[:, b], int(contact[b]), O.MODE_EXACT)
        f[:, b] = fb; ok[b] = info[1] == 1
    return f, ok


def to_ref9(des):
    """des [12] -> (ref[9] of the a1mpc_inputs layout, yaw_d, root_pos_d x/y): the arguments of oracle/ref_py.py::compute_grf"""
    d = np.asarray(des)
    ref9 = np.array([d[0], d[1], d[9], d[10], d[11], d[6], d[7], d[8], d[5]])
    return ref9, float(d[2]), (float(d[3]), float(d[4]))
