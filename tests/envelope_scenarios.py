"""MPC states outside the benchmark's trot distribution, as the rest of the controller produces them, for the envelope suites
(tests/test_emu_envelope.py on the CPU emulator, tests/test_gpu_envelope.py through the C ABI).

a1mpc_gen_states draws roll and pitch with sigma 0.02 rad, heights of 0.25-0.32 m against a fixed 0.30 m reference, zero roll and
pitch references and commands of at most 0.6 m/s.  The controller leaves that box: a1mpc_command_batch moves the height reference
anywhere in [0.10, 0.32] m, a1mpc_terrain_pitch_batch writes pitch references up to +-0.5 rad, early contact produces any stance
mask, and a pushed robot has velocity errors of metres per second.  Each family starts from a1mpc.gen_states(B, 4, seed), draws
the stance mask uniformly from 1..15 and moves the state into one of those regions.  Deterministic: numpy, seeded."""
import numpy as np

FAMILIES = ("height", "tilt", "push", "combined")
CENSUS_TOL = 1e-6     # N: a force is "on" a face when it is within this of it


def _rot_rows(roll, pitch, yaw):
    """Rz(yaw) Ry(pitch) Rx(roll), row-major [9,B] (the layout of a1mpc_inputs::rot)"""
    cr, sr, cp, sp, cy, sy = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    return np.stack([cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr,
                     sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr,
                     -sp, cp * sr, cp * cr])


def _height(st, rng, B):
    st["ref"][8] = rng.uniform(0.10, 0.32, B)          # the whole clamp of a1mpc_command_batch's height command
    st["x0"][11] = rng.uniform(-1.0, 1.0, B)           # vertical velocity


def _push(st, rng, B):
    st["x0"][9:11] += rng.uniform(-1.5, 1.5, (2, B))    # horizontal velocity error
    st["x0"][6:9] += rng.normal(0.0, 1.5, (3, B))       # angular velocity
    st["ref"][4] = rng.uniform(-2.0, 2.0, B)            # yaw-rate command


def _tilt(st, rng, B):
    st["ref"][1] = rng.uniform(-0.5, 0.5, B)            # terrain-pitch reference (a1mpc_terrain_pitch_batch's range)
    st["ref"][0] = rng.uniform(-0.2, 0.2, B)
    roll, pitch = rng.normal(0.0, 0.2, (2, B))
    yaw = st["x0"][2]
    R_old = st["rot"].T.reshape(B, 3, 3)
    body = np.einsum("bji,blj->bli", R_old, st["foot"].T.reshape(B, 4, 3))     # R_old' foot: the body-frame footholds
    st["x0"][0], st["x0"][1] = roll, pitch
    st["rot"] = _rot_rows(roll, pitch, yaw)
    R_new = st["rot"].T.reshape(B, 3, 3)
    st["foot"] = np.einsum("bij,blj->bli", R_new, body).reshape(B, 12).T.copy()


def family(a1, name, B, seed):
    """B states of family `name` (FAMILIES): dict x0, rot, foot, ref [rows, B], contact [B] with every mask 1..15"""
    st = a1.gen_states(B, 4, seed)
    st = {k: v.copy() for k, v in st.items()}
    rng = np.random.default_rng([seed, FAMILIES.index(name)])
    st["contact"] = rng.integers(1, 16, size=B).astype(np.uint32)
    if name == "height":
        _height(st, rng, B)
    elif name == "tilt":
        _tilt(st, rng, B)
    elif name == "push":
        _push(st, rng, B)
    elif name == "combined":
        _height(st, rng, B)
        _push(st, rng, B)
        st["ref"][1] = rng.uniform(-0.5, 0.5, B)
    else:
        raise ValueError(name)
    return st


def census(u_full, contact, mu=0.3, fz_max=180.0, tol=CENSUS_TOL, sched=None):
    """How many QPs have at least one stance foot-step on each face of the friction pyramid, from a whole-horizon solution
    u_full [B, 12N] (world frame, step-major, as O.compute_grf_batch(..., want_u=True) returns it):
      fzmax   -- fz = fz_max
      vertex  -- f = 0 (the cone's apex: fz = 0, hence fx = fy = 0)
      edge    -- |fx| = mu fz or |fy| = mu fz with fz above the vertex
      foot0   -- a whole stance foot at the vertex over the horizon
    sched [N,B] (optional): per-step stance masks instead of one mask for the whole horizon."""
    B, n = u_full.shape
    N = n // 12
    u = u_full.reshape(B, N, 4, 3)
    fx, fy, fz = u[..., 0], u[..., 1], u[..., 2]
    if sched is None:
        stance = ((np.asarray(contact, dtype=np.int64)[:, None] >> np.arange(4)) & 1).astype(bool)[:, None, :].repeat(N, axis=1)
    else:
        stance = ((np.asarray(sched, dtype=np.int64).T[:, :, None] >> np.arange(4)) & 1).astype(bool)
    vertex = stance & (fz <= tol)
    edge = stance & ~vertex & ((np.abs(np.abs(fx) - mu * fz) <= tol) | (np.abs(np.abs(fy) - mu * fz) <= tol))
    top = stance & (fz >= fz_max - tol)
    leg_in = stance.any(axis=1)
    foot0 = leg_in & (vertex | ~stance).all(axis=1)
    return {"fzmax": int(top.any(axis=(1, 2)).sum()), "vertex": int(vertex.any(axis=(1, 2)).sum()),
            "edge": int(edge.any(axis=(1, 2)).sum()), "foot0": int(foot0.any(axis=1).sum()), "B": int(B)}


def check_census(name, c, floors):
    """prints the census and asserts each floor (a fraction of the QPs): a later edit of a family cannot drift back into easy states"""
    print("census %-9s B=%-5d fz_max %5d  vertex %5d  edge %5d  foot at vertex %5d" % (name, c["B"], c["fzmax"], c["vertex"], c["edge"], c["foot0"]))
    for k, frac in floors.items():
        assert c[k] >= frac * c["B"], (name, k, c[k], frac * c["B"])
