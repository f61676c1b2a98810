"""-m gpu: every batch entry point of the C ABI, once with host arrays and once with the same data on device pointers.  The two
calls must give the same outputs bit for bit (in/out arrays and device-resident state included) and launch the same number of
kernels.  Cases cover ld > B, precision 32 and optional outputs left NULL.

Then the side rule: a call whose batch arrays are not all host or all device, or that passes a device pointer for a batch-uniform
parameter read on the host, fails with A1MPC_EINVAL before anything is enqueued (no launch, host outputs untouched), and the handle
keeps working."""
import ctypes as C

import numpy as np
import pytest

from common import estimation_scenario
from swing_scenarios import KD_RESET, KP_RESET

pytestmark = pytest.mark.gpu

B, LD_IN, LD_OUT = 40, 47, 53    # ld > B: a slice of wider caller arrays, with different leading dimensions in and out
N = 10
DT = 0.0025


@pytest.fixture(scope="module")
def a1(built):
    import a1mpc
    return a1mpc


@pytest.fixture(scope="module")
def engines(a1):
    es = {}

    def engine(prec):
        if prec not in es:
            es[prec] = a1.Engine(a1.default_config(precision=prec))
        return es[prec]
    yield engine
    for e in es.values():
        e.close()


class Case:
    """arrays: name -> (role, initial contents), role "in" or "out" (outs and in/outs are compared after the call; the
    contents of an out are a fill pattern that the call must leave alone where it does not write); params: batch-uniform
    host arrays; call(a1, eng, p) makes the call with p: name -> pointer (missing names are NULL); state(a1, eng, p) returns a
    freshly prepared device state buffer and its size, passed as p["state"] (p: host pointers to fresh copies of the arrays)"""

    def __init__(self, arrays, call, params=None, state=None, prec=64):
        self.arrays, self.call, self.params, self.state, self.prec = arrays, call, params or {}, state, prec


def _solve_arrays(prec, ld_in=B, ld_out=B, ext=False, optional=True, seed=3):
    ft = np.float32 if prec == 32 else np.float64
    import a1mpc
    st = a1mpc.gen_states(ld_in, 4, seed)
    st["x0"][:, B:] = 1e6                       # columns past B belong to someone else: never read
    arrs = {k: ("in", np.ascontiguousarray(v, dtype=(np.uint32 if k == "contact" else ft))) for k, v in st.items()}
    if ext:
        sched, normals = a1mpc.gen_schedule(ld_in, N, 4, seed)
        sched[:, B:] = 0b1111
        arrs["sched"] = ("in", sched)
        arrs["normals"] = ("in", normals.astype(ft))
    arrs["f_body"] = ("out", np.full((12, ld_out), 7.5, dtype=ft))
    arrs["status"] = ("out", np.full(B, -7, dtype=np.int32))
    if optional:
        arrs["iters"] = ("out", np.full(B, -7, dtype=np.int32))
        arrs["u_full"] = ("out", np.full((12 * N, ld_out), 7.5, dtype=ft))
    return arrs


def _solve_call(fn, ld_in=B, ld_out=B, ext=False, warm=False):
    def call(a1, eng, p):
        inp = a1.Inputs(p.get("x0"), p.get("rot"), p.get("foot"), p.get("ref"), p.get("contact"), ld_in)
        out = a1.Outputs(p.get("f_body"), p.get("status"), p.get("iters"), p.get("u_full"), ld_out)
        args = [eng.h, B, C.byref(inp)]
        if ext:
            args.append(C.byref(a1.InputsExt(p.get("sched"), p.get("normals"))))
        args.append(C.byref(out))
        if warm:
            args += [p["state"], 1 if ext else 0]
        return getattr(a1.lib(), fn)(*args)
    return call


def _warm_state(call):
    """a warm-start buffer primed by one host-array call of the case itself, so that the compared call starts from guesses"""
    def state(a1, eng, p):
        w = eng.warm_alloc(B)
        assert call(a1, eng, dict(p, state=w.value)) == 0, a1.lib().a1mpc_last_error()
        return w, a1.lib().a1mpc_warm_bytes(eng.h, B)
    return state


def _solve_case(fn, prec=64, ld_in=B, ld_out=B, ext=False, warm=False, optional=True):
    call = _solve_call(fn, ld_in, ld_out, ext, warm)
    return Case(_solve_arrays(prec, ld_in, ld_out, ext, optional), call, state=_warm_state(call) if warm else None, prec=prec)


def _dense_arrays(rng):
    n, m = 12 * N, 20 * N
    M = rng.standard_normal((B, n, n))
    H = M @ M.transpose(0, 2, 1) + n * np.eye(n)
    contact = rng.choice([0b1001, 0b0110, 0b1111, 0], B).astype(np.uint32)
    return n, m, H, rng.standard_normal((B, n)), contact


def _cases():
    import a1mpc
    rng = np.random.default_rng(17)
    cases = {}
    cases["solve"] = _solve_case("a1mpc_solve_batch")
    cases["solve_ld"] = _solve_case("a1mpc_solve_batch", ld_in=LD_IN, ld_out=LD_OUT)
    cases["solve_f32"] = _solve_case("a1mpc_solve_batch", prec=32)
    cases["solve_optional_null"] = _solve_case("a1mpc_solve_batch", optional=False)
    cases["solve_warm"] = _solve_case("a1mpc_solve_batch_warm", warm=True)
    cases["solve_ext"] = _solve_case("a1mpc_solve_batch_ext", ext=True)
    cases["solve_ext_ld"] = _solve_case("a1mpc_solve_batch_ext", ld_in=LD_IN, ld_out=LD_OUT, ext=True)
    cases["solve_ext_f32"] = _solve_case("a1mpc_solve_batch_ext", prec=32, ext=True)
    cases["solve_ext_warm"] = _solve_case("a1mpc_solve_batch_ext_warm", ext=True, warm=True)
    cases["solve_ext_warm_ld"] = _solve_case("a1mpc_solve_batch_ext_warm", ld_in=LD_IN, ld_out=LD_OUT, ext=True, warm=True)

    n, m, H, g, contact = _dense_arrays(rng)
    states = a1mpc.gen_states(B, 2, 5)
    cases["build_qp"] = Case(dict({k: ("in", v) for k, v in states.items()}, H=("out", np.zeros((B, n, n))), g=("out", np.zeros((B, n))), lb=("out", np.zeros((B, m))),
                                  ub=("out", np.zeros((B, m)))),
                             lambda a1, eng, p: a1.lib().a1mpc_build_qp_batch(eng.h, B, C.byref(a1.Inputs(p["x0"], p["rot"], p["foot"], p["ref"], p["contact"], B)),
                                                                              p.get("H"), p.get("g"), p.get("lb"), p.get("ub")))
    model = dict(A_d=("in", np.eye(13) + 0.1 * rng.standard_normal((B, 13, 13))), B_d_list=("in", rng.standard_normal((B, 13 * N, 12))),
                 x0=("in", rng.standard_normal((B, 13))), x_d=("in", rng.standard_normal((B, 13 * N))))
    mats = dict(H=("out", np.zeros((B, n, n))), g=("out", np.zeros((B, n))))
    cases["qp_mats"] = Case(dict(model, **mats), lambda a1, eng, p: a1.lib().a1mpc_qp_mats_batch(eng.h, B, p["A_d"], p["B_d_list"], p["x0"], p["x_d"],
                                                                                                   p.get("H"), p.get("g")))
    cases["qp_rollout"] = Case(dict(model, A_qp=("out", np.zeros((B, 13 * N, 13))), B_qp=("out", np.zeros((B, 13 * N, n))), **mats),
                               lambda a1, eng, p: a1.lib().a1mpc_qp_rollout_batch(eng.h, B, p["A_d"], p["B_d_list"], p["x0"], p["x_d"], p.get("A_qp"),
                                                                                  p.get("B_qp"), p.get("H"), p.get("g")))
    cases["solve_dense"] = Case(dict(H=("in", H), g=("in", g), contact=("in", contact), u=("out", np.zeros((B, n))),
                                     status=("out", np.full(B, -7, dtype=np.int32))),
                                lambda a1, eng, p: a1.lib().a1mpc_solve_dense_batch(eng.h, B, p["H"], p["g"], p["contact"], p["u"], p["status"]))
    yaw = rng.uniform(-3, 3, B)
    rot_z = np.stack([np.cos(yaw), -np.sin(yaw), 0 * yaw, np.sin(yaw), np.cos(yaw), 0 * yaw, 0 * yaw, 0 * yaw, 1 + 0 * yaw])
    acc = np.stack([rng.normal(0, 20, B), rng.normal(0, 20, B), 12 * 9.8 + rng.normal(0, 30, B), rng.normal(0, 5, B), rng.normal(0, 5, B),
                    rng.normal(0, 2, B)], axis=1)
    cases["grf_qp"] = Case(dict(root_acc=("in", acc), rot_z=("in", rot_z.T.copy()), rot=("in", states["rot"].T.copy()), foot=("in", states["foot"].T.copy()),
                                contact=("in", contact), f_body=("out", np.zeros((B, 12))), status=("out", np.full(B, -7, dtype=np.int32))),
                           lambda a1, eng, p: a1.lib().a1mpc_grf_qp_batch(eng.h, B, p["root_acc"], p["rot_z"], p["rot"], p["foot"], p["contact"],
                                                                          p["f_body"], p["status"]))
    jac = (0.2 * np.eye(3).reshape(1, 3, 3, 1) + 0.15 * rng.standard_normal((4, 3, 3, B))).reshape(36, B)
    f_kin = 30.0 * rng.standard_normal((12, B))
    f_kin[4, 7] = np.nan                      # that torque keeps its previous value
    cases["joint_torques"] = Case(dict(f_grf=("in", 50 * rng.standard_normal((12, B))), f_kin=("in", f_kin), jac=("in", jac), contact=("in", contact),
                                       tau=("out", rng.standard_normal((12, B)))),
                                  lambda a1, eng, p: a1.lib().a1mpc_joint_torques_batch(eng.h, B, p["f_grf"], p["f_kin"], p["jac"], p["contact"],
                                                                                        p["km_foot"], p["torques_gravity"], p["tau"]),
                                  params=dict(km_foot=np.array([0.1, 0.1, 0.1]), torques_gravity=np.array([0.8, 0, 0, -0.8, 0, 0, 0.8, 0, 0, -0.8, 0, 0])))

    gp = a1mpc.default_gait_params(N)
    plan_in = dict(gait_counter=("out", rng.uniform(0, 240, (4, B))), gait_counter_speed=("in", rng.choice([1.4, 1.5, 2.0], (4, B))),
                   movement_mode=("in", (rng.uniform(size=B) < 0.8).astype(np.uint32)), lin_vel=("in", rng.normal(0, 0.5, (3, B))),
                   lin_vel_d=("in", rng.normal(0, 0.5, (3, B))), rot_z=("in", rot_z), rot=("in", states["rot"]), root_pos=("in", rng.normal(0, 1, (3, B))))

    def plan_call(a1, eng, p):
        return a1.lib().a1mpc_update_plan_batch(eng.h, B, C.byref(gp), p["gait_counter"], p["gait_counter_speed"], p["movement_mode"], p.get("lin_vel"),
                                                p.get("lin_vel_d"), p.get("rot_z"), p.get("rot"), p.get("root_pos"), p["plan_contacts"], p.get("contact_sched"),
                                                p.get("t_rel"), p.get("t_abs"), p.get("t_world"))
    plan_out = dict(plan_contacts=("out", np.zeros(B, dtype=np.uint32)))
    cases["update_plan"] = Case(dict(plan_in, contact_sched=("out", np.zeros((N, B), dtype=np.uint32)), t_rel=("out", np.zeros((12, B))),
                                     t_abs=("out", np.zeros((12, B))), t_world=("out", np.zeros((12, B))), **plan_out), plan_call)
    # no foothold output: the foothold inputs are not copied, but their side is still checked
    cases["update_plan_optional_null"] = Case(dict(plan_in, **plan_out), plan_call)

    _, rho_opt, rho_fix, q, dq, rot = estimation_scenario(B, 5)
    cases["leg_kinematics"] = Case(dict(joint_pos=("in", q), joint_vel=("in", dq), rot=("in", rot), foot_pos_rel=("out", np.zeros((12, B))),
                                        jac=("out", np.zeros((36, B))), foot_vel_rel=("out", np.zeros((12, B))), foot_pos_abs=("out", np.zeros((12, B))),
                                        foot_vel_abs=("out", np.zeros((12, B)))),
                                   lambda a1, eng, p: a1.lib().a1mpc_leg_kinematics_batch(eng.h, B, p["joint_pos"], p.get("joint_vel"), p.get("rot"), p["rho_opt"],
                                                                                          p["rho_fix"], p.get("foot_pos_rel"), p.get("jac"), p.get("foot_vel_rel"),
                                                                                          p.get("foot_pos_abs"), p.get("foot_vel_abs")),
                                   params=dict(rho_opt=rho_opt.reshape(12).copy(), rho_fix=rho_fix.reshape(20).copy()))
    fpr = np.tile(np.array([0.18, -0.13, -0.3, 0.18, 0.13, -0.3, -0.18, -0.13, -0.3, -0.18, 0.13, -0.3])[:, None], (1, B)) + rng.normal(0, 0.02, (12, B))

    def ekf_state(a1, eng, p):
        s = eng.ekf_alloc(B)
        a1._check(a1.lib().a1mpc_ekf_init_batch(eng.h, B, s, fpr.ctypes.data, rot.ctypes.data))
        return s, a1.lib().a1mpc_ekf_bytes(B)
    cases["ekf_init"] = Case(dict(foot_pos_rel=("in", fpr), rot=("in", rot)),
                             lambda a1, eng, p: a1.lib().a1mpc_ekf_init_batch(eng.h, B, p["state"], p["foot_pos_rel"], p["rot"]),
                             state=lambda a1, eng, p: (_h2d(a1, eng, np.zeros(a1.lib().a1mpc_ekf_bytes(B), dtype=np.uint8)), a1.lib().a1mpc_ekf_bytes(B)))
    cases["ekf_update"] = Case(dict(movement_mode=("in", np.ones(B, dtype=np.uint32)), imu_acc=("in", rng.normal([0, 0, 9.8], 0.5, (B, 3)).T.copy()),
                                    imu_ang_vel=("in", rng.normal(0, 0.3, (3, B))), rot=("in", rot), foot_pos_rel=("in", fpr),
                                    foot_vel_rel=("in", rng.normal(0, 0.2, (12, B))), foot_force=("in", rng.uniform(0, 80, (4, B))),
                                    root_pos=("out", np.zeros((3, B))), root_lin_vel=("out", np.zeros((3, B))),
                                    estimated_contacts=("out", np.zeros(B, dtype=np.uint32)), status=("out", np.full(B, -7, dtype=np.int32))),
                               lambda a1, eng, p: a1.lib().a1mpc_ekf_update_batch(eng.h, B, p["state"], C.c_double(DT), 0, p["movement_mode"], p["imu_acc"],
                                                                                  p["imu_ang_vel"], p["rot"], p["foot_pos_rel"], p["foot_vel_rel"], p["foot_force"],
                                                                                  p.get("root_pos"), p.get("root_lin_vel"), p.get("estimated_contacts"),
                                                                                  p.get("status")),
                               state=ekf_state)

    fabs = np.einsum("ijb,ljb->lib", rot.reshape(3, 3, B), fpr.reshape(4, 3, B)).reshape(12, B).copy()
    legs = dict(gait_counter=("in", rng.uniform(0, 240, (4, B))), plan_contacts=("in", rng.integers(0, 16, B).astype(np.uint32)), rot_z=("in", rot_z),
                foot_pos_abs=("in", fabs), foot_pos_target_rel=("in", fpr + rng.normal(0, 0.03, (12, B))), foot_force=("in", rng.uniform(0, 80, (4, B))))

    def legs_call(a1, eng, p):
        return a1.lib().a1mpc_swing_legs_batch(eng.h, B, C.byref(gp), p["kp_foot"], p["kd_foot"], p["state"], C.c_double(DT), p["gait_counter"],
                                               p["plan_contacts"], p["rot_z"], p["foot_pos_abs"], p["foot_pos_target_rel"], p["foot_force"], p["f_kin"],
                                               p["contacts"], p.get("foot_pos_cur"), p.get("foot_pos_recent_contact"))
    gains = dict(kp_foot=KP_RESET.copy(), kd_foot=KD_RESET.copy())

    def swing_state(a1, eng, p):
        s = eng.swing_alloc(B)
        host = {k: v.ctypes.data for k, (_, v) in legs.items()}
        scratch = [np.zeros((12, B)), np.zeros(B, dtype=np.uint32), np.zeros((12, B)), np.zeros((12, B))]
        host.update(zip(("f_kin", "contacts", "foot_pos_cur", "foot_pos_recent_contact"), (a.ctypes.data for a in scratch)))
        host.update({k: v.ctypes.data for k, v in gains.items()}, state=s.value)
        assert legs_call(a1, eng, host) == 0, a1.lib().a1mpc_last_error()    # one tick: the recent-contact filters hold points
        return s, a1.lib().a1mpc_swing_bytes(B)
    cases["swing_legs"] = Case(dict(legs, f_kin=("out", np.zeros((12, B))), contacts=("out", np.zeros(B, dtype=np.uint32)),
                                    foot_pos_cur=("out", np.zeros((12, B))), foot_pos_recent_contact=("out", np.zeros((12, B)))),
                               legs_call, params=gains, state=lambda a1, eng, p: (eng.swing_alloc(B), a1.lib().a1mpc_swing_bytes(B)))
    root_pos = np.stack([rng.normal(0, 1, B), rng.normal(0, 1, B), rng.uniform(0.2, 0.35, B)])

    def terrain(adapt, ld):
        return lambda a1, eng, p: a1.lib().a1mpc_terrain_pitch_batch(eng.h, B, p["state"], adapt, p["root_pos"], p.get("ref"), ld, p.get("terrain_pitch"))
    for name, adapt, ld, pitch in (("terrain_pitch", 1, B, True), ("terrain_pitch_ld", 1, LD_IN, True), ("terrain_pitch_optional_null", 1, B, False),
                                   ("terrain_pitch_no_adapt", 0, B, True)):
        arrs = dict(root_pos=("in", root_pos), ref=("out", np.full((9, ld), 5.0)))
        if pitch:
            arrs["terrain_pitch"] = ("out", np.full(B, 9.0))
        cases[name] = Case(arrs, terrain(adapt, ld), state=swing_state)
    return cases


NAMES = ["solve", "solve_ld", "solve_f32", "solve_optional_null", "solve_warm", "solve_ext", "solve_ext_ld", "solve_ext_f32", "solve_ext_warm",
         "solve_ext_warm_ld", "build_qp", "qp_mats", "qp_rollout", "solve_dense", "grf_qp", "joint_torques", "update_plan",
         "update_plan_optional_null", "leg_kinematics", "ekf_init", "ekf_update", "swing_legs", "terrain_pitch", "terrain_pitch_ld",
         "terrain_pitch_optional_null", "terrain_pitch_no_adapt"]
# the mixed-pointer rows run on one case per entry point, plus the cases with a batch array the call does not read
ENTRY = ["solve", "solve_warm", "solve_ext", "solve_ext_warm", "build_qp", "qp_mats", "qp_rollout", "solve_dense", "grf_qp", "joint_torques",
         "update_plan", "update_plan_optional_null", "leg_kinematics", "ekf_init", "ekf_update", "swing_legs", "terrain_pitch", "terrain_pitch_no_adapt"]
WITH_HOST_PARAMS = {"joint_torques", "leg_kinematics", "swing_legs"}


@pytest.fixture(scope="module")
def cases(a1):
    c = _cases()
    assert list(c) == NAMES
    return c


def _h2d(a1, eng, x):
    d = eng.dalloc(max(x.nbytes, 8))
    a1._check(a1.lib().a1mpc_memcpy_h2d(eng.h, d, x.ctypes.data, x.nbytes))
    return d


def _d2h(a1, eng, d, like):
    x = np.empty_like(like)
    a1._check(a1.lib().a1mpc_memcpy_d2h(eng.h, x.ctypes.data, d, x.nbytes))
    eng.sync()
    return x


class Call:
    """one call of a case: each array on the side on_device(name) says, each parameter on the side param_on_device(name) says"""

    def __init__(self, a1, eng, case, on_device=lambda name: False, param_on_device=lambda name: False):
        self.a1, self.eng, self.case = a1, eng, case
        self.host = {k: v.copy() for k, (_, v) in case.arrays.items()}
        self.dev = {k: _h2d(a1, eng, v) for k, v in self.host.items() if on_device(k)}
        self.pdev = {k: _h2d(a1, eng, v) for k, v in case.params.items() if param_on_device(k)}
        self.p = {k: (self.dev[k].value if k in self.dev else v.ctypes.data) for k, v in self.host.items()}
        self.p.update({k: (self.pdev[k].value if k in self.pdev else v.ctypes.data) for k, v in case.params.items()})
        self.state = None
        if case.state:
            primer = {k: v.copy() for k, (_, v) in case.arrays.items()}
            primer_p = {k: v.ctypes.data for k, v in primer.items()}
            primer_p.update({k: v.ctypes.data for k, v in case.params.items()})
            self.state, self.state_bytes = case.state(a1, eng, primer_p)
            self.p["state"] = self.state.value
        eng.sync()

    def __call__(self):
        return self.case.call(self.a1, self.eng, self.p)

    def results(self):
        out = {k: (_d2h(self.a1, self.eng, self.dev[k], v) if k in self.dev else v) for k, v in self.host.items() if self.case.arrays[k][0] == "out"}
        if self.state is not None:
            out["state"] = _d2h(self.a1, self.eng, self.state, np.zeros(self.state_bytes, dtype=np.uint8))
        return out

    def free(self):
        for d in list(self.dev.values()) + list(self.pdev.values()) + ([self.state] if self.state is not None else []):
            self.a1.lib().a1mpc_device_free(self.eng.h, d)


@pytest.mark.parametrize("name", NAMES)
def test_host_and_device_arrays_give_the_same_results(a1, engines, cases, name):
    case = cases[name]
    eng = engines(case.prec)
    res, launches = {}, {}
    for side in ("host", "device"):
        call = Call(a1, eng, case, on_device=lambda k: side == "device")
        n0 = eng.launches()
        assert call() == 0, (side, a1.lib().a1mpc_last_error())
        eng.sync()
        launches[side] = eng.launches() - n0
        res[side] = call.results()
        call.free()
    assert launches["host"] == launches["device"] > 0
    for k, h in res["host"].items():
        assert np.array_equal(h, res["device"][k], equal_nan=h.dtype.kind == "f"), k
    if "status" in res["host"] and name.startswith("solve") and name != "solve_dense":
        assert (res["host"]["status"] == a1.STATUS_OPTIMAL).mean() > 0.5      # the solve cases solve real problems
    if name.endswith("_ld"):                                                  # ld > B: the columns past B are the caller's
        for k, (role, v) in case.arrays.items():
            if role == "out" and v.shape[-1] > B:
                assert np.array_equal(res["host"][k][..., B:], v[..., B:]), k


def _rows():
    for name in ENTRY:
        yield name, "one_host_among_device"
        yield name, "one_device_among_host"
        if name != "ekf_init":       # (no outputs)
            yield name, "inputs_device_outputs_host"
        if name in WITH_HOST_PARAMS:
            yield name, "host_param_on_device"


@pytest.mark.parametrize("name,mix", list(_rows()))
def test_mixed_sides_are_rejected_before_anything_is_enqueued(a1, engines, cases, name, mix):
    case = cases[name]
    eng = engines(case.prec)
    L = a1.lib()
    if mix == "host_param_on_device":
        variants = [dict(param_on_device=lambda k, odd=odd: k == odd) for odd in case.params]
    elif mix == "one_host_among_device":
        variants = [dict(on_device=lambda k, odd=odd: k != odd) for odd in case.arrays]
    elif mix == "one_device_among_host":
        variants = [dict(on_device=lambda k, odd=odd: k == odd) for odd in case.arrays]
    else:
        variants = [dict(on_device=lambda k: case.arrays[k][0] == "in")]
    for v in variants:
        call = Call(a1, eng, case, **v)
        n0 = eng.launches()
        assert call() == -1
        msg = L.a1mpc_last_error()
        assert (b"host array" if mix == "host_param_on_device" else b"all-host or all-device") in msg, msg
        assert eng.launches() == n0
        for k, (role, init) in case.arrays.items():
            if role == "out" and k not in call.dev:
                assert np.array_equal(call.host[k], init, equal_nan=True), k
        call.free()
        # the handle is still healthy
        st = a1.gen_states(32, 2, 64)
        f, s, _ = eng.solve(st)
        assert (s == 0).all()
