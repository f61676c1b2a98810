import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "a1-qp-mpc-controller_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def built():
    """the shared libraries must exist AND be up to date.  In the development container (no GPU) `make` runs every time -- a no-op
    when nothing changed; a stale liba1mpc.so after an edit of a header used to pass the GPU tests happily.  On a GPU box the
    libraries shipped with the snapshot are used as they are (build/ does not travel, so `make` there would recompile everything
    on charged GPU time); only a missing library is built."""
    import subprocess
    have = os.path.exists(os.path.join(ROOT, "a1-qp-mpc-controller_b200", "liba1mpc.so")) and os.path.exists(os.path.join(ROOT, "oracle", "liba1mpc_oracle.so"))
    if not have or not os.path.exists("/dev/nvidia0"):
        subprocess.check_call(["make", "-C", ROOT, "-j8", "-s", "all"])
    return True


@pytest.fixture(scope="session")
def gpu_engine(built):
    import a1mpc
    eng = a1mpc.Engine(a1mpc.default_config(), device=0)
    yield eng
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# A1MPC_EMU_ENGINE=1: replay the solver-dependent `-m gpu` tests on the CPU emulator (tests/emu) -- a development aid for
# machines without a GPU (every algorithmic change of the kernels is replayed against the exact inputs of the GPU suite
# before it is committed).  The real GPU suite never sets this variable.
#     A1MPC_EMU_ENGINE=1 python -m pytest tests/test_gpu_parity.py -m gpu -q
# ---------------------------------------------------------------------------------------------------------------------
_EMU_SKIP = {"test_p0_build_parity", "test_p0_build_parity_n20", "test_ragged_ld_and_device_pointers", "test_qp_mats_general_rollout",
             "test_joint_torques_next_row", "test_update_plan_previous_row", "test_fp64_peak_probe_and_profile_api",
             "test_cpp_shims_mirror_of_test_mpc", "test_warm_start_argument_errors", "test_leg_kinematics_batch_chains_into_the_solver",
             "test_compact_schedule_class_matches_oracle_and_general_kernel",
             "test_gpu_certified_means_optimal_every_qp_checked"}   # (65 536 QPs: its emulator twin is in test_emu.py)


def pytest_collection_modifyitems(config, items):
    if os.environ.get("A1MPC_EMU_ENGINE") != "1":
        return
    skip = pytest.mark.skip(reason="needs the real C ABI / GPU (not covered by the emulator replay)")
    for it in items:
        if it.name.split("[")[0] in _EMU_SKIP:
            it.add_marker(skip)


if os.environ.get("A1MPC_EMU_ENGINE") == "1":
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import ctypes as _C

    import a1mpc as _a1probe
    if _a1probe.lib().a1mpc_device_count() > 0:
        # never let the replay stand in for the real thing: with a GPU present the `-m gpu` suite must run the CUDA library
        raise pytest.UsageError("A1MPC_EMU_ENGINE=1 is a CPU-only development aid; a CUDA device is visible -- unset it")

    import numpy as _np

    import a1mpc as _a1
    import emu_py as _E
    from oracle import oracle_py as _O

    class _EmuEngine:
        """the subset of a1mpc.Engine the solver-dependent tests use, on the emulator (build_qp: the oracle's dense build)"""

        def __init__(self, cfg=None, device=0):
            self.cfg = cfg if cfg is not None else _a1.default_config()
            self.h = None

        def close(self):
            pass

        def _ocfg(self):
            c = self.cfg
            return _O.make_config(horizon=c.horizon, dt=c.dt, mu=c.mu, fz_max=c.fz_max, mass=c.mass, inertia=tuple(c.inertia), q=tuple(c.q), r=tuple(c.r))

        def solve(self, st, want_u=False):
            res = _E.solve(self.cfg, st, want_u=want_u, order=2)
            return res[:-1]

        def solve_ext(self, st, sched=None, normals=None, want_u=False):
            if normals is not None:
                r = list(self.cfg.r)
                if any(r[3 * i] != r[3 * i + 1] or r[3 * i] != r[3 * i + 2] for i in range(4)):
                    raise _a1.A1MpcError("terrain normals need isotropic r weights per foot")
            res = _E.solve(self.cfg, st, sched=sched, normals=normals, want_u=want_u, order=2)
            return res[:-1]

        def solve_ptrs(self, B, inp, out):
            if B <= 0:
                raise _a1.A1MpcError("B must be positive")
            raise NotImplementedError

        def build_qp(self, st):
            ob = _O.Batch(st["x0"], st["rot"], st["foot"], st["ref"], st["contact"])
            parts = [_O.build_qp(self._ocfg(), ob, b) for b in range(ob.B)]
            return tuple(_np.stack([p[i] for p in parts]) for i in (0, 1, 3, 4))

        def solve_dense(self, H, g, contact):
            return _E.solve_dense(self.cfg, H, g, contact, order=2)

        def grf_qp(self, root_acc, rot_z, rot, foot, contact):
            return _E.grf_qp(root_acc, rot_z, rot, foot, contact, order=2)

        def warm_alloc(self, B):
            return _np.zeros((B, 4 + 4 * self.cfg.horizon), dtype=_np.uint32)

        def solve_warm(self, st, warm, shift=0):
            if self.cfg.horizon != 10:
                raise _a1.A1MpcError("warm start is implemented for horizon 10")
            return _E.solve(self.cfg, st, warm=warm, shift=shift, order=2)[:-1]

        def leg_kinematics(self, joint_pos, joint_vel, rot, rho_opt, rho_fix):
            return _E.leg_kinematics(joint_pos, joint_vel, rot, rho_opt, rho_fix)

        def ekf_alloc(self, B):
            return {"B": B}

        def ekf_init(self, ekf, foot_pos_rel, rot):
            ekf["s"] = _E.ekf_init(foot_pos_rel, rot)

        def ekf_update(self, ekf, dt, flat, mode, acc, gyro, rot, fpr, fvr, force):
            return _E.ekf_update(ekf["s"], dt, flat, mode, acc, gyro, rot, fpr, fvr, force, order=2)

        def ekf_state(self, ekf, B):
            return ekf["s"][:, :18].copy(), ekf["s"][:, 18:].reshape(B, 18, 18).copy()

    class _EmuLib:
        """a1mpc.lib() stand-in for the two raw calls the warm-start test makes"""

        def __getattr__(self, name):
            return getattr(_REAL_LIB, name)

        def a1mpc_warm_reset(self, h, warm, B):
            warm[:] = 0
            return 0

    _REAL_LIB = _a1.lib()
    _a1.Engine = _EmuEngine
    _a1.lib = lambda: _EmuLib()
