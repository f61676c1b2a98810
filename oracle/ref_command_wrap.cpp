// oracle/ref_command_wrap.cpp -- TEST INFRASTRUCTURE.  Calls the REFERENCE'S OWN Utils::quat_to_euler (utils/Utils.cpp, compiled
// unmodified against the header stand-ins of oracle/ref_shim/) and its MovingWindowFilter (utils/filter.hpp), which
// `make -C oracle -f command.mk ref` builds into oracle/_ref/libref_command.so.  tests/test_command_ref_pin.py checks the oracle's
// restatement (command_oracle.cpp) against them bit for bit, and tests/golden/make_command_golden.py records them.
// Nothing here is product code; nothing under a1-qp-mpc-controller_b200/ may link it.
#include <Eigen/Dense>
#include "utils/Utils.h"
#include "utils/filter.hpp"

extern "C" {

// quat [4][n] (w, x, y, z as the adapters pass them to Quaterniond) -> euler [3][n]
int ref_quat_to_euler(int n, const double* quat, double* euler) {
  for (int b = 0; b < n; ++b) {
    const Eigen::Quaterniond q(quat[b], quat[n + b], quat[2 * n + b], quat[3 * n + b]);
    const Eigen::Vector3d e = Utils::quat_to_euler(q);
    for (int a = 0; a < 3; ++a) euler[a * n + b] = e[a];
  }
  return 0;
}

// one MovingWindowFilter(W) over T samples -> the T averages CalculateAverage returns
int ref_window(int W, int T, const double* x, double* y) {
  MovingWindowFilter f(W);
  for (int t = 0; t < T; ++t) y[t] = f.CalculateAverage(x[t]);
  return 0;
}

}  // extern "C"
