// Host build of the device expert policies (metaworld_b200/csrc/mw_policies.cuh) for the CPU tests: the same source the
// kernel k_expert runs, compiled by g++ with contraction off (-ffp-contract=off, as nvcc --fmad=false), so both builds
// round every operation as written.  Test infrastructure only.
#include "../../metaworld_b200/csrc/mw_policies.cuh"

// actions [n, 4] for the double observations obs [n, stride] (first 39 columns read) of tasks task_ids [n]
extern "C" void host_expert_actions(const int* task_ids, const double* obs, int stride, int n, float* actions) {
  for (int i = 0; i < n; i++) policy_action(task_ids[i], obs + (long)i * stride, actions + 4L * i);
}
