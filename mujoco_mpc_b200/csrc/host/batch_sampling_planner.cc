// batch_sampling_planner.cc - see batch_sampling_planner.h.  Compiled into libmjpc_b200.so next to the engine.
#include "batch_sampling_planner.h"

namespace mjpc_b200_host {

int BatchSamplingPlanner::Initialize(const mjpc_model_blob* model, int num_problems, int num_trajectory,
                                     int num_spline_points, int interpolation, double exploration, double timestep,
                                     const double* ctrlrange, const uint32_t* seeds, int max_horizon, int device) {
  if (num_problems < 1 || num_trajectory < 1) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (int rc = Attach(model, num_problems, num_problems * num_trajectory, max_horizon, device)) return rc;
  for (int b = 0; b < num_problems; b++) {
    auto* p = new SamplingPlanner;
    problems_.emplace_back(p);
    if (int rc = p->Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, 0.0, timestep,
                               ctrlrange, seeds[b], num_trajectory, max_horizon, device, gpu_))
      return rc;
  }
  return 0;
}

int BatchSamplingPlanner::OptimizePolicy(int horizon) {
  const int B = NumProblems();
  // per problem, as SamplingPlanner::OptimizePolicyCandidates up to its launch
  std::vector<const SplineCandidates*> cands(B);
  for (int b = 0; b < B; b++) cands[b] = &planner(b).PrepareOptimize(horizon);
  if (int rc = LaunchSpline(gpu_, cands, horizon)) return rc;
  // per problem, as SamplingPlanner::OptimizePolicy after its launch
  const int N = cands[0]->N;
  for (int b = 0; b < B; b++) {
    const size_t o = (size_t)b * N;
    planner(b).InstallRollouts(N, horizon, returns_.data() + o, failure_.data() + o, order_.data() + o, (int)o);
    planner(b).InstallBest();
  }
  return 0;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
// (the calls every batch kind shares are in batch_planner.cc)
using mjpc_b200_host::BatchPlanner;
using mjpc_b200_host::BatchSamplingPlanner;

extern "C" {

int mjpc_b200_batch_planner_create(const mjpc_model_blob* model, int num_problems, int num_trajectory, int num_spline_points,
                                   int interpolation, double exploration, double timestep, const double* ctrlrange,
                                   const uint32_t* seeds, int max_horizon, int device, void** out) {
  if (!model || !model->data || !ctrlrange || !seeds || !out) return MJPC_B200_ERR_BAD_ARGUMENT;
  *out = nullptr;
  auto* p = new BatchSamplingPlanner;
  int rc = p->Initialize(model, num_problems, num_trajectory, num_spline_points, interpolation, exploration, timestep,
                         ctrlrange, seeds, max_horizon, device);
  if (rc) { delete p; return rc; }
  *out = static_cast<BatchPlanner*>(p);
  return 0;
}
// sampling batches only: another kind is refused
int mjpc_b200_batch_planner_get_result(void* p, int problem, int* winner, double* improvement, float* returns,
                                       double* knots, double* knot_times) {
  auto* bp = dynamic_cast<BatchSamplingPlanner*>(reinterpret_cast<BatchPlanner*>(p));
  if (!bp || problem < 0 || problem >= bp->NumProblems()) return MJPC_B200_ERR_BAD_ARGUMENT;
  return mjpc_b200_sampling_planner_get_result(mjpc_b200_host::ToHandle(&bp->planner(problem)), winner, improvement,
                                               returns, knots, knot_times);
}

}  // extern "C"
