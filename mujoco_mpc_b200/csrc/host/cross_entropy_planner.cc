// cross_entropy_planner.cc - see cross_entropy_planner.h.  Reference: mjpc/planners/cross_entropy/planner.cc.
#include "cross_entropy_planner.h"

#include <algorithm>
#include <cmath>
#include <mutex>
#include <numeric>

namespace mjpc_b200_host {

int CrossEntropyPlanner::Initialize(const mjpc_model_blob* model, int num_trajectory, int n_elite, int num_spline_points,
                                    int interpolation, double std_initial, double std_min, double explore_fraction,
                                    double timestep, const double* ctrlrange, uint32_t seed, int max_horizon, int device,
                                    mjpc_b200_t* engine) {
  // N noisy candidates + the nominal trajectory share one launch
  if (int rc = AttachEngine(model, num_trajectory + 1, max_horizon, device, engine)) return rc;
  nu_ = info_.nu;
  num_trajectory_ = num_trajectory;
  n_elite_ = n_elite > 0 ? n_elite : std::max(num_trajectory / 10, 2);   // planner.cc:69-71
  interpolation_ = (SplineInterpolation)interpolation;
  std_initial_ = std_initial; std_min_ = std_min; explore_fraction_ = explore_fraction;
  timestep_ = timestep; seed_ = seed;
  policy.plan = TimeSpline(nu_, interpolation_);
  policy.num_spline_points = num_spline_points;
  policy.ctrlrange.assign(ctrlrange, ctrlrange + 2 * nu_);
  resampled_policy = policy; previous_policy = policy;
  candidate_policy.assign(num_trajectory, policy);
  returns_.assign(num_trajectory + 1, 0.f); failure_.assign(num_trajectory + 1, 0);
  trajectory_order.resize(num_trajectory);
  std::iota(trajectory_order.begin(), trajectory_order.end(), 0);
  Reset(max_horizon, nullptr);
  return 0;
}

void CrossEntropyPlanner::Reset(int, const double* initial_repeated_action) {
  policy.plan.Clear();
  if (initial_repeated_action) policy.plan.AddNode(0, initial_repeated_action);
  resampled_policy = policy; previous_policy = policy;
  for (auto& cp : candidate_policy) cp = policy;
  variance.assign((size_t)policy.num_spline_points * nu_, std_initial_ * std_initial_);
  times_scratch_.assign(policy.num_spline_points, 0.0);
  improvement = 0; iteration = 0;
}

void CrossEntropyPlanner::ResamplePolicy(int horizon) {
  const int P = resampled_policy.num_spline_points;
  double nominal_time = time_;
  const double time_shift = std::max((horizon - 1) * timestep_ / (P - 1), 1.0e-5);
  TimeSpline scratch(nu_, policy.plan.Interpolation());
  std::vector<double> v(nu_);
  for (int t = 0; t < P; t++) {
    times_scratch_[t] = nominal_time;
    resampled_policy.Action(v.data(), nominal_time);
    scratch.AddNode(nominal_time, v.data());
    nominal_time += time_shift;
  }
  resampled_policy.plan = scratch;
}

void CrossEntropyPlanner::AddNoiseToPolicy(int i, double std_min) {
  TimeSpline& plan = candidate_policy[i].plan;
  for (int k = 0; k < plan.Size(); k++) {
    double* node = plan.NodeValues(k);
    for (int d = 0; d < nu_; d++) {
      const double sd = std::max(std::sqrt(variance[(size_t)k * nu_ + d]), std_min);
      node[d] += sd * PhiloxNormal(seed_, (uint32_t)iteration, (uint32_t)i, (uint32_t)k, (uint32_t)d);
      node[d] = std::max(policy.ctrlrange[2 * d], std::min(policy.ctrlrange[2 * d + 1], node[d]));
    }
  }
}

const SplineCandidates& CrossEntropyPlanner::PrepareCandidates(int horizon) {
  resampled_policy.plan.SetInterpolation(interpolation_);
  const int num_trajectory = num_trajectory_;
  n_elite_ = std::min(n_elite_, num_trajectory);
  {
    const std::shared_lock<std::shared_mutex> lock(mtx_);
    resampled_policy = policy;
  }
  resampled_policy.plan.SetInterpolation(interpolation_);
  ResamplePolicy(horizon);
  // Rollouts (:414-459): the N noisy candidates, then the nominal as candidate N (NominalTrajectory, :295-307)
  const int P = resampled_policy.plan.Size();
  cands_.Resize(num_trajectory + 1, P, nu_);
  cands_.interpolation = (int)interpolation_;
  for (int i = 0; i <= num_trajectory; i++) {
    const SamplingPolicy* src = &resampled_policy;
    if (i < num_trajectory) {
      const double std = i < num_trajectory * explore_fraction_ ? std_initial_ : std_min_;
      candidate_policy[i] = resampled_policy;
      AddNoiseToPolicy(i, std);
      src = &candidate_policy[i];
    }
    for (int k = 0; k < P; k++) {
      const double* node = src->plan.NodeValues(k);
      for (int d = 0; d < nu_; d++) cands_.knots[((size_t)i * P + k) * nu_ + d] = (float)node[d];
    }
  }
  std::copy(times_scratch_.begin(), times_scratch_.begin() + P, cands_.knot_times.begin());
  return cands_;
}

int CrossEntropyPlanner::Iterate(const std::vector<CrossEntropyPlanner*>& ps, const TaskRows& rows, int horizon,
                                 SplineLaunch* launch) {
  std::vector<const SplineCandidates*> cands;
  for (CrossEntropyPlanner* p : ps) cands.push_back(&p->PrepareCandidates(horizon));
  if (int rc = launch->Run(std::vector<const Planner*>(ps.begin(), ps.end()), cands, rows, horizon)) return rc;
  const int N1 = cands[0]->N;
  for (size_t b = 0; b < ps.size(); b++) {
    const size_t o = b * N1;
    ps[b]->InstallRollouts(horizon, launch->returns.data() + o, launch->failure.data() + o, launch->order.data() + o,
                           (int)o);
  }
  return 0;
}

int CrossEntropyPlanner::OptimizePolicy(int horizon) {
  return Iterate({this}, TaskRows(), horizon, &launch_) ? -1 : 0;
}

void CrossEntropyPlanner::InstallRollouts(int horizon, const float* returns, const uint8_t* failure, const int* order,
                                          int offset) {
  const int num_trajectory = num_trajectory_, n_elite = n_elite_;
  std::copy(returns, returns + num_trajectory + 1, returns_.begin());
  std::copy(failure, failure + num_trajectory + 1, failure_.begin());
  launch_offset_ = offset; horizon_ = horizon;
  // the device ranked all N+1 launches; the elite ranking is over the N noisy candidates only (:181-193)
  int r = 0;
  for (int k = 0; k <= num_trajectory; k++) if (order[k] < num_trajectory) trajectory_order[r++] = order[k];
  const int P = resampled_policy.num_spline_points, num_parameters = P * nu_;
  std::vector<double> mean(num_parameters, 0.0);
  double avg_return = 0;
  for (int e = 0; e < n_elite; e++) {
    const int idx = trajectory_order[e];
    const TimeSpline& plan = candidate_policy[idx].plan;
    for (int t = 0; t < P; t++)
      for (int j = 0; j < nu_; j++) mean[(size_t)t * nu_ + j] += plan.NodeValues(t)[j];
    avg_return += returns_[idx];
  }
  for (double& x : mean) x /= n_elite;
  avg_return /= n_elite;
  std::fill(variance.begin(), variance.end(), 0.0);
  for (int e = 0; e < n_elite; e++) {
    const TimeSpline& plan = candidate_policy[trajectory_order[e]].plan;
    for (int t = 0; t < P; t++)
      for (int j = 0; j < nu_; j++) {
        const double diff = plan.NodeValues(t)[j] - mean[(size_t)t * nu_ + j];
        variance[(size_t)t * nu_ + j] += diff * diff / (n_elite - 1);
      }
  }
  {
    const std::unique_lock<std::shared_mutex> lock(mtx_);
    policy.plan.Clear();
    policy.plan.SetInterpolation(interpolation_);
    for (int t = 0; t < P; t++) policy.plan.AddNode(times_scratch_[t], mean.data() + (size_t)t * nu_);
  }
  improvement = std::max(avg_return - (double)returns_[trajectory_order[0]], 0.0);
  iteration++;
}

void CrossEntropyPlanner::ActionFromPolicy(double* action, const double*, double time, bool use_previous) {
  const std::shared_lock<std::shared_mutex> lock(mtx_);
  (use_previous ? previous_policy : policy).Action(action, time);
}

const Trajectory* CrossEntropyPlanner::BestTrajectory() {
  if (FetchTrajectory(num_trajectory_, horizon_, &nominal_)) return nullptr;
  nominal_.total_return = returns_[num_trajectory_];
  nominal_.failure = failure_[num_trajectory_];
  return &nominal_;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::CrossEntropyPlanner;
using mjpc_b200_host::PlannerOf;

extern "C" {

int mjpc_b200_ce_planner_create(const mjpc_model_blob* model, int num_trajectory, int n_elite, int num_spline_points,
                                int interpolation, double std_initial, double std_min, double explore_fraction,
                                double timestep, const double* ctrlrange, uint32_t seed, int max_horizon, int device,
                                mjpc_b200_planner_t** out) {
  if (!model || !ctrlrange || !out || num_trajectory < 2 || num_spline_points < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  auto* p = new CrossEntropyPlanner;
  int rc = p->Initialize(model, num_trajectory, n_elite, num_spline_points, interpolation, std_initial, std_min,
                         explore_fraction, timestep, ctrlrange, seed, max_horizon, device);
  if (rc) { delete p; *out = nullptr; return rc; }
  *out = mjpc_b200_host::ToHandle(p);
  return 0;
}
// improvement, returns [N+1] (the last one is the nominal), elite order [N], installed policy knots/times, variance
int mjpc_b200_ce_planner_get_result(mjpc_b200_planner_t* h, double* improvement, float* returns, int* order,
                                    double* knots, double* knot_times, double* variance) {
  auto* p = PlannerOf<CrossEntropyPlanner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  if (improvement) *improvement = p->improvement;
  if (returns) std::copy(p->returns().begin(), p->returns().end(), returns);
  if (order) std::copy(p->trajectory_order.begin(), p->trajectory_order.end(), order);
  if (variance) std::copy(p->variance.begin(), p->variance.end(), variance);
  return p->policy.plan.Export(knots, knot_times);
}

}  // extern "C"
