// sample_gradient_planner.cc - see sample_gradient_planner.h.  Reference: mjpc/planners/sample_gradient/planner.cc.
#include "sample_gradient_planner.h"

#include <algorithm>
#include <cmath>
#include <mutex>
#include <numeric>

namespace mjpc_b200_host {

int SampleGradientPlanner::Initialize(const mjpc_model_blob* model, int num_trajectory, int num_gradient,
                                      int num_spline_points, int interpolation, double exploration,
                                      double gradient_filter, double timestep, const double* ctrlrange, uint32_t seed,
                                      int max_horizon, int device, mjpc_b200_t* engine) {
  if (num_trajectory < 1 || num_spline_points < 2) return MJPC_B200_ERR_BAD_ARGUMENT;   // ResamplePolicy divides by P - 1
  // the nominal, the noisy samples and the gradient candidates share one launch
  if (int rc = AttachEngine(model, num_trajectory, max_horizon, device, engine)) return rc;
  nu_ = info_.nu;
  num_trajectory_ = num_trajectory;
  num_gradient_ = std::max(num_gradient, 0);
  interpolation_ = (SplineInterpolation)interpolation;
  noise_exploration_ = exploration; gradient_filter_ = gradient_filter;
  timestep_ = timestep; seed_ = seed;
  policy.plan = TimeSpline(nu_, interpolation_);
  policy.num_spline_points = num_spline_points;
  policy.ctrlrange.assign(ctrlrange, ctrlrange + 2 * nu_);
  candidate_policy.assign(num_trajectory, policy);
  returns_.assign(num_trajectory, 0.f); failure_.assign(num_trajectory, 0);
  trajectory_order.resize(num_trajectory);
  std::iota(trajectory_order.begin(), trajectory_order.end(), 0);
  Reset(max_horizon, nullptr);
  return 0;
}

void SampleGradientPlanner::Reset(int, const double* initial_repeated_action) {
  policy.plan.Clear();
  if (initial_repeated_action) policy.plan.AddNode(0, initial_repeated_action);
  resampled_policy = policy; previous_policy = policy;
  for (auto& cp : candidate_policy) { cp = policy; cp.plan.Clear(); }   // candidate_policy[i].Reset(horizon)
  const size_t num_parameters = (size_t)policy.num_spline_points * nu_;
  noise.assign((size_t)num_trajectory_ * num_parameters, 0.0);
  gradient.assign(num_parameters, 0.0); gradient_previous.assign(num_parameters, 0.0);
  improvement = 0; winner = 0; winner_type = kNominal; iteration = 0;
}

void SampleGradientPlanner::ResamplePolicy(SamplingPolicy& p, int horizon, int num_spline_points) {
  // shift = (H-1) dt / (P-1) for every interpolation: not the sampling planner's zero-spline rule
  double nominal_time = time_;
  const double time_shift = std::max((horizon - 1) * timestep_ / (num_spline_points - 1), 1.0e-5);
  TimeSpline scratch(nu_, p.plan.Interpolation());
  std::vector<double> v(nu_);
  knot_times_.resize(num_spline_points);
  for (int t = 0; t < num_spline_points; t++) {
    knot_times_[t] = nominal_time;
    p.Action(v.data(), nominal_time);                  // an empty plan samples to zeros (spline.cc:108-111), clamped
    scratch.AddNode(nominal_time, v.data());
    nominal_time += time_shift;
  }
  p.plan = scratch;
  p.num_spline_points = num_spline_points;
}

void SampleGradientPlanner::AddNoiseToPolicy(int i) {
  TimeSpline& plan = candidate_policy[i].plan;
  double* z = noise.data() + (size_t)i * policy.num_spline_points * nu_;
  for (int k = 0; k < plan.Size(); k++) {
    double* node = plan.NodeValues(k);
    for (int d = 0; d < nu_; d++) {
      z[k * nu_ + d] = PhiloxNormal(seed_, (uint32_t)iteration, (uint32_t)i, (uint32_t)k, (uint32_t)d);
      node[d] += z[k * nu_ + d] * noise_exploration_;
      node[d] = std::max(policy.ctrlrange[2 * d], std::min(policy.ctrlrange[2 * d + 1], node[d]));
    }
  }
}

const SplineCandidates& SampleGradientPlanner::PrepareCandidates(int horizon) {
  const int num_trajectory = num_trajectory_;
  num_gradient_ = std::min(num_gradient_, num_trajectory - 1);
  const int num_gradient = num_gradient_, num_noisy = num_trajectory - num_gradient;
  {
    const int P = policy.num_spline_points;
    {
      const std::shared_lock<std::shared_mutex> lock(mtx_);
      resampled_policy = policy;
    }
    // the reference sets the live policy's interpolation here, outside any lock; it is always interpolation_ in this
    // class, so setting it on the copy has the same effect without racing ActionFromPolicy
    resampled_policy.plan.SetInterpolation(interpolation_);
    ResamplePolicy(resampled_policy, horizon, P);
    for (int i = 0; i < num_gradient; i++) ResamplePolicy(candidate_policy[num_noisy + i], horizon, P);
  }
  // Rollouts (:358-398)
  const int P = resampled_policy.plan.Size();
  cands_.Resize(num_trajectory, P, nu_);
  cands_.interpolation = (int)interpolation_;
  for (int i = 0; i < num_trajectory; i++) {
    if (i < num_noisy) {                               // nominal and noisy candidates; gradient ones are ready
      candidate_policy[i] = resampled_policy;
      if (i > 0) AddNoiseToPolicy(i);
    }
    for (int k = 0; k < P; k++) {
      const double* node = candidate_policy[i].plan.NodeValues(k);
      for (int d = 0; d < nu_; d++) cands_.knots[((size_t)i * P + k) * nu_ + d] = (float)node[d];
    }
  }
  std::copy(knot_times_.begin(), knot_times_.begin() + P, cands_.knot_times.begin());
  return cands_;
}

int SampleGradientPlanner::Iterate(const std::vector<SampleGradientPlanner*>& ps, const TaskRows& rows, int horizon,
                                   SplineLaunch* launch) {
  std::vector<const SplineCandidates*> cands;
  for (SampleGradientPlanner* p : ps) cands.push_back(&p->PrepareCandidates(horizon));
  // the device ranks all N (lower index first on ties): replaces the partial_sort of OptimizePolicy (:219-229)
  if (int rc = launch->Run(std::vector<const Planner*>(ps.begin(), ps.end()), cands, rows, horizon)) return rc;
  const int N = cands[0]->N;
  for (size_t b = 0; b < ps.size(); b++) {
    const size_t o = b * N;
    ps[b]->InstallRollouts(horizon, launch->returns.data() + o, launch->failure.data() + o, launch->order.data() + o,
                           (int)o);
  }
  return 0;
}

int SampleGradientPlanner::OptimizePolicy(int horizon) {
  return Iterate({this}, TaskRows(), horizon, &launch_) ? -1 : 0;
}

void SampleGradientPlanner::InstallRollouts(int horizon, const float* returns, const uint8_t* failure, const int* order,
                                            int offset) {
  const int num_trajectory = num_trajectory_, num_gradient = num_gradient_, num_noisy = num_trajectory - num_gradient;
  std::copy(returns, returns + num_trajectory, returns_.begin());
  std::copy(failure, failure + num_trajectory, failure_.begin());
  std::copy(order, order + num_trajectory, trajectory_order.begin());
  launch_offset_ = offset; horizon_ = horizon;
  winner = returns_[trajectory_order[0]] < returns_[0] ? trajectory_order[0] : 0;
  winner_type = winner == 0 ? kNominal : (winner < num_noisy ? kPerturb : kGradient);
  {
    // the reference installs the plan under a shared lock (planner.cc:251-254); a concurrent ActionFromPolicy also
    // holds a shared lock, so this write takes the unique lock
    const std::unique_lock<std::shared_mutex> lock(mtx_);
    policy.plan = candidate_policy[winner].plan;
  }
  improvement = std::max((double)returns_[0] - (double)returns_[winner], 0.0);
  GradientCandidates(num_trajectory, num_gradient);
  iteration++;
}

void SampleGradientPlanner::GradientCandidates(int num_trajectory, int num_gradient) {
  if (num_gradient < 1) return;
  const int P = resampled_policy.num_spline_points, num_parameters = P * nu_;
  const int num_noisy = num_trajectory - num_gradient;
  gradient_previous = gradient;
  // fitness shaping (planner.cc:417-450), restated with its quirks (DESIGN.md §8): the weights are cached while the
  // number of noisy samples is unchanged, and on the call that computes them they are indexed by candidate index
  // (order[i] + 1), not by rank.  NaN returns sort after every number, as the device ranking puts them: a bare `<`
  // is no strict weak ordering once a NaN is present, and left NaN candidates where they stood
  if ((int)return_weight_.size() != num_noisy) {
    return_weight_.resize(num_noisy);
    std::iota(trajectory_order.begin(), trajectory_order.begin() + num_noisy, 0);
    std::stable_sort(trajectory_order.begin(), trajectory_order.begin() + num_noisy, [&](int a, int b) {
      const float ra = returns_[a], rb = returns_[b];
      return ra < rb || (rb != rb && ra == ra);
    });
    const double f0 = std::log(0.5 * num_noisy + 1.0);
    double den = 0.0;
    for (int i = 0; i < num_noisy; i++) den += std::max(0.0, f0 - std::log(trajectory_order[i] + 1));
    for (int i = 0; i < num_noisy; i++)
      return_weight_[i] = std::max(0.0, f0 - std::log(trajectory_order[i] + 1)) / den - 1.0 / num_noisy;
  }
  // on later calls trajectory_order is the ranking of all N: entries on slot 0 or a gradient slot add zero noise
  std::fill(gradient.begin(), gradient.end(), 0.0);
  for (int i = 0; i < num_noisy; i++) {
    const double* z = noise.data() + (size_t)trajectory_order[i] * num_parameters;
    const double scl = return_weight_[i] / num_noisy;
    for (int j = 0; j < num_parameters; j++) gradient[j] += z[j] * scl;
  }
  if ((int)step_size_.size() != num_gradient) {
    step_size_.resize(num_gradient);
    LogScale(step_size_.data(), gradient_max_step_size, gradient_min_step_size, num_gradient);
  }
  // candidates along -(f * gradient + (1 - f) * gradient_previous), rolled out in the next iteration
  for (int i = num_noisy; i < num_trajectory; i++) {
    candidate_policy[i] = resampled_policy;
    const double scaling = step_size_[i - num_noisy] / noise_exploration_;
    const double s0 = -scaling * gradient_filter_, s1 = -scaling * (1.0 - gradient_filter_);
    TimeSpline& plan = candidate_policy[i].plan;
    for (int t = 0; t < plan.Size(); t++) {
      double* node = plan.NodeValues(t);
      for (int d = 0; d < nu_; d++) node[d] += gradient[(size_t)t * nu_ + d] * s0;
      for (int d = 0; d < nu_; d++) node[d] += gradient_previous[(size_t)t * nu_ + d] * s1;
      for (int d = 0; d < nu_; d++)
        node[d] = std::max(policy.ctrlrange[2 * d], std::min(policy.ctrlrange[2 * d + 1], node[d]));
    }
  }
}

int SampleGradientPlanner::NominalTrajectory(int horizon) {
  // trajectory[0] <- resampled_policy as it stands; an empty plan is the clamped zero action
  const int P = std::max(resampled_policy.plan.Size(), 1);
  cands_.Resize(1, P, nu_);
  cands_.interpolation = (int)resampled_policy.plan.Interpolation();
  std::fill(cands_.knots.begin(), cands_.knots.end(), 0.f);
  std::fill(cands_.knot_times.begin(), cands_.knot_times.end(), time_);
  std::vector<double> v(nu_);
  if (resampled_policy.plan.Size() == 0) {
    resampled_policy.Action(v.data(), time_);
    std::copy(v.begin(), v.end(), cands_.knots.begin());
  }
  for (int k = 0; k < resampled_policy.plan.Size(); k++) {
    cands_.knot_times[k] = resampled_policy.plan.NodeTime(k);
    const double* node = resampled_policy.plan.NodeValues(k);
    std::copy(node, node + nu_, cands_.knots.begin() + (size_t)k * nu_);
  }
  if (int rc = launch_.Run({this}, {&cands_}, TaskRows(), horizon)) return rc;
  returns_[0] = launch_.returns[0]; failure_[0] = launch_.failure[0]; trajectory_order[0] = launch_.order[0];
  launch_offset_ = 0; horizon_ = horizon;
  return 0;
}

void SampleGradientPlanner::ActionFromPolicy(double* action, const double*, double time, bool use_previous) {
  // previous_policy is set only by Reset, as in the reference
  const std::shared_lock<std::shared_mutex> lock(mtx_);
  (use_previous ? previous_policy : policy).Action(action, time);
}

const Trajectory* SampleGradientPlanner::BestTrajectory() {
  if (FetchTrajectory(winner, horizon_, &best_)) return nullptr;
  best_.total_return = returns_[winner];
  best_.failure = failure_[winner];
  return &best_;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::PlannerOf;
using mjpc_b200_host::SampleGradientPlanner;

extern "C" {

int mjpc_b200_sg_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_gradient, int num_spline_points,
                                int interpolation, double exploration, double gradient_filter, double timestep,
                                const double* ctrlrange, uint32_t seed, int max_horizon, int device,
                                mjpc_b200_planner_t** out) {
  if (!model || !ctrlrange || !out || num_trajectory < 1 || num_spline_points < 2) return MJPC_B200_ERR_BAD_ARGUMENT;
  auto* p = new SampleGradientPlanner;
  int rc = p->Initialize(model, num_trajectory, num_gradient, num_spline_points, interpolation, exploration,
                         gradient_filter, timestep, ctrlrange, seed, max_horizon, device);
  if (rc) { delete p; *out = nullptr; return rc; }
  *out = mjpc_b200_host::ToHandle(p);
  return 0;
}
int mjpc_b200_sg_planner_get_result(mjpc_b200_planner_t* h, int* winner, int* winner_type, double* improvement,
                                    float* returns, int* order, double* knots, double* knot_times,
                                    double* gradient_knots, double* gradient) {
  auto* p = PlannerOf<SampleGradientPlanner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  const int N = p->num_trajectory(), G = p->num_gradient();
  if (winner) *winner = p->winner;
  if (winner_type) *winner_type = p->winner_type;
  if (improvement) *improvement = p->improvement;
  if (returns) std::copy(p->returns().begin(), p->returns().end(), returns);
  if (order) std::copy(p->trajectory_order.begin(), p->trajectory_order.end(), order);
  if (gradient) std::copy(p->gradient.begin(), p->gradient.end(), gradient);
  const int P = p->policy.num_spline_points, nu = p->policy.plan.Dim();
  for (int j = 0; gradient_knots && j < G; j++) {
    const auto& gp = p->candidate_policy[N - G + j].plan;
    std::fill(gradient_knots + (size_t)j * P * nu, gradient_knots + (size_t)(j + 1) * P * nu, 0.0);
    for (int k = 0; k < std::min(gp.Size(), P); k++)
      std::copy(gp.NodeValues(k), gp.NodeValues(k) + nu, gradient_knots + ((size_t)j * P + k) * nu);
  }
  return p->policy.plan.Export(knots, knot_times);
}

}  // extern "C"
