// robust_planner.cc - see robust_planner.h.  Reference: mjpc/planners/robust/robust_planner.cc.
#include "robust_planner.h"

#include <algorithm>

namespace mjpc_b200_host {

int RobustPlanner::Initialize(std::unique_ptr<SamplingPlanner> delegate, const mjpc_model_blob* model,
                              int noisy_candidates, int max_horizon, int device) {
  delegate_ = std::move(delegate);
  return AttachEngine(model, noisy_candidates, max_horizon, device);
}

void RobustPlanner::Configure(int sampling_trajectories, int ncandidates, int nrepetitions, double xfrc_std,
                              double xfrc_rate, uint32_t seed) {
  nrepetitions_ = nrepetitions > 0 ? nrepetitions : 5;
  ncandidates_ = ncandidates != -1 ? ncandidates : sampling_trajectories / nrepetitions_;
  xfrc_std_ = xfrc_std; xfrc_rate_ = xfrc_rate; seed_ = seed;
}

void RobustPlanner::SetState(const double* state, double time, const double* mocap) {
  delegate_->SetState(state, time, mocap);
  Planner::SetState(state, time, mocap);
}

int RobustPlanner::OptimizePolicy(int horizon) {
  SamplingPlanner& d = *delegate_;
  const int ncandidates = d.OptimizePolicyCandidates(ncandidates_, horizon);
  scores_.clear();
  if (ncandidates < 0) return -1;
  if (ncandidates == 0) return 0;
  if (ncandidates == 1) {
    d.CopyCandidateToPolicy(0);
    d.iteration++;
    return 0;
  }
  const int rep = nrepetitions_;
  const std::vector<float>& clean = d.returns();         // scores of the clean rollouts, indexed by candidate
  const std::vector<int>& order = d.trajectory_order;    // ... and their ranking
  const TimeSpline& nominal = d.policy.plan;
  const int P = nominal.Size(), nu = nominal.Dim();
  std::vector<float> knots((size_t)ncandidates * rep * P * nu), ret((size_t)ncandidates * rep);
  std::vector<uint8_t> fail((size_t)ncandidates * rep);
  std::vector<double> knot_times(P);
  for (int k = 0; k < P; k++) knot_times[k] = nominal.NodeTime(k);
  for (int c = 0; c < ncandidates; c++)
    for (int j = 0; j < rep; j++)
      for (int k = 0; k < P; k++) {
        const double* node = d.candidate_policy[order[c]].plan.NodeValues(k);
        for (int a = 0; a < nu; a++) knots[(((size_t)c * rep + j) * P + k) * nu + a] = (float)node[a];
      }
  if (mjpc_b200_set_xfrc_noise(gpu_, xfrc_std_, xfrc_rate_, seed_ + (uint32_t)d.iteration)) return -1;
  if (RolloutSpline(knots.data(), knot_times.data(), (int)nominal.Interpolation(), P, ncandidates * rep, horizon,
                    ret.data(), fail.data(), nullptr))
    return -1;
  // for each candidate the mean of its valid noisy returns; pick the best mean (robust_planner.cc:131-154)
  int best_candidate = -1;
  double best_score = 0;
  for (int c = 0; c < ncandidates; c++) {
    double mean_return = clean[order[c]];
    int valid = 0;
    for (int j = 0; j < rep; j++) {
      if (fail[(size_t)rep * c + j]) continue;
      mean_return = (valid * mean_return + (double)ret[(size_t)rep * c + j]) / (valid + 1);
      valid++;
    }
    scores_.push_back(mean_return);
    if (best_candidate == -1 || mean_return < best_score) { best_candidate = c; best_score = mean_return; }
  }
  d.CopyCandidateToPolicy(best_candidate);
  d.improvement = std::max((double)clean[0] - (double)clean[d.winner], 0.0);
  d.iteration++;
  return 0;
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::RobustPlanner;
using mjpc_b200_host::SamplingPlanner;

extern "C" {

int mjpc_b200_robust_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_spline_points,
                                    int interpolation, double exploration, double timestep, const double* ctrlrange,
                                    uint32_t seed, int ncandidates, int nrepetitions, double xfrc_std, double xfrc_rate,
                                    int max_horizon, int device, void** out) {
  if (!model || !ctrlrange || !out) return MJPC_B200_ERR_BAD_ARGUMENT;
  const int rep = nrepetitions > 0 ? nrepetitions : 5;
  const int nc = ncandidates != -1 ? ncandidates : num_trajectory / rep;
  std::unique_ptr<SamplingPlanner> d(new SamplingPlanner);
  int rc = d->Initialize(model, num_trajectory, num_spline_points, interpolation, exploration, 0.0, timestep, ctrlrange,
                         seed, num_trajectory, max_horizon, device);
  if (rc) { *out = nullptr; return rc; }
  auto* p = new RobustPlanner;
  rc = p->Initialize(std::move(d), model, std::max(nc * rep, 1), max_horizon, device);
  if (rc) { delete p; *out = nullptr; return rc; }
  p->Configure(num_trajectory, ncandidates, nrepetitions, xfrc_std, xfrc_rate, seed);
  *out = p;
  return 0;
}
void mjpc_b200_robust_planner_destroy(void* p) { delete (RobustPlanner*)p; }
void mjpc_b200_robust_planner_reset(void* p, int horizon, const double* initial_repeated_action) {
  ((RobustPlanner*)p)->Reset(horizon, initial_repeated_action);
}
void mjpc_b200_robust_planner_set_state(void* p, const double* state, double time, const double* mocap) {
  ((RobustPlanner*)p)->SetState(state, time, mocap);
}
int mjpc_b200_robust_planner_optimize_policy(void* p, int horizon) { return ((RobustPlanner*)p)->OptimizePolicy(horizon); }
void mjpc_b200_robust_planner_action_from_policy(void* p, double* action, double time, int use_previous) {
  ((RobustPlanner*)p)->ActionFromPolicy(action, nullptr, time, use_previous != 0);
}
// winner (candidate index of the clean launch), robust scores [ncandidates] (mean noisy return per top candidate),
// clean returns [num_trajectory], installed knots / times; returns the number of scores written
int mjpc_b200_robust_planner_get_result(void* pv, int* winner, double* scores, float* returns, double* knots,
                                        double* knot_times) {
  auto* p = (RobustPlanner*)pv;
  SamplingPlanner* d = p->delegate();
  if (winner) *winner = d->winner;
  if (scores) std::copy(p->scores().begin(), p->scores().end(), scores);
  if (returns) std::copy(d->returns().begin(), d->returns().end(), returns);
  d->policy.plan.Export(knots, knot_times);
  return (int)p->scores().size();
}

}  // extern "C"
