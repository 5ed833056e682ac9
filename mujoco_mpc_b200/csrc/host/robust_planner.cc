// robust_planner.cc - see robust_planner.h.  Reference: mjpc/planners/robust/robust_planner.cc.
#include "robust_planner.h"

#include <algorithm>

namespace mjpc_b200_host {

int RobustPlanner::Initialize(std::unique_ptr<SamplingPlanner> delegate, const mjpc_model_blob* model,
                              int noisy_candidates, int max_horizon, int device, mjpc_b200_t* engine) {
  delegate_ = std::move(delegate);
  return AttachEngine(model, noisy_candidates, max_horizon, device, engine);
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

int RobustPlanner::Iterate(const std::vector<RobustPlanner*>& ps, const TaskRows& rows, int horizon,
                           SplineLaunch* launch) {
  const size_t B = ps.size();
  // the delegates' OptimizePolicyCandidates: one clean launch on their handle
  std::vector<const Planner*> from(B);
  std::vector<const SplineCandidates*> cands(B);
  for (size_t b = 0; b < B; b++) {
    from[b] = ps[b]->delegate();
    cands[b] = &ps[b]->delegate()->PrepareOptimize(horizon);
  }
  if (int rc = launch->Run(from, cands, rows, horizon)) return rc;
  const int N = cands[0]->N;
  int noisy = 0;
  std::vector<uint32_t> seeds(B);
  for (size_t b = 0; b < B; b++) {
    RobustPlanner& p = *ps[b];
    const size_t o = b * N;
    p.delegate()->InstallRollouts(N, horizon, launch->returns.data() + o, launch->failure.data() + o,
                                  launch->order.data() + o, (int)o);
    noisy = p.PrepareNoisy(p.TopCandidates());   // the same for every problem: ncandidates and N are common
    from[b] = &p;                                // the noisy handle
    cands[b] = &p.noisy_;
    seeds[b] = p.NoiseSeed();
  }
  if (noisy <= 0) return noisy;
  // the noisy re-evaluations: one launch, each problem with its own noise key
  if (int rc = mjpc_b200_set_xfrc_noise_batched(ps[0]->gpu_, ps[0]->xfrc_std_, ps[0]->xfrc_rate_, (int)B, seeds.data()))
    return rc;
  if (int rc = launch->Run(from, cands, rows, horizon)) return rc;
  for (size_t b = 0; b < B; b++)
    ps[b]->InstallNoisy(launch->returns.data() + b * noisy, launch->failure.data() + b * noisy);
  return 0;
}

int RobustPlanner::OptimizePolicy(int horizon) {
  return Iterate({this}, TaskRows(), horizon, &launch_) ? -1 : 0;
}

int RobustPlanner::PrepareNoisy(int ncandidates) {
  SamplingPlanner& d = *delegate_;
  scores_.clear();
  if (ncandidates < 0) return -1;
  if (ncandidates == 0) return 0;
  if (ncandidates == 1) {
    d.CopyCandidateToPolicy(0);
    d.iteration++;
    return 0;
  }
  const int rep = nrepetitions_;
  const std::vector<int>& order = d.trajectory_order;    // the ranking of the clean rollouts
  const TimeSpline& nominal = d.policy.plan;
  const int P = nominal.Size(), nu = nominal.Dim();
  noisy_.Resize(ncandidates * rep, P, nu);
  noisy_.interpolation = (int)nominal.Interpolation();
  for (int k = 0; k < P; k++) noisy_.knot_times[k] = nominal.NodeTime(k);
  for (int c = 0; c < ncandidates; c++)
    for (int j = 0; j < rep; j++)
      for (int k = 0; k < P; k++) {
        const double* node = d.candidate_policy[order[c]].plan.NodeValues(k);
        for (int a = 0; a < nu; a++) noisy_.knots[(((size_t)c * rep + j) * P + k) * nu + a] = (float)node[a];
      }
  ncandidates_now_ = ncandidates;
  return noisy_.N;
}

void RobustPlanner::InstallNoisy(const float* ret, const uint8_t* fail) {
  SamplingPlanner& d = *delegate_;
  const int ncandidates = ncandidates_now_, rep = nrepetitions_;
  const std::vector<float>& clean = d.returns();         // scores of the clean rollouts, indexed by candidate
  const std::vector<int>& order = d.trajectory_order;    // ... and their ranking
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
}

}  // namespace mjpc_b200_host

// ------------------------------------------------------------------------------------------ C entry points
using mjpc_b200_host::PlannerOf;
using mjpc_b200_host::RobustPlanner;
using mjpc_b200_host::SamplingPlanner;

extern "C" {

int mjpc_b200_robust_planner_create(const mjpc_model_blob* model, int num_trajectory, int num_spline_points,
                                    int interpolation, double exploration, double timestep, const double* ctrlrange,
                                    uint32_t seed, int ncandidates, int nrepetitions, double xfrc_std, double xfrc_rate,
                                    int max_horizon, int device, mjpc_b200_planner_t** out) {
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
  *out = mjpc_b200_host::ToHandle(p);
  return 0;
}
// winner (candidate index of the clean launch), robust scores [ncandidates] (mean noisy return per top candidate),
// clean returns [num_trajectory], installed knots / times; returns the number of scores written
int mjpc_b200_robust_planner_get_result(mjpc_b200_planner_t* h, int* winner, double* scores, float* returns,
                                        double* knots, double* knot_times) {
  auto* p = PlannerOf<RobustPlanner>(h);
  if (!p) return MJPC_B200_ERR_BAD_ARGUMENT;
  SamplingPlanner* d = p->delegate();
  if (winner) *winner = d->winner;
  if (scores) std::copy(p->scores().begin(), p->scores().end(), scores);
  if (returns) std::copy(d->returns().begin(), d->returns().end(), returns);
  d->policy.plan.Export(knots, knot_times);
  return (int)p->scores().size();
}

}  // extern "C"
