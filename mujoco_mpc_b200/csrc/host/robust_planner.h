// robust_planner.h - C++ host side of the Robust planner (mjpc/planners/robust/robust_planner.h:30-76,
// robust_planner.cc:40-160) over the SamplingPlanner delegate.  The ncandidates x nrepetitions NoisyRollouts the
// reference schedules on its ThreadPool (robust_planner.cc:110-129) are ONE spline launch with the
// handle's force noise switched on (mjpc_b200_set_xfrc_noise_batched; injected Philox stream, seed + iteration).
#pragma once
#include <algorithm>
#include <memory>

#include "sampling_planner.h"

namespace mjpc_b200_host {

class RobustPlanner : public Planner {
 public:
  // the perturbed rollouts run on an engine handle of their own (max_candidates = noisy_candidates), so the delegate's
  // clean trajectories (what BestTrajectory returns, robust_planner.cc:163-165) survive the second launch
  // (engine != nullptr: that handle, not owned, instead of one of its own)
  int Initialize(std::unique_ptr<SamplingPlanner> delegate, const mjpc_model_blob* model, int noisy_candidates,
                 int max_horizon, int device, mjpc_b200_t* engine = nullptr);
  // robust_repetitions (5), robust_candidates (-1 -> sampling_trajectories / repetitions), robust_xfrc (0.1),
  // robust_xfrc_rate (0.1): robust_planner.cc:44-57
  void Configure(int sampling_trajectories, int ncandidates, int nrepetitions, double xfrc_std, double xfrc_rate, uint32_t seed);
  void Reset(int horizon, const double* initial_repeated_action) override { delegate_->Reset(horizon, initial_repeated_action); }
  void SetState(const double* state, double time, const double* mocap) override;
  int OptimizePolicy(int horizon) override;                            // :91-157: Iterate over this planner alone
  // OptimizePolicy of every planner of ps, which plan on one pair of handles: ONE clean launch of all the delegates'
  // candidates, then ONE noisy launch where each problem draws its force noise with its own key (NoiseSeed); problem
  // b reads task row b of `rows`.  0, -1 for ncandidates < 0, or a launch's error code
  static int Iterate(const std::vector<RobustPlanner*>& ps, const TaskRows& rows, int horizon, SplineLaunch* launch);
  // OptimizePolicy between the delegate's clean launch (its PrepareOptimize + InstallRollouts) and the noisy one: the
  // top `ncandidates` each repeated nrepetitions times into the noisy candidates.  Returns their number, 0 when there is
  // no noisy launch to make (fewer than two candidates: the policy is installed already) or -1 for ncandidates < 0.
  int PrepareNoisy(int ncandidates);
  uint32_t NoiseSeed() const { return seed_ + (uint32_t)delegate_->iteration; }   // the noisy launch's force-noise key
  int TopCandidates() const { return std::min(ncandidates_, delegate_->num_trajectory()); }
  // ... after the noisy launch: its returns and failure flags [ncandidates][nrepetitions]; the mean-return scores
  // (robust_planner.cc:131-154), the installed policy and improvement
  void InstallNoisy(const float* returns, const uint8_t* failure);
  int NominalTrajectory(int) override { return 0; }   // not restated: planning disabled leaves the plan as it is
  void ActionFromPolicy(double* action, const double* state, double time, bool use_previous = false) override {
    delegate_->ActionFromPolicy(action, state, time, use_previous);
  }
  const Trajectory* BestTrajectory() override { return delegate_->BestTrajectory(); }
  std::vector<mjpc_b200_t*> Handles() override { return {delegate_->gpu(), gpu_}; }
  SamplingPlanner* delegate() { return delegate_.get(); }
  const std::vector<double>& scores() const { return scores_; }

 private:
  std::unique_ptr<SamplingPlanner> delegate_;
  int ncandidates_ = 12, nrepetitions_ = 5;
  double xfrc_std_ = 0.1, xfrc_rate_ = 0.1;
  uint32_t seed_ = 0x5EED;
  std::vector<double> scores_;
  SplineCandidates noisy_;
  int ncandidates_now_ = 0;                           // of the noisy candidates PrepareNoisy made
};

}  // namespace mjpc_b200_host
