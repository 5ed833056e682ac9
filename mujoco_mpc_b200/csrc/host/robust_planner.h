// robust_planner.h - C++ host side of the Robust planner (mjpc/planners/robust/robust_planner.h:30-76,
// robust_planner.cc:40-160) over the SamplingPlanner delegate.  The ncandidates x nrepetitions NoisyRollouts the
// reference schedules on its ThreadPool (robust_planner.cc:110-129) are ONE mjpc_b200_rollout_spline launch with the
// handle's force noise switched on (mjpc_b200_set_xfrc_noise; injected Philox stream, seed + iteration).
#pragma once
#include <memory>

#include "sampling_planner.h"

namespace mjpc_b200_host {

class RobustPlanner : public Planner {
 public:
  // the perturbed rollouts run on an engine handle of their own (max_candidates = noisy_candidates), so the delegate's
  // clean trajectories (what BestTrajectory returns, robust_planner.cc:163-165) survive the second launch
  int Initialize(std::unique_ptr<SamplingPlanner> delegate, const mjpc_model_blob* model, int noisy_candidates,
                 int max_horizon, int device);
  // robust_repetitions (5), robust_candidates (-1 -> sampling_trajectories / repetitions), robust_xfrc (0.1),
  // robust_xfrc_rate (0.1): robust_planner.cc:44-57
  void Configure(int sampling_trajectories, int ncandidates, int nrepetitions, double xfrc_std, double xfrc_rate, uint32_t seed);
  void Reset(int horizon, const double* initial_repeated_action) override { delegate_->Reset(horizon, initial_repeated_action); }
  void SetState(const double* state, double time, const double* mocap) override;
  int OptimizePolicy(int horizon) override;                            // :91-157
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
};

}  // namespace mjpc_b200_host
