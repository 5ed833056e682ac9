// batch_ilqg_planner.h - several independent iLQG problems planned together: one engine handle, one iLQGPlanner per
// problem (its own state, mocap, task snapshot, policy, regularisation and policy lock), and per iteration one batched
// launch per sweep for all problems:
//   feedback rollouts of every NominalTrajectory -> derivatives -> cost derivatives -> backward passes of the problems
//   still failing, round by round, each with its own regularisation -> action rollouts of the problems that succeeded.
// Each problem runs exactly the host steps iLQGPlanner runs around its own calls (the prepare / install halves), so
// its result is bitwise the one an iLQGPlanner with the same inputs computes with its own launches.
#pragma once
#include <cstdint>
#include <memory>
#include <vector>

#include "ilqg_planner.h"

namespace mjpc_b200_host {

class BatchILQGPlanner {
 public:
  ~BatchILQGPlanner();
  int Initialize(const mjpc_model_blob* model, int num_problems, int num_rollouts, int representation, int max_horizon,
                 int device);
  int NumProblems() const { return (int)problems_.size(); }
  iLQGPlanner& problem(int b) { return *problems_[b]; }
  // Task::weight / parameters / task-state block of problem b; NULL members keep the current value
  void SetTask(int b, const double* weight, const double* parameters, const double* task_state);
  // iLQGPlanner::NominalTrajectory of every problem in one launch; <0 on error
  int NominalTrajectory(int horizon);
  // iLQGPlanner::OptimizePolicy of every problem; updated[b] (may be NULL) receives its 1/0; <0 on error
  int OptimizePolicy(int horizon, int* updated);

  iLQGSettings settings;   // shared by every problem

 private:
  int Nominal(int horizon);
  int Iterate(int horizon, int* updated);
  // inputs of one feedback launch for the problems `idx` (flat candidate j*K + i for problem idx[j])
  int FeedbackLaunch(const std::vector<int>& idx, int horizon, bool with_du, int mode);

  mjpc_b200_t* gpu_ = nullptr;
  std::vector<std::unique_ptr<iLQGPlanner>> problems_;
  int K_ = 0, representation_ = 0, nu_ = 0, ds_ = 0, n_ = 0, nr_ = 0, nmocap7_ = 0;
  std::vector<double> weight_, parameters_, task_state_;   // [B][num_term], [B][num_parameters], [B][task_state_size]
  int nw_ = 0, np_ = 0, nts_ = 0;
  // launch staging ([problems of the launch][..])
  std::vector<float> st_, mc_, x_, u_, g_, du_, steps_, res_, ret_;
  std::vector<double> times_, t_, w_, p_, ts_;
  std::vector<uint8_t> fail_;
  std::vector<int> order_;
  std::vector<float> A_, B_, C_, D_, cx_, cu_, cxx_, cuu_, cxu_;           // [B][H][..] of the iteration
  std::vector<float> sA_, sB_, scx_, scu_, scxx_, scxu_, scuu_, sact_, mu_, K_out_, du_out_, dV_out_;   // retry subset
  std::vector<int> status_;
};

}  // namespace mjpc_b200_host
