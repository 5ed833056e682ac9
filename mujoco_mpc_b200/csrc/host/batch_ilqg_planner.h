// batch_ilqg_planner.h - several independent iLQG problems planned together: one engine handle, one iLQGPlanner per
// problem (its own state, mocap, task snapshot, policy, regularisation and policy lock), and per iteration one batched
// launch per sweep for all problems:
//   feedback rollouts of every NominalTrajectory -> derivatives -> cost derivatives -> backward passes of the problems
//   still failing, round by round, each with its own regularisation -> action rollouts of the problems that succeeded.
// Each problem runs exactly the host steps iLQGPlanner runs around its own calls (the prepare / install halves), so
// its result is bitwise the one an iLQGPlanner with the same inputs computes with its own launches.  The sweeps
// themselves (ILQGSweeps) run over any subset of planners on a handle; BatchILQSPlanner uses them for its iLQG halves.
#pragma once
#include <cstdint>
#include <memory>
#include <vector>

#include "ilqg_planner.h"

namespace mjpc_b200_host {

// the task snapshots of a batch's problems: rows [..][nw], [..][np], [..][nts]; a NULL array when the model has none
struct TaskRows {
  const double *w = nullptr, *p = nullptr, *ts = nullptr;
  int nw = 0, np = 0, nts = 0;
};

// The batched iLQG sweeps over any subset of iLQGPlanners that plan on one handle (the planners need not be owned by
// it): planner ps[j] reads task snapshot row task[j].  Every planner of a call must have the same settings.
class ILQGSweeps {
 public:
  void Attach(mjpc_b200_t* gpu, int num_rollouts, int representation);
  // iLQGPlanner::NominalTrajectory of each planner, one feedback launch; <0 on error
  int Nominal(const std::vector<iLQGPlanner*>& ps, const std::vector<int>& task, const TaskRows& rows, int horizon);
  // iLQGPlanner::Iteration of each planner; updated[j] (may be NULL) receives its 1/0; <0 on error
  int Iterate(const std::vector<iLQGPlanner*>& ps, const std::vector<int>& task, const TaskRows& rows, int horizon,
              int* updated);

 private:
  // one feedback launch of the candidate policies of ps (flat candidate j*K + i for ps[j])
  int FeedbackLaunch(const std::vector<iLQGPlanner*>& ps, const std::vector<int>& task, const TaskRows& rows,
                     int horizon, bool with_du, int mode);

  mjpc_b200_t* gpu_ = nullptr;
  int K_ = 0, representation_ = 0, nu_ = 0, ds_ = 0, n_ = 0, nr_ = 0, nmocap7_ = 0;
  // launch staging ([problems of the launch][..])
  std::vector<float> st_, mc_, x_, u_, g_, du_, steps_, res_;
  std::vector<double> times_, t_, w_, p_, ts_;
  std::vector<float> A_, B_, C_, D_, cx_, cu_, cxx_, cuu_, cxu_;           // [J][H][..] of the iteration
  std::vector<float> sA_, sB_, scx_, scu_, scxx_, scxu_, scuu_, sact_, mu_, K_out_, du_out_, dV_out_;   // retry subset
  std::vector<int> status_;
  std::vector<float> ret_;   // [J][K] of the last feedback launch
  std::vector<uint8_t> fail_;
  std::vector<int> order_;
};

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
  TaskRows Rows() const;

  mjpc_b200_t* gpu_ = nullptr;
  std::vector<std::unique_ptr<iLQGPlanner>> problems_;
  std::vector<iLQGPlanner*> all_;
  std::vector<int> all_idx_;
  std::vector<double> weight_, parameters_, task_state_;   // [B][num_term], [B][num_parameters], [B][task_state_size]
  int nw_ = 0, np_ = 0, nts_ = 0;
  ILQGSweeps sweeps_;
};

}  // namespace mjpc_b200_host
