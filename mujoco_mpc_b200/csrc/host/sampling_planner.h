// sampling_planner.h - C++ host side above the C ABI: the Predictive Sampling planner with the reference's
// method names (mjpc/planners/sampling/planner.h:40-160, planner.cc:40-560), TimeSpline (mjpc/spline/spline.h)
// and SamplingPolicy (mjpc/planners/sampling/policy.cc:52-59).  Only Rollouts differs from the reference: it
// is ONE spline launch (SplineLaunch) instead of N closures scheduled on a ThreadPool.
//
// The reference's absl::BitGen cannot be seeded (planner.cc:331), so the noise source is injected:
// Philox4x32-10, key (seed, 0), counter (iteration, candidate, knot, dof), Box-Muller on the first two words.
#pragma once
#include <cstdint>
#include <shared_mutex>
#include <vector>

#include "planner.h"

namespace mjpc_b200_host {

enum SplineInterpolation : int { kZeroSpline = 0, kLinearSpline = 1, kCubicSpline = 2 };

// time-indexed knots, values row-major [node][dim]
class TimeSpline {
 public:
  explicit TimeSpline(int dim = 0, SplineInterpolation interp = kZeroSpline) : dim_(dim), interpolation_(interp) {}
  int Dim() const { return dim_; }
  int Size() const { return (int)times_.size(); }
  void Clear() { times_.clear(); values_.clear(); }
  void SetInterpolation(SplineInterpolation i) { interpolation_ = i; }
  SplineInterpolation Interpolation() const { return interpolation_; }
  void AddNode(double time, const double* values);   // values == nullptr -> zeros
  double NodeTime(int i) const { return times_[i]; }
  double* NodeValues(int i) { return values_.data() + (size_t)i * dim_; }
  const double* NodeValues(int i) const { return values_.data() + (size_t)i * dim_; }
  void Sample(double time, double* out) const;       // spline.cc:103-156
  // the nodes' values [Size()][Dim()] and times [Size()] (either may be NULL); returns Size()
  int Export(double* values, double* times) const;
 private:
  double Slope(int node, int k) const;               // spline.cc:269-287
  int dim_;
  SplineInterpolation interpolation_;
  std::vector<double> times_, values_;
};

struct SamplingPolicy {
  TimeSpline plan;
  std::vector<double> ctrlrange;  // [nu][2]
  int num_spline_points = 3;
  void Action(double* action, double time) const;    // Sample + Clamp
};

void Philox4x32(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]);
double PhiloxNormal(uint32_t seed, uint32_t iteration, uint32_t candidate, uint32_t knot, uint32_t dof);

// LogScale (utilities.cc:819-825): `steps` values ascending from min_value to max_value, evenly spaced in log
void LogScale(double* values, double max_value, double min_value, int steps);

class SamplingPlanner : public Planner {
 public:
  // model blob + settings that the reference reads from <custom> numerics (planner.cc:54-68).  engine != nullptr: roll
  // out on that handle (shared with other planners, not owned) instead of creating one
  int Initialize(const mjpc_model_blob* model, int num_trajectory, int num_spline_points, int interpolation,
                 double exploration, double exploration2, double timestep, const double* ctrlrange, uint32_t seed,
                 int max_candidates, int max_horizon, int device, mjpc_b200_t* engine = nullptr);
  void Reset(int horizon, const double* initial_repeated_action) override;
  int OptimizePolicy(int horizon) override;           // planner.cc:197-212: Iterate over this planner alone
  // OptimizePolicy of every planner of ps, which plan on one handle, with ONE launch of all their candidates; problem
  // b reads task row b of `rows`.  0, or the launch's error code
  static int Iterate(const std::vector<SamplingPlanner*>& ps, const TaskRows& rows, int horizon, SplineLaunch* launch);
  int NominalTrajectory(int horizon) override;        // UpdateNominalPolicy + the rollout of the nominal alone
  void UpdateNominalPolicy(int horizon);              // :240-323 (non-sliding resample)
  void AddNoiseToPolicy(int i);                       // :326-352
  // Rollouts (:355-393) in two halves around one launch, which may be shared with other planners:
  // the candidates (nominal + noise) as knots [num_trajectory][P][nu] and knot times [P]; returns P
  int PrepareCandidates(int num_trajectory, float* knots, double* knot_times);
  // ... the same into the planner's own SplineCandidates
  const SplineCandidates& Candidates(int num_trajectory);
  // OptimizePolicyCandidates (:155-194) up to its launch: the nominal update and the num_trajectory candidates
  const SplineCandidates& PrepareOptimize(int horizon);
  // the launch's horizon, and the returns, failure flags and ranking of these candidates, which it held from flat
  // index `offset` on
  void InstallRollouts(int num_trajectory, int horizon, const float* returns, const uint8_t* failure, const int* order,
                       int offset);
  void InstallBest();                                 // OptimizePolicy after the rollouts: winner, improvement, iteration
  // :229-237; the policy does not depend on the state
  void ActionFromPolicy(double* action, const double* state, double time, bool use_previous = false) override;
  void CopyCandidateToPolicy(int candidate);          // :534-543
  const Trajectory* BestTrajectory() override;
  int SetEnsemble(const mjpc_model_blob* models, int K, int worst) override { return ModelEnsemble(models, K, worst); }
  int SetStateEnsemble(int K, int worst, uint32_t seed) override { return StateEnsemble(K, worst, seed); }
  int SetStateCovariance(const double* covariance) override { return StateCovariance(covariance); }
  uint32_t PlanIteration() const override { return (uint32_t)iteration; }
  int CandidateTrajectory(int candidate, int horizon, Trajectory* out);   // trajectory[candidate] of the last Rollouts
  void SetPolicy(const double* times, const double* parameters, int num_nodes);   // policy.plan = nodes (ilqs/planner.cc:160-172)
  double timestep() const { return timestep_; }
  int num_trajectory() const { return num_trajectory_; }
  SplineInterpolation interpolation() const { return interpolation_; }
  double CandidateScore(int candidate) const { return returns_[trajectory_order[candidate]]; }
  int NumParameters() const { return nu_ * policy.num_spline_points; }

  SamplingPolicy policy, previous_policy;
  std::vector<SamplingPolicy> candidate_policy;
  std::vector<int> trajectory_order;
  int winner = 0;
  double improvement = 0;
  int iteration = 0;
  const std::vector<float>& returns() const { return returns_; }
  // noise_exploration[0..1] (sampling/planner.cc:85-88)
  void SetExploration(double e0, double e1) { noise_exploration_[0] = e0; noise_exploration_[1] = e1; }

 private:
  int num_trajectory_ = 0, nu_ = 0;
  SplineInterpolation interpolation_ = kCubicSpline;
  double noise_exploration_[2] = {0.1, 0.0};
  double timestep_ = 0.01;
  uint32_t seed_ = 0x5EED;
  SplineCandidates cands_;
  std::vector<float> returns_;
  std::vector<uint8_t> failure_;
  Trajectory best_;
  mutable std::shared_mutex mtx_;
};

}  // namespace mjpc_b200_host
