// unscented.h - MJPC's Unscented state estimator (mjpc/estimators/unscented.{h,cc}) on the engine: the 2 ndstate + 1
// sigma-point steps with their measurement sensors are one mjpc_b200_step_sensors launch; the filter arithmetic is
// double precision on the host.  Method names are the reference's; the engine plumbing is Estimator's (estimator.h).
//
// Documented differences from the reference:
//  * a failed factorisation (covariance or sensor covariance) returns MJPC_B200_ERR_BAD_ARGUMENT with a message naming
//    the factor and leaves state, covariance and time untouched (the reference calls mju_error);
//  * every sigma point warm-starts the constraint solver from the nominal point's qacc of the previous update (zeros
//    after Reset); the reference reuses one mjData, so each point starts from the previous point's qacc;
//  * Update takes mocap (the reference's mjData keeps the model's) and the measured sensor slice [nsensordata];
//  * settings are arguments: the blob carries no custom numerics (mujoco_mpc_b200.estimator.CppUnscented reads them).
#pragma once
#include <vector>

#include "estimator.h"

namespace mjpc_b200_host {

class Unscented : public Estimator {
 public:
  Unscented() : Estimator("unscented") {}
  // unscented.cc:31-168: alpha, beta, timestep, sensor range (Estimator::InitializeBase)
  int Initialize(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep, double alpha,
                 double beta, int device);
  int Update(const double* ctrl, const double* sensor, const float* mocap) override;   // unscented.cc:496-574
  // {ndstate, nsigma, nsensordata, warnings, timestep}
  void GetScalars(double* scalars) const override;
  void SigmaPoints();                                                           // :293-349 (factor checked by Update)
  int EvaluateSigmaPoints(const double* ctrl, const float* mocap);             // :353-394
  void QuaternionMeans();                                                       // :578-626
  void SigmaPointDifferences();                                                 // :397-428
  void SigmaCovariances();                                                      // :431-494

  int nsigma = 0;
  double sigma_step = 0, weight_mean0 = 0, weight_covariance0 = 0, weight_sigma = 0;

 private:
  std::vector<double> factor_, next_states_, sensors_, state_mean_, sensor_mean_, state_difference_,
      sensor_difference_, cov_yy_, cov_sy_, cov_ss_;
};

}  // namespace mjpc_b200_host
