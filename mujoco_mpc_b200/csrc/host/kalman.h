// kalman.h - MJPC's Kalman state estimator (mjpc/estimators/kalman.{h,cc}) on the engine: the finite-difference
// Jacobians are one mjpc_b200_step_sensors launch each (the centre state and its ndstate, or 2 ndstate when centred,
// tangent-space perturbations); the filter arithmetic is double precision on the host.  Method names are the
// reference's; the engine plumbing is Estimator's (estimator.h).
//
//   UpdateMeasurement (kalman.cc:188-276)  C = d sensors / d state of the pre-step states and y_hat = the centre's
//                                          sensors from one launch; gain P C' (C P C' + R)^-1, correction, P -= ...,
//                                          symmetrised
//   UpdatePrediction  (kalman.cc:279-323)  A = d next state / d state (tangent-space differences) and the new state =
//                                          the centre's next state from one launch; P = A P A' + diag(process noise),
//                                          symmetrised
//
// Documented differences from the reference:
//  * a failed sensor-covariance factorisation returns MJPC_B200_ERR_BAD_ARGUMENT with a message naming the factor and
//    leaves state, covariance and time untouched (the reference calls mju_error);
//  * every state of a launch warm-starts the constraint solver from the centre state's qacc of the previous launch
//    (zeros after Reset); the reference reuses one mjData, so each perturbed step starts from the previous one's qacc;
//  * UpdateMeasurement takes mocap (the reference's mjData keeps the model's); UpdatePrediction uses the ctrl and
//    mocap of the last measurement, as the reference's mjData does;
//  * UpdateMeasurement takes the measured sensor slice [nsensordata], not the whole sensordata;
//  * time: both launches run at `time`; UpdatePrediction advances it by the timestep (the reference leaves its `time`
//    member alone and its mjData's clock advances inside mj_step);
//  * settings are arguments: the blob carries no custom numerics (mujoco_mpc_b200.estimator.CppKalman reads them), and
//    the engine default for the finite differences is centred with a larger epsilon than the reference's fp64 1e-6
//    one-sided (DESIGN.md, "Kalman filter").
#pragma once
#include <vector>

#include "estimator.h"

namespace mjpc_b200_host {

class Kalman : public Estimator {
 public:
  Kalman() : Estimator("kalman") {}
  // kalman.cc:31-110: timestep, sensor range (Estimator::InitializeBase), finite-difference settings
  int Initialize(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep, double epsilon,
                 bool centered, int device);
  // kalman.cc:113-185: Estimator::Reset, and the ctrl and mocap of the last measurement = zeros and the model's mocap
  void Reset(const double* state, double time, double covariance_scale, double process_scale,
             double sensor_scale) override;
  int UpdateMeasurement(const double* ctrl, const double* sensor, const float* mocap);   // kalman.cc:188-276
  int UpdatePrediction();                                                                 // kalman.cc:279-323
  int Update(const double* ctrl, const double* sensor, const float* mocap) override;   // UpdateMeasurement, UpdatePrediction
  // {ndstate, nstates, nsensordata, warnings, timestep, epsilon}
  void GetScalars(double* scalars) const override;

  int nstates = 0;
  double epsilon = 0;
  bool centered = false;

 private:
  // the centre state and its perturbations x (+) eps e_i (then x (+) -eps e_i when centred) stepped in one launch
  int Perturbed(const double* ctrl, const float* mocap);
  std::vector<double> ctrl_, jacobian_;
  std::vector<float> mocap_;
};

}  // namespace mjpc_b200_host
