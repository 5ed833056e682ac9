// estimator.h - MJPC's Unscented and Kalman state estimators (mjpc/estimators/unscented.{h,cc}, kalman.{h,cc}; the
// reference's Estimator base, mjpc/estimators/estimator.h) as a bank of num_filters independent filters of one kind
// and one model on one engine handle, each with its own state, covariance, time, noise, warm start, ctrl, sensors and
// mocap.  A single filter (mjpc_b200_unscented_create, mjpc_b200_kalman_create) is the bank of one.  Every update runs
// on the device: the filter arithmetic in fp64 (estimator_kernels.cuh) and the rows of all filters as one step_batch
// launch per sigma-point set or Jacobian (filter_bank.h).  The host uploads ctrl, sensors and mocap once per update and
// downloads one status per filter; state and covariance stay on the device until Get.
//
//   Unscented          the 2 ndstate + 1 sigma points (nominal last) stepped with their measurement sensors in one
//                      launch; means (QuaternionMeans for free and ball joints), differences, covariances, gain update
//   Kalman measurement (kalman.cc:188-276)  C = d sensors / d state of the pre-step states and y_hat = the centre's
//                      sensors from one launch; gain P C' (C P C' + R)^-1, correction, P -= ..., symmetrised
//   Kalman prediction  (kalman.cc:279-323)  A = d next state / d state (tangent-space differences) and the new state
//                      = the centre's next state from one launch; P = A P A' + diag(process noise), symmetrised
//
// Documented differences from the reference:
//  * a failed factorisation (the Unscented covariance, or either kind's sensor covariance) reports which factor failed
//    and leaves the filter's state, covariance, time, warm start and warnings untouched (the reference calls
//    mju_error);
//  * a factorisation fails on a pivot below 1e-15 or one that is not finite (the reference's mju_cholFactor(.., 0)
//    accepts pivots >= 0 and divides by a zero one);
//  * an update whose new state or covariance would not be finite fails the same way, untouched (status
//    NONFINITE_RESULT); ctrl, sensor and mocap values, and those of Reset, Set and SetNoise, that are not finite are
//    refused with MJPC_B200_ERR_BAD_ARGUMENT and nothing changed (the reference takes them);
//  * every row of a launch warm-starts the constraint solver from the centre (Kalman) or nominal (Unscented) row's qacc
//    of the filter's previous successful launch (zeros after Reset); the reference reuses one mjData, so each row
//    starts from the previous row's qacc;
//  * updates take mocap (the reference's mjData keeps the model's) and the measured sensor slice [nsensordata], not the
//    whole sensordata;
//  * Kalman: the prediction uses the ctrl and mocap of the last successful measurement, as the reference's mjData does;
//    both launches run at `time` and the prediction advances it by the timestep (the reference leaves its `time` member
//    alone and its mjData's clock advances inside mj_step);
//  * settings are arguments: the blob carries no custom numerics (mujoco_mpc_b200.estimator reads them), and the
//    engine default for the Kalman finite differences is centred with a larger epsilon than the reference's fp64 1e-6
//    one-sided (DESIGN.md, "Kalman filter").
#pragma once
#include <string>
#include <vector>

#include "planner.h"

namespace mjpc_b200_host {

constexpr int kKalman = 1, kUnscented = 2;   // the reference's `estimator` numeric
// step rows of one handle: num_filters x (rows per filter) above it is refused at create (MJPC_B200_ERR_CAPACITY)
constexpr int kEstimatorMaxRows = 65536;

class Estimator {
 public:
  ~Estimator();
  // kKalman (settings {epsilon, centered}) or kUnscented (settings {alpha, beta}), measuring the sensors
  // [sensor_start, sensor_start + nsensor); every filter starts as Reset(b, NULL, 0, 1e-4, 1e-4, 1e-4) leaves it
  int Initialize(const mjpc_model_blob* model, int kind, int num_filters, int sensor_start, int nsensor,
                 double timestep, const double* settings, int device);
  // filter b: state NULL -> the model's first keyframe if it has one, else qpos0 and zero qvel; covariance =
  // covariance_scale I, diagonal process / sensor noise, zero warm start and warnings; the ctrl and mocap of the last
  // measurement = zeros and the model's mocap
  int Reset(int b, const double* state, double time, double covariance_scale, double process_scale,
            double sensor_scale);
  int SetNoise(int b, const double* process, const double* sensor);             // NULL keeps one
  int Set(int b, const double* state, const double* covariance, double time);   // NULL keeps one
  // every filter from ctrl [B][nu], sensor [B][nsensordata] and mocap [B][7 nmocap] (NULL: the model's for every
  // filter); status [B] = mjpc_b200_bank::Status.  phases: the Kalman kind's steps (mjpc_b200_bank::Phases); a
  // prediction alone ignores ctrl, sensor and mocap and steps each filter with those of its last successful measurement
  int Update(const double* ctrl, const double* sensor, const float* mocap, int phases, int* status);
  // filter b's state, covariance, time and scalars {ndstate, rows, nsensordata, warnings, timestep} (Kalman: then
  // epsilon); any pointer may be NULL
  int Get(int b, double* state, double* covariance, double* time, double* scalars);
  // test hooks (mjpc_b200_bank::DebugRows / DebugFinish): the step rows of `phase` from ctrl [B][nu] and mocap
  // [B][7 nmocap] (NULL: the model's), and that phase's update from the caller's step outputs; status [B] is the raw
  // mjpc_b200_bank::Status
  int DebugRows(int phase, const double* ctrl, const float* mocap, float* qpos, float* qvel, float* warm, int* status);
  int DebugFinish(int phase, const double* sensor, const float* next_qpos, const float* next_qvel, const float* qacc,
                  const float* sensordata, const int* counts, int* status);
  // filter b runs on models[b] from now on (mjpc_b200_set_model_variants), and its Reset state and default mocap are
  // that model's; count is num_filters, or 0 for the bank's model again.  The filters' states are kept.
  int SetModels(const mjpc_model_blob* models, int count);
  const char* Name() const { return kind == kKalman ? "kalman" : kind == kUnscented ? "unscented" : "estimator"; }

  int kind = 0, num_filters = 0, ndstate = 0, nsensordata = 0, rows = 0;
  double timestep = 0, epsilon = 0;
  std::string error;

 private:
  int Fail(int rc, const std::string& what);
  // ctrl [B][nu] in float and mocap [B][7 nmocap] (NULL: each filter's model's) into fctrl_ / fmocap_; refuses values
  // that are not finite
  int StageInputs(const double* ctrl, const float* mocap);
  mjpc_b200_t* engine_ = nullptr;
  HostModel m_;
  int nmocap_ = 0;
  std::vector<double> model_key_state_;   // the bank's model's Reset state [nq + nv] and mocap [7 nmocap]
  std::vector<float> model_mocap0_;
  std::vector<double> key_state_;         // [B][nq + nv], [B][7 nmocap]: those of each filter's model
  std::vector<float> mocap0_;
  std::vector<float> fctrl_, fmocap_;   // [B][nu], [B][7 nmocap]: the inputs of the update being made
  std::vector<float> ctrl_, mocap_;     // [B][nu], [B][7 nmocap]: those of each filter's last successful measurement
};

}  // namespace mjpc_b200_host
