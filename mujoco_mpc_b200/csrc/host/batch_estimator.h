// batch_estimator.h - B independent Kalman or Unscented filters of one model on one engine handle, each with its own
// state, covariance, time, noise, warm start, ctrl, sensors and mocap.  Every update runs on the device: the filter
// arithmetic in fp64 (estimator_kernels.cuh) and the rows of all B filters as one step_batch launch per Jacobian /
// sigma-point set (filter_bank.h).  The host uploads ctrl, sensors and mocap once per update and downloads one status
// per filter; state and covariance stay on the device until Get.
//
// Each filter restates the single filter of its kind (unscented.h, kalman.h) with its documented differences, and
// computes what that filter computes from the same state, covariance, time, noise and warm start: the device sums in
// the host's order, so the two differ only by the last bits of sin, cos and atan2 in the quaternion maps.  A failed
// factorisation in filter b returns MJPC_B200_ERR_BAD_ARGUMENT in status[b] and leaves filter b untouched; the other
// filters update normally.
#pragma once
#include <string>
#include <vector>

#include "planner.h"

namespace mjpc_b200_host {

// step rows of one handle: num_filters x (rows per filter) above it is refused at create (MJPC_B200_ERR_CAPACITY)
constexpr int kBatchEstimatorMaxRows = 65536;

class BatchEstimator {
 public:
  ~BatchEstimator();
  // kind 1 Kalman (settings {epsilon, centered}), 2 Unscented (settings {alpha, beta}); the sensor range and timestep
  // as the single filters take them
  int Initialize(const mjpc_model_blob* model, int kind, int num_filters, int sensor_start, int nsensor,
                 double timestep, const double* settings, int device);
  // Estimator::Reset of filter b
  int Reset(int b, const double* state, double time, double covariance_scale, double process_scale,
            double sensor_scale);
  int SetNoise(int b, const double* process, const double* sensor);
  int Set(int b, const double* state, const double* covariance, double time);
  // ctrl [B][nu], sensor [B][nsensordata], mocap [B][7 nmocap] or NULL (the model's for every filter), status [B]
  int Update(const double* ctrl, const double* sensor, const float* mocap, int* status);
  // state, covariance, time and the scalars of the single filter of this kind (any pointer may be NULL)
  int Get(int b, double* state, double* covariance, double* time, double* scalars);

  int kind = 0, num_filters = 0, ndstate = 0, nsensordata = 0, rows = 0;
  double timestep = 0, epsilon = 0;
  std::string error;

 private:
  int Fail(int rc, const std::string& what);
  mjpc_b200_t* engine_ = nullptr;
  HostModel m_;
  int nmocap_ = 0;
  std::vector<float> mocap0_, fctrl_, fmocap_;
  std::vector<double> key_state_;
};

}  // namespace mjpc_b200_host
