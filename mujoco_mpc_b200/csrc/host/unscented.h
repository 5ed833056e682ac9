// unscented.h - MJPC's Unscented state estimator (mjpc/estimators/unscented.{h,cc}) on the engine: the 2 ndstate + 1
// sigma-point steps with their measurement sensors are one mjpc_b200_step_sensors launch; the filter arithmetic is
// double precision on the host.  Method names are the reference's.
//
// Documented differences from the reference:
//  * a failed factorisation (covariance or sensor covariance) returns MJPC_B200_ERR_BAD_ARGUMENT with a message naming
//    the factor and leaves state, covariance and time untouched (the reference calls mju_error);
//  * every sigma point warm-starts the constraint solver from the nominal point's qacc of the previous update (zeros
//    after Reset); the reference reuses one mjData, so each point starts from the previous point's qacc;
//  * Update takes mocap (the reference's mjData keeps the model's) and the measured sensor slice [nsensordata];
//  * settings are arguments: the blob carries no custom numerics (mujoco_mpc_b200.estimator.CppUnscented reads them).
#pragma once
#include <string>
#include <vector>

#include "ilqg_planner.h"

namespace mjpc_b200_host {

// What the estimators read from the blob besides iLQGPolicyModel: every sensor's dimension, the model's mocap poses
// [7 nmocap] and the Reset state (the first keyframe, else qpos0 and zero qvel).  0, or MJPC_B200_ERR_BAD_BLOB for a
// blob without sensor entries.
int LoadEstimatorBlob(const mjpc_model_blob* model, const iLQGPolicyModel& m, std::vector<int>* dims, int* nmocap,
                      std::vector<float>* mocap0, std::vector<double>* key_state);

class Unscented {
 public:
  ~Unscented();
  // unscented.cc:31-168: alpha, beta, timestep, sensor range; the engine handle holds nsigma candidates
  int Initialize(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep, double alpha,
                 double beta, int device);
  // unscented.cc:171-290: state NULL -> the model's first keyframe if it has one, else qpos0 and zero qvel
  void Reset(const double* state, double time, double covariance_scale, double process_scale, double sensor_scale);
  int Update(const double* ctrl, const double* sensor, const float* mocap);   // unscented.cc:496-574
  void SigmaPoints();                                                           // :293-349 (factor checked by Update)
  int EvaluateSigmaPoints(const double* ctrl, const float* mocap);             // :353-394
  void QuaternionMeans();                                                       // :578-626
  void SigmaPointDifferences();                                                 // :397-428
  void SigmaCovariances();                                                      // :431-494

  std::vector<double> state, covariance, noise_process, noise_sensor;
  double time = 0;
  int warnings = 0;   // sigma-point steps that raised a warning since Reset
  int ndstate = 0, nsigma = 0, nsensordata = 0;
  double sigma_step = 0, weight_mean0 = 0, weight_covariance0 = 0, weight_sigma = 0, timestep = 0;
  std::string error;

 private:
  mjpc_b200_t* engine_ = nullptr;
  iLQGPolicyModel m_;
  int sensor_start_ = 0, nsensor_ = 0, nmocap_ = 0;
  std::vector<double> key_state_, factor_, sigma_, states_, sensors_, state_mean_, sensor_mean_, state_difference_,
      sensor_difference_, cov_yy_, cov_sy_, cov_ss_, qacc_warmstart_;
  std::vector<float> fstates_, fnext_, fsensor_, fqacc_, fwarm_, mocap0_;
  std::vector<int> counts_;
};

}  // namespace mjpc_b200_host
