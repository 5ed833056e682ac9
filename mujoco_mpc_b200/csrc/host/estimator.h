// estimator.h - the base every host state estimator derives from (the reference's virtual Estimator,
// mjpc/estimators/estimator.h, limited to what exists here) and the engine plumbing the estimators share: the engine
// handle holding 2 ndstate + 1 states (the most any filter steps in one launch), the blob's sensor range, mocap and
// Reset state, the float staging of one mjpc_b200_step_sensors launch with its warm start, and the double-precision
// gain step, symmetrisation and tangent-space state addition.
#pragma once
#include <string>
#include <vector>

#include "planner.h"

namespace mjpc_b200_host {

// What the estimators read from the blob besides HostModel: every sensor's dimension, the model's mocap poses
// [7 nmocap] and the Reset state (the first keyframe, else qpos0 and zero qvel).  0, or MJPC_B200_ERR_BAD_BLOB for a
// blob without sensor entries.
int LoadEstimatorBlob(const mjpc_model_blob* model, const HostModel& m, std::vector<int>* dims, int* nmocap,
                      std::vector<float>* mocap0, std::vector<double>* key_state);

class Estimator {
 public:
  virtual ~Estimator();
  // state NULL -> the model's first keyframe if it has one, else qpos0 and zero qvel; covariance = covariance_scale I,
  // diagonal process / sensor noise, zero warm start and warnings
  virtual void Reset(const double* state, double time, double covariance_scale, double process_scale,
                     double sensor_scale);
  // one filter update from ctrl [nu], the measured sensor slice [nsensordata] and mocap [7 nmocap] (NULL: the model's)
  virtual int Update(const double* ctrl, const double* sensor, const float* mocap) = 0;
  // the filter's scalars of mjpc_b200_estimator_get
  virtual void GetScalars(double* scalars) const = 0;

  std::vector<double> state, covariance, noise_process, noise_sensor;
  double time = 0;
  int warnings = 0;   // steps that raised a warning since Reset
  int ndstate = 0, nsensordata = 0;
  double timestep = 0;
  std::string error;

 protected:
  explicit Estimator(const char* name) : name_(name) {}
  // Loads the blob, checks the sensor range, creates the engine handle, sets the timestep and Resets.  Then it steps
  // the reset state once, so a range with a sensor the engine does not evaluate is refused here
  // (MJPC_B200_ERR_UNSUPPORTED) rather than at the first update, and Resets again.
  int InitializeBase(const mjpc_model_blob* model, int sensor_start, int nsensor, double timestep, int device);
  // steps the first n rows of states_ [n][nq+nv] from ctrl [nu] and mocap (NULL: the model's) at `time`, each
  // warm-started from qacc_warmstart_, into fnext_ / fsensor_ / fqacc_ / counts_
  int StepSensors(int n, const double* ctrl, const float* mocap);
  // after a successful update: the warm start from row `centre` of the last launch, and that launch's warnings
  void Commit(int centre);
  // corr [ndstate] = X S^-1 innovation and P = P0 - X S^-1 X', symmetrised, for X [ndstate][nsensordata] and
  // S [nsensordata]^2.  S is overwritten by its Cholesky factor and innovation by S^-1 innovation.  A factor that is
  // not full rank: MJPC_B200_ERR_BAD_ARGUMENT with corr and P untouched.  P may alias P0.
  int GainUpdate(const double* X, double* S, double* innovation, const double* P0, double* corr, double* P);
  void Symmetrize(double* P) const;                                 // P [ndstate]^2 = (P + P') / 2
  void StateAdd(double* x, const double* dx, double scale) const;   // x (+) scale dx: IntegratePos, velocities added

  const char* name_;   // the prefix of every error message
  mjpc_b200_t* engine_ = nullptr;
  HostModel m_;
  int sensor_start_ = 0, nsensor_ = 0, nmocap_ = 0, nstepped_ = 0;
  std::vector<double> key_state_, qacc_warmstart_, states_;
  std::vector<float> fstates_, fnext_, fsensor_, fqacc_, fwarm_, mocap0_;
  std::vector<int> counts_;
};

// mjpc_b200_estimator_t* is the Estimator base of the filter, whatever its kind
inline mjpc_b200_estimator_t* ToHandle(Estimator* f) { return reinterpret_cast<mjpc_b200_estimator_t*>(f); }
// the filter behind a handle if it is a T, else nullptr (a NULL handle, or one of another kind)
template <class T>
T* EstimatorOf(mjpc_b200_estimator_t* h) { return dynamic_cast<T*>(reinterpret_cast<Estimator*>(h)); }

}  // namespace mjpc_b200_host
