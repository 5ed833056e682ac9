// filter_bank.h - the engine side of the state estimators (csrc/host/estimator.h): B filters of one kind whose state,
// covariance, time, noise, warm start and warnings live in device memory of an engine handle, and whose update is the
// kernels of estimator_kernels.cuh around step_batch launches of all their rows.  Internal to libmjpc_b200.so:
// engine.cu implements it, estimator.cc calls it.
#pragma once
#include "../../include/mjpc_b200.h"

namespace mjpc_b200_bank {

struct Desc {
  int kind;          // 1 Kalman, 2 Unscented
  int num_filters;
  int rows;          // step rows per filter: Unscented nsigma, Kalman nstates
  int sensor_start, nsensor;
  double timestep;
  double sigma_step, weight_mean0, weight_covariance0, weight_sigma;   // Unscented
  double epsilon;                                                      // Kalman
  int centered;
  int njnt;                                                    // the model's joints, for the state arithmetic
  const int *jnt_type, *jnt_qposadr, *jnt_dofadr;
};

// one filter's field: STATE [nq+nv], COVARIANCE [ndstate^2], TIME [1], NOISE_PROCESS [ndstate], NOISE_SENSOR
// [nsensordata] (double); WARMSTART [nv] (float); WARNINGS [1] (int)
enum Field { STATE, COVARIANCE, TIME, NOISE_PROCESS, NOISE_SENSOR, WARMSTART, WARNINGS };

// the steps of a Kalman update; the Unscented kind has one step and ignores the choice
enum Phases { MEASUREMENT = 1, PREDICTION = 2, MEASUREMENT_AND_PREDICTION = 3 };

// a filter's status after an update: updated, or what failed and left it untouched: a factorisation (a pivot below
// 1e-15 or not finite), or a new state or covariance that would not be finite
enum Status { UPDATED = 0, SENSOR_FACTOR_FAILED = 1, COVARIANCE_FACTOR_FAILED = 2, NONFINITE_RESULT = 3 };

// The handle's filter bank for d (replacing any earlier one), every field zero.  A sensor range outside the model's
// sensors: MJPC_B200_ERR_BAD_ARGUMENT; a sensor the engine does not evaluate: MJPC_B200_ERR_UNSUPPORTED;
// num_filters x rows above the handle's max_candidates: MJPC_B200_ERR_CAPACITY.
int Init(mjpc_b200_t* h, const Desc& d);
// copies filter b's field to (write = 0) or from (write = 1) `data`
int Access(mjpc_b200_t* h, int b, int field, void* data, int write);
// one update of every filter from ctrl [B][nu], sensor [B][nsensordata] and mocap [B][7 nmocap]; status [B] = Status.
// phases: Phases.  A Kalman prediction alone reads no sensor (it may be NULL) and steps with the ctrl and mocap given.
int Update(mjpc_b200_t* h, const float* ctrl, const double* sensor, const float* mocap, int phases, int* status);

// Test hooks on the bank's real kernels, with its launch shape and stream.  phase: 0 the Unscented sigma points, 1 the
// Kalman measurement, 2 the Kalman prediction (the bank's kind must run it).
// DebugRows stages ctrl [B][nu] and mocap [B][7 nmocap] as Update does, runs estimator_rows_kernel and returns the step
// rows qpos [B rows][nq], qvel [B rows][nv], their warm starts warm [B rows][nv] and status [B] (phases 0 and 1 set
// it; phase 2 leaves the bank's).
// DebugFinish stages sensor [B][nsensordata] (NULL for phase 2), clears every status, writes next_qpos, next_qvel,
// qacc [B rows][nv], sensordata [B rows][nsensordata] and counts [B rows][4] where the step launch writes them, runs
// the phase's update kernel and returns status [B].
int DebugRows(mjpc_b200_t* h, int phase, const float* ctrl, const float* mocap, float* qpos, float* qvel, float* warm,
              int* status);
int DebugFinish(mjpc_b200_t* h, int phase, const double* sensor, const float* next_qpos, const float* next_qvel,
                const float* qacc, const float* sensordata, const int* counts, int* status);

}  // namespace mjpc_b200_bank
