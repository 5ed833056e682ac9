// plant_bank.h - the closed-loop plants of an engine handle (mjpc_b200_plant_* in include/mjpc_b200.h): B plants whose
// state stays in device memory and which plant_step_kernel (rollout_kernels.cuh) advances by one step each per launch.
// Internal to libmjpc_b200.so: engine.cu implements the entry points on it.
//
// One device allocation holds, every piece 256-byte aligned:
//   the plants    qpos [B][nq], qvel [B][nv], warm start [B][nv] (float); time, cost sum [B] (double);
//                 steps, warnings, status [B] (int)
//   disturbances  settings [B] (PlantDisturbance); OU states ctrl noise [B][nu], force noise [B][6 nbody]; the held
//                 wrench [B][6 nbody]; this step's uncommitted OU states [B][nu + 6 nbody] (float)
//   the upload    ctrl [B][nu], mocap [B][7 nmocap], task state [B][size] rebased to each plant's time, weight
//                 [B][num_term], parameters [B][num_parameters] (float): one H2D copy per step
//   the outputs   time [B] (double), state [B][nq+nv], cost [B] (float), status [B] (int), sensordata [B][dim],
//                 applied ctrl [B][nu] (float): one D2H copy per step
// The pinned staging mirrors the upload and the outputs byte for byte.  The host keeps each plant's mocap and task rows
// (task state in absolute time) and a copy of its time, from which it stages every step's upload.
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "device_memory.h"
#include "rollout_kernels.cuh"

struct PlantBank {
  mjpc_dev::PlantArgs a;   // device pointers into d_mem; the launch fills in the model, the pack and the instance
  int nsd = 0;             // sensor dimension of the plants' sensor range (0: no sensors)
  mjpc_mem::DeviceArray<unsigned char> d_mem;
  unsigned char* d_in = nullptr;    // the upload
  unsigned char* d_out = nullptr;   // the outputs
  mjpc_mem::PinnedArray<unsigned char> h_stage;   // [upload][outputs]
  size_t in_bytes = 0, out_bytes = 0;
  size_t o_ctrl = 0, o_mocap = 0, o_ts = 0, o_weight = 0, o_par = 0;                   // within the upload
  size_t o_time = 0, o_state = 0, o_cost = 0, o_status = 0, o_sens = 0, o_ctrl_out = 0;  // within the outputs
  std::vector<float> mocap;                                   // [B][7 nmocap]
  std::vector<mjpc_dev::PlantDisturbance> dist;               // [B], as on the device
  std::vector<double> weight, parameters, task_state, time;   // [B][..], task state in absolute time; time [B]
};
