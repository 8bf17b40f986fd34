/*
 * host_model.h — a built-in dynamics model as its host twin sees it, and the roll-forward mppib_compute_control runs on
 * it (csrc/host_twins.cpp). Internal to the library: the exported entries are in include/mppi_b200/host_twins.h.
 */
#pragma once
#include "../../include/mppi_b200/host_twins.h"

namespace mppib
{
// Autorally's 6-32-32-4 network with its first two weight matrices transposed to [in][out], once per call, for the host
// forward pass
struct FnnT
{
  float WT1[6 * 32], b1[32], WT2[32 * 32], b2[32], W3[4 * 32], b3[4];  // W3 keeps the reference's [out][in] order
};
void fnn_transpose(const float* theta, FnnT& t);

// What a model does not use may be NULL.
struct HostModel
{
  int dyn_id;
  const void* params;                          // the MPPIB_BLOB_DYN_PARAMS blob
  const FnnT* fnn;                             // Autorally's network
  const mppib_host_lstm* lstm;                 // the RACER steering LSTM; its `map` is not read, `elevation` is
  const mppib_elevation_map_header* elevation; // NULL: flat ground
  const mppib_elevation_map_header* normals;   // NULL: every normal (0, 0, 1)
};

// Controller::computeOutputTrajectoryHelper (controller.cuh:643-663): states [T][S] and outputs [T][O] from x0 and the
// controls u [T][C]; an LSTM starts from the initial state its weight blob carries. MPPIB_ERR_UNSUPPORTED for an id that
// is not a built-in model.
int roll_forward(const HostModel& m, const float* x0, const float* u, int T, float dt, float* states, float* outputs);
}  // namespace mppib
