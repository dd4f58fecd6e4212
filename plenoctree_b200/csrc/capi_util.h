// capi_util.h — helpers shared by the extern "C" translation units (capi.cu, pipeline.cu, projection.cu).
#pragma once
#include <cuda_runtime.h>

#include "kernels.h"

int pob_fail(const char* where, const char* what);
int pob_cuda_fail(const char* where, cudaError_t e);
// the SM count the kernels split their work for (capi.cu: sm_count), or 0 with the reason recorded under `where`
int pob_sms_or_fail(const char* where);
// sh_deg, the packed weights pointer and precision of an MLP call, then the device: its SM count, or 0 after a
// refusal recorded under `where`
int pob_check_common(const char* where, const void* packed, int sh_deg, int precision);
// POB_SIGMA_RELU or POB_SIGMA_SOFTPLUS, else pob_fail
int pob_check_sigma_activation(const char* where, int sigma_activation);
// NULL -> the reference default (relu trunk); else the descriptor if 0 <= min_deg <= max_deg <= 10, legacy_order is
// 0 / 1 and net_activation a POB_NET_* code, otherwise pob_fail
struct pob_posenc;
int pob_check_posenc(const char* where, const pob_posenc* posenc, pob::NetDesc& out);
// the FwdParams of one MLP (weights, sh_deg and network; no source or output)
pob::FwdParams pob_base_params(const void* packed, int sh_deg, pob::NetDesc net);
// the first checks of every point evaluator, pob_check_common then pob_check_posenc: the SM count and, in p, the
// base params of the network, or 0 after a refusal recorded under `where`.  Internal to each translation unit, so the
// library exports no symbol for it.
static inline int pob_eval_setup(const char* where, const void* packed, int sh_deg, const pob_posenc* posenc,
                                 int precision, pob::FwdParams& p) {
  const int sms = pob_check_common(where, packed, sh_deg, precision);
  if (!sms) return 0;
  pob::NetDesc net;
  if (pob_check_posenc(where, posenc, net)) return 0;
  p = pob_base_params(packed, sh_deg, net);
  return sms;
}

// vanilla NeRF (pob_view_branch): deg_view in [0, 32] and the four arrays of MLPs 0 .. n_mlps - 1, else pob_fail
struct pob_view_branch;
int pob_check_view(const char* where, const pob_view_branch* view, int n_mlps);
// the FwdParams of one vanilla MLP (OUT_VANILLA, heads VANILLA_NH wide) with view-branch MLP `mlp` and table `t`
pob::FwdParams pob_vanilla_params(const void* packed, pob::NetDesc net, const pob_view_branch& view, int mlp,
                                  const float* t);

#define POB_CUDA(where, call)                               \
  do {                                                      \
    cudaError_t _e = (call);                                \
    if (_e != cudaSuccess) return pob_cuda_fail(where, _e); \
  } while (0)

// ---- instrumentation (bench.py): kernel launch counter and per-phase CUDA-event timing ---------
// pob_timing_read reports the first POB_PH_LEGACY_COUNT classes, pob_timing_read_phases all POB_PH_COUNT
enum PobPhase { POB_PH_FWD = 0, POB_PH_BWD, POB_PH_WGRAD, POB_PH_RENDER, POB_PH_OPTIM, POB_PH_QUANT, POB_PH_COUNT };
constexpr int POB_PH_LEGACY_COUNT = 5;
void pob_count_launch(int n = 1);
// records an event pair around [begin, end) of one kernel launch when timing is enabled
struct PobPhaseTimer {
  PobPhaseTimer(int phase, cudaStream_t st);
  ~PobPhaseTimer();
  int slot;
  cudaStream_t st;
};

// one kernel launch on stream `st`: counted, timed under `phase` and its error returned from the caller
#define POB_LAUNCH(where, phase, st, call) \
  do {                                     \
    pob_count_launch();                    \
    PobPhaseTimer _t(phase, st);           \
    POB_CUDA(where, call);                 \
  } while (0)
