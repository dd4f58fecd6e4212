// capi_util.h — helpers shared by the extern "C" translation units (capi.cu, pipeline.cu).
#pragma once
#include <cuda_runtime.h>

#include "kernels.h"

int pob_fail(const char* where, const char* what);
int pob_cuda_fail(const char* where, cudaError_t e);
// the SM count the kernels split their work for (capi.cu: sm_count), or 0 with the reason recorded under `where`
int pob_sms_or_fail(const char* where);
int pob_check_common(const char* where, const void* packed, int sh_deg, int precision);
// POB_SIGMA_RELU or POB_SIGMA_SOFTPLUS, else pob_fail
int pob_check_sigma_activation(const char* where, int sigma_activation);
// NULL -> the reference default (relu trunk); else the descriptor if 0 <= min_deg <= max_deg <= 10, legacy_order is
// 0 / 1 and net_activation a POB_NET_* code, otherwise pob_fail
struct pob_posenc;
int pob_check_posenc(const char* where, const pob_posenc* posenc, pob::NetDesc& out);
pob::FwdParams pob_base_params(const void* packed, int sh_deg, pob::NetDesc net);

#define POB_CUDA(where, call)                               \
  do {                                                      \
    cudaError_t _e = (call);                                \
    if (_e != cudaSuccess) return pob_cuda_fail(where, _e); \
  } while (0)

// ---- instrumentation (bench.py): kernel launch counter and per-phase CUDA-event timing ---------
enum PobPhase { POB_PH_FWD = 0, POB_PH_BWD, POB_PH_WGRAD, POB_PH_RENDER, POB_PH_OPTIM, POB_PH_COUNT };
void pob_count_launch(int n = 1);
// records an event pair around [begin, end) of one kernel launch when timing is enabled
struct PobPhaseTimer {
  PobPhaseTimer(int phase, cudaStream_t st);
  ~PobPhaseTimer();
  int slot;
  cudaStream_t st;
};
