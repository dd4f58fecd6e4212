// capi.cu — extern "C" entry points declared in include/plenoctree_b200.h.
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "../../include/plenoctree_b200.h"
#include "capi_util.h"
#include "common.cuh"
#include "kernels.h"

static thread_local std::string g_err = "";

int pob_fail(const char* where, const char* what) {
  g_err = std::string(where) + ": " + what;
  return 1;
}
int pob_cuda_fail(const char* where, cudaError_t e) { return pob_fail(where, cudaGetErrorString(e)); }

// ---- instrumentation ---------------------------------------------------------------------------
#include <atomic>
#include <vector>
static std::atomic<long long> g_launches{0};
void pob_count_launch(int n) { g_launches += n; }
static bool g_timing = false;
struct TimedSlot {
  int phase;
  cudaEvent_t a, b;
};
static std::vector<TimedSlot> g_slots;
static double g_phase_ms[POB_PH_COUNT] = {};
static long long g_phase_n[POB_PH_COUNT] = {};
PobPhaseTimer::PobPhaseTimer(int phase, cudaStream_t s) : slot(-1), st(s) {
  if (!g_timing) return;
  TimedSlot t;
  t.phase = phase;
  cudaEventCreate(&t.a);
  cudaEventCreate(&t.b);
  cudaEventRecord(t.a, st);
  g_slots.push_back(t);
  slot = int(g_slots.size()) - 1;
}
PobPhaseTimer::~PobPhaseTimer() {
  if (slot >= 0) cudaEventRecord(g_slots[slot].b, st);
}
static void drain_slots() {
  for (auto& t : g_slots) {
    cudaEventSynchronize(t.b);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) {
      g_phase_ms[t.phase] += ms;
      g_phase_n[t.phase] += 1;
    }
    cudaEventDestroy(t.a);
    cudaEventDestroy(t.b);
  }
  g_slots.clear();
}

namespace {

// The weight gradient has 16 units of work (optim.cu: wgrad_assign_roles), each needing a CTA of its own; from 16
// SMs up the data gradient keeps at least one CTA, and its CTAs plus the weight gradient's fit on the device.
constexpr int MIN_SPLIT_SMS = 16;
int g_device_sms = -1;
thread_local std::string g_sm_count_env;   // the refused POB_SM_COUNT value, for the message

// SM count the kernels split their work for: the device's, or POB_SM_COUNT when set (read on every call).
// -1: no CUDA device, -2: not compute capability 9.0, -3: POB_SM_COUNT is not an integer in [16, device SMs].
int sm_count() {
  if (g_device_sms <= 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
    int major = 0, minor = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
    if (major != 9 || minor != 0) return -2;  // sm_90a only (wgmma)
    g_device_sms = n;
  }
  const char* e = getenv("POB_SM_COUNT");
  if (!e) return g_device_sms;
  char* end = nullptr;
  errno = 0;
  const long v = strtol(e, &end, 10);
  if (end == e || *end != '\0' || errno != 0 || v < MIN_SPLIT_SMS || v > g_device_sms) {
    g_sm_count_env = e;
    return -3;
  }
  return int(v);
}

// packed blob layout of one MLP
struct BlobLayout {
  size_t w_hi, w_lo, wt_hi, total;
};
BlobLayout blob_layout(int K) {
  const int NH = pob::heads_width(K);
  auto up = [](size_t x) { return (x + 1023) / 1024 * 1024; };
  BlobLayout b;
  b.w_hi = 0;
  b.w_lo = up(b.w_hi + pob::fwd_image_bytes(NH));
  b.wt_hi = up(b.w_lo + pob::fwd_image_bytes(NH));
  b.total = up(b.wt_hi + pob::bwd_image_bytes(NH));
  return b;
}
pob::MlpPacked packed_view(const void* blob, int K) {
  const BlobLayout b = blob_layout(K);
  const uint8_t* p = static_cast<const uint8_t*>(blob);
  pob::MlpPacked w;
  w.w_hi = p + b.w_hi;
  w.w_lo = p + b.w_lo;
  w.wt_hi = p + b.wt_hi;
  return w;
}

// packed blob of one vanilla MLP: its forward image (fp16) only
size_t vanilla_blob_bytes() { return (pob::fwd_image_bytes(pob::VANILLA_NH) + 1023) / 1024 * 1024; }

}  // namespace

int pob_check_view(const char* where, const pob_view_branch* view, int n_mlps) {
  if (!view) return pob_fail(where, "view branch descriptor is NULL");
  if (view->deg_view < 0 || view->deg_view > pob::MAX_DEG_VIEW)
    return pob_fail(where, "deg_view must be in [0, 32] (the posenc scale 2^(deg_view - 1) of a unit direction)");
  for (int i = 0; i < n_mlps; ++i) {
    const pob_view_mlp& v = view->mlp[i];
    if (!v.w10e_dev || !v.c_dev || !v.w11_dev || !v.b11_dev) return pob_fail(where, "NULL view branch array");
  }
  return 0;
}
pob::FwdParams pob_vanilla_params(const void* packed, pob::NetDesc net, const pob_view_branch& view, int mlp,
                                  const float* t) {
  pob::FwdParams p = pob_base_params(packed, -1, net);
  p.NH = pob::VANILLA_NH;
  p.w.w_lo = nullptr;    // the vanilla blob holds the fp16 forward image only
  p.w.wt_hi = nullptr;
  p.out_mode = pob::OUT_VANILLA;
  p.view_t = t;
  p.view_w11 = view.mlp[mlp].w11_dev;
  p.view_b11 = view.mlp[mlp].b11_dev;
  return p;
}

int pob_sms_or_fail(const char* where) {
  const int n = sm_count();
  if (n > 0) return n;
  if (n == -3)
    pob_fail(where, ("POB_SM_COUNT=\"" + g_sm_count_env + "\" is not an integer from " +
                     std::to_string(MIN_SPLIT_SMS) + " to the device's " + std::to_string(g_device_sms) + " SMs")
                        .c_str());
  else if (n == -2)
    pob_fail(where, "device is not compute capability 9.0 (sm_90a build)");
  else
    pob_fail(where, "no sm_90 CUDA device (there is no CPU fallback)");
  return 0;
}
int pob_check_common(const char* where, const void* packed, int sh_deg, int precision) {
  const char* what = nullptr;
  if (!pob::valid_deg(sh_deg))
    what = "sh_deg must be in [-1, 4]";
  else if (!packed)
    what = "packed weights pointer is NULL";
  else if (precision != POB_PREC_FP16 && precision != POB_PREC_FP16X3)
    what = "precision must be POB_PREC_FP16 or POB_PREC_FP16X3";
  if (what) {
    pob_fail(where, what);
    return 0;
  }
  return pob_sms_or_fail(where);
}
pob::FwdParams pob_base_params(const void* packed, int sh_deg, pob::NetDesc net) {
  pob::FwdParams p;
  memset(&p, 0, sizeof(p));
  p.pe = net.pe;
  p.net_act = net.net_act;
  p.sh_deg = sh_deg;
  p.K = pob::K_of(sh_deg);
  p.NH = pob::heads_width(p.K);
  p.w = packed_view(packed, p.K);
  return p;
}
int pob_check_posenc(const char* where, const pob_posenc* posenc, pob::NetDesc& out) {
  out = {pob::POSENC_DEFAULT, pob::NET_RELU};
  if (!posenc) return 0;
  const pob::NetDesc net = {{posenc->min_deg, posenc->max_deg, posenc->legacy_order}, posenc->net_activation};
  if (!pob::posenc_valid(net.pe) || !pob::net_act_valid(net.net_act))
    return pob_fail(where, "posenc needs 0 <= min_deg <= max_deg <= 10 (width 3 + 6 (max_deg - min_deg) <= 63, the "
                           "64-column posenc tile with its constant-one bias column), legacy_order 0 or 1 and "
                           "net_activation one of POB_NET_RELU, POB_NET_ELU, POB_NET_SOFTPLUS, POB_NET_TANH");
  out = net;
  return 0;
}
int pob_check_sigma_activation(const char* where, int sigma_activation) {
  if (sigma_activation != POB_SIGMA_RELU && sigma_activation != POB_SIGMA_SOFTPLUS)
    return pob_fail(where, "sigma_activation must be POB_SIGMA_RELU or POB_SIGMA_SOFTPLUS");
  return 0;
}

extern "C" {

// pob_posenc (pob_render_config.posenc, the *_pe entry points) left the version at 8, which callers pin; a caller
// detects the descriptor by the presence of pob_param_count_pe
int pob_abi_version(void) { return 8; }   // 8: pob_render_config.sigma_activation, pob_eval_points_act; 7:pob_octree_sgd_momentum_step; 6: pob_train_workspace_bytes, pob_loss_and_grad_prec (fp16x3 training); 5: sm_90a, no debug-trace / descriptor-probe entry points; 4: pob_loss_and_grad(mlp0_done_event), pob_adam_update(lr_step_dev)

long long pob_launch_count(void) { return g_launches.load(); }

void pob_timing_enable(int on) {
  drain_slots();
  g_timing = on != 0;
  for (int i = 0; i < POB_PH_COUNT; ++i) {
    g_phase_ms[i] = 0;
    g_phase_n[i] = 0;
  }
}

int pob_timing_read_phases(int n, double* ms_out, long long* launches_out) {
  drain_slots();
  for (int i = 0; i < n && i < POB_PH_COUNT; ++i) {
    if (ms_out) ms_out[i] = g_phase_ms[i];
    if (launches_out) launches_out[i] = g_phase_n[i];
  }
  return POB_PH_COUNT;
}
int pob_timing_read(double* ms_out, long long* launches_out) {
  pob_timing_read_phases(POB_PH_LEGACY_COUNT, ms_out, launches_out);
  return POB_PH_LEGACY_COUNT;
}
const char* pob_last_error(void) { return g_err.c_str(); }
int pob_sm_count(void) { return sm_count(); }

int64_t pob_param_count_pe(int sh_deg, const pob_posenc* posenc) {
  pob::NetDesc net;
  if (!pob::valid_deg(sh_deg) || pob_check_posenc("pob_param_count", posenc, net)) return -1;
  return pob::flat_layout(pob::K_of(sh_deg), pob::posenc_width(net.pe)).total;
}
int64_t pob_param_count(int sh_deg) { return pob_param_count_pe(sh_deg, nullptr); }
int64_t pob_packed_bytes(int sh_deg) {
  if (!pob::valid_deg(sh_deg)) return -1;
  return (int64_t)blob_layout(pob::K_of(sh_deg)).total;
}

int pob_pack_weights_pe(const float* flat_dev, int sh_deg, const pob_posenc* posenc, void* packed_dev, void* stream) {
  if (!pob::valid_deg(sh_deg)) return pob_fail("pob_pack_weights", "sh_deg must be in [-1, 4]");
  pob::NetDesc net;
  if (int e = pob_check_posenc("pob_pack_weights", posenc, net)) return e;
  if (!flat_dev || !packed_dev) return pob_fail("pob_pack_weights", "NULL pointer");
  const int K = pob::K_of(sh_deg);
  const BlobLayout b = blob_layout(K);
  uint8_t* p = static_cast<uint8_t*>(packed_dev);
  cudaStream_t st = (cudaStream_t)stream;
  POB_LAUNCH("pob_pack_weights", POB_PH_OPTIM, st,
             pob::launch_pack_weights(flat_dev, K, pob::posenc_width(net.pe), p + b.w_hi, p + b.w_lo, p + b.wt_hi, st));
  return 0;
}
int pob_pack_weights(const float* flat_dev, int sh_deg, void* packed_dev, void* stream) {
  return pob_pack_weights_pe(flat_dev, sh_deg, nullptr, packed_dev, stream);
}

int pob_eval_points_raw_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc, const float* points_dev,
                           int64_t m, float* raw_rgb_dev, float* raw_sigma_dev, int precision, void* stream) {
  const char* where = "pob_eval_points_raw";
  pob::FwdParams p;
  const int sms = pob_eval_setup(where, packed_dev, sh_deg, posenc, precision, p);
  if (!sms) return 1;
  if (m < 0) return pob_fail(where, "negative point count");
  if (m == 0) return 0;
  if (!points_dev || !raw_sigma_dev) return pob_fail(where, "NULL pointer");
  p.src_mode = pob::SRC_POINTS;
  p.M = m;
  p.points = points_dev;
  p.out_mode = raw_rgb_dev ? pob::OUT_RAW : pob::OUT_SIGMA;
  p.out_rgb = raw_rgb_dev;
  p.out_sigma = raw_sigma_dev;
  cudaStream_t st = (cudaStream_t)stream;
  POB_LAUNCH(where, POB_PH_FWD, st, pob::launch_mlp_fwd(p, precision, sms, st));
  return 0;
}
int pob_eval_points_raw(const void* packed_dev, int sh_deg, const float* points_dev, int64_t m,
                        float* raw_rgb_dev, float* raw_sigma_dev, int precision, void* stream) {
  return pob_eval_points_raw_pe(packed_dev, sh_deg, nullptr, points_dev, m, raw_rgb_dev, raw_sigma_dev, precision,
                                stream);
}

int pob_eval_points_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc, const float* points_dev,
                       const float* viewdirs_dev, int64_t m, float* out_rgbs_dev, int sigma_activation, int precision,
                       void* stream) {
  const char* where = "pob_eval_points";
  pob::FwdParams p;
  const int sms = pob_eval_setup(where, packed_dev, sh_deg, posenc, precision, p);
  if (!sms) return 1;
  if (int e = pob_check_sigma_activation(where, sigma_activation)) return e;
  if (m < 0) return pob_fail(where, "negative point count");
  if (m == 0) return 0;
  if (!points_dev || !out_rgbs_dev) return pob_fail(where, "NULL pointer");
  if (sh_deg >= 0 && !viewdirs_dev)
    return pob_fail(where, "viewdirs required when sh_deg >= 0 (models.py:199)");
  p.src_mode = pob::SRC_POINTS;
  p.M = m;
  p.points = points_dev;
  p.viewdirs = viewdirs_dev ? viewdirs_dev : points_dev;
  p.out_mode = pob::OUT_RGBS;
  p.out_rgbs = reinterpret_cast<float4*>(out_rgbs_dev);
  p.sigma_act = sigma_activation;
  cudaStream_t st = (cudaStream_t)stream;
  POB_LAUNCH(where, POB_PH_FWD, st, pob::launch_mlp_fwd(p, precision, sms, st));
  return 0;
}

int pob_eval_points_act(const void* packed_dev, int sh_deg, const float* points_dev,
                        const float* viewdirs_dev, int64_t m, float* out_rgbs_dev, int sigma_activation,
                        int precision, void* stream) {
  return pob_eval_points_pe(packed_dev, sh_deg, nullptr, points_dev, viewdirs_dev, m, out_rgbs_dev, sigma_activation,
                            precision, stream);
}

int pob_eval_points(const void* packed_dev, int sh_deg, const float* points_dev,
                    const float* viewdirs_dev, int64_t m, float* out_rgbs_dev, int precision,
                    void* stream) {
  return pob_eval_points_act(packed_dev, sh_deg, points_dev, viewdirs_dev, m, out_rgbs_dev, POB_SIGMA_RELU, precision,
                             stream);
}

int pob_eval_cells_mean_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc, const float* points_dev,
                           int64_t n_cells, int samples_per_cell, float* out_dev, int precision, void* stream) {
  const char* where = "pob_eval_cells_mean";
  pob::FwdParams p;
  const int sms = pob_eval_setup(where, packed_dev, sh_deg, posenc, precision, p);
  if (!sms) return 1;
  if (n_cells < 0 || samples_per_cell <= 0) return pob_fail(where, "bad sizes");
  if (n_cells == 0) return 0;
  if (!points_dev || !out_dev) return pob_fail(where, "NULL pointer");
  p.src_mode = pob::SRC_POINTS;
  p.M = n_cells * (int64_t)samples_per_cell;
  p.points = points_dev;
  p.out_mode = pob::OUT_CELL_MEAN;
  p.out_cell = out_dev;
  p.cell_S = samples_per_cell;
  cudaStream_t st = (cudaStream_t)stream;
  POB_CUDA(where, cudaMemsetAsync(out_dev, 0, sizeof(float) * n_cells * (3 * p.K + 1), st));
  POB_LAUNCH(where, POB_PH_FWD, st, pob::launch_mlp_fwd(p, precision, sms, st));
  return 0;
}
int pob_eval_cells_mean(const void* packed_dev, int sh_deg, const float* points_dev, int64_t n_cells,
                        int samples_per_cell, float* out_dev, int precision, void* stream) {
  return pob_eval_cells_mean_pe(packed_dev, sh_deg, nullptr, points_dev, n_cells, samples_per_cell, out_dev,
                                precision, stream);
}

int pob_eval_grid_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc, int reso, int x0, int nx, int ny,
                     int nz, const float offset[3], const float scale[3], float* raw_rgb_dev, float* raw_sigma_dev,
                     int precision, void* stream) {
  const char* where = "pob_eval_grid";
  pob::FwdParams p;
  const int sms = pob_eval_setup(where, packed_dev, sh_deg, posenc, precision, p);
  if (!sms) return 1;
  if (reso <= 0 || (reso & (reso - 1))) return pob_fail(where, "reso must be a power of two (extraction.py:246,290)");
  if (x0 < 0 || nx < 0 || ny < 0 || nz < 0 || x0 + nx > reso || ny > reso || nz > reso)
    return pob_fail(where, "slab out of range");
  if (!offset || !scale || !raw_sigma_dev) return pob_fail(where, "NULL pointer");
  const long long m = (long long)nx * ny * nz;
  if (m == 0) return 0;
  p.src_mode = pob::SRC_GRID;
  p.M = m;
  p.g_reso = reso;
  p.g_x0 = x0;
  p.g_nx = nx;
  p.g_ny = ny;
  p.g_nz = nz;
  for (int a = 0; a < 3; ++a) {
    p.g_offset[a] = offset[a];
    p.g_scale[a] = scale[a];
  }
  p.out_mode = raw_rgb_dev ? pob::OUT_RAW : pob::OUT_SIGMA;
  p.out_rgb = raw_rgb_dev;
  p.out_sigma = raw_sigma_dev;
  cudaStream_t st = (cudaStream_t)stream;
  POB_LAUNCH(where, POB_PH_FWD, st, pob::launch_mlp_fwd(p, precision, sms, st));
  return 0;
}
int pob_eval_grid(const void* packed_dev, int sh_deg, int reso, int x0, int nx, int ny, int nz,
                  const float offset[3], const float scale[3], float* raw_rgb_dev,
                  float* raw_sigma_dev, int precision, void* stream) {
  return pob_eval_grid_pe(packed_dev, sh_deg, nullptr, reso, x0, nx, ny, nz, offset, scale, raw_rgb_dev,
                          raw_sigma_dev, precision, stream);
}

int pob_eval_points_raw_host_pe(const void* packed_dev, int sh_deg, const pob_posenc* posenc,
                                const float* points_host, int64_t m, float* raw_rgb_host, float* raw_sigma_host,
                                int precision) {
  const char* where = "pob_eval_points_raw_host";
  pob::FwdParams p;
  if (!pob_eval_setup(where, packed_dev, sh_deg, posenc, precision, p)) return 1;
  if (m <= 0) return m == 0 ? 0 : pob_fail(where, "negative point count");
  if (!points_host || !raw_sigma_host) return pob_fail(where, "NULL pointer");
  float *d_pts = nullptr, *d_rgb = nullptr, *d_sig = nullptr;
  cudaStream_t st = 0;
  int rc = 0;
  do {
    if (cudaMalloc(&d_pts, sizeof(float) * 3 * m) != cudaSuccess ||
        cudaMalloc(&d_sig, sizeof(float) * m) != cudaSuccess ||
        (raw_rgb_host && cudaMalloc(&d_rgb, sizeof(float) * 3 * p.K * m) != cudaSuccess)) {
      rc = pob_fail(where, "cudaMalloc failed");
      break;
    }
    if (cudaMemcpyAsync(d_pts, points_host, sizeof(float) * 3 * m, cudaMemcpyHostToDevice, st) !=
        cudaSuccess) {
      rc = pob_fail(where, "H2D copy failed");
      break;
    }
    rc = pob_eval_points_raw_pe(packed_dev, sh_deg, posenc, d_pts, m, d_rgb, d_sig, precision, st);
    if (rc) break;
    if (raw_rgb_host)
      cudaMemcpyAsync(raw_rgb_host, d_rgb, sizeof(float) * 3 * p.K * m, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(raw_sigma_host, d_sig, sizeof(float) * m, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) rc = pob_cuda_fail(where, e);
  } while (0);
  cudaFree(d_pts);
  cudaFree(d_rgb);
  cudaFree(d_sig);
  return rc;
}
int pob_eval_points_raw_host(const void* packed_dev, int sh_deg, const float* points_host,
                             int64_t m, float* raw_rgb_host, float* raw_sigma_host,
                             int precision) {
  return pob_eval_points_raw_host_pe(packed_dev, sh_deg, nullptr, points_host, m, raw_rgb_host, raw_sigma_host,
                                     precision);
}

int64_t pob_vanilla_param_count(const pob_posenc* posenc) {
  pob::NetDesc net;
  if (pob_check_posenc("pob_vanilla_param_count", posenc, net)) return -1;
  return pob::vanilla_flat_layout(pob::posenc_width(net.pe)).total;
}
int64_t pob_vanilla_packed_bytes(void) { return int64_t(vanilla_blob_bytes()); }

int pob_pack_vanilla(const float* flat_dev, const pob_posenc* posenc, void* packed_dev, void* stream) {
  const char* where = "pob_pack_vanilla";
  pob::NetDesc net;
  if (int e = pob_check_posenc(where, posenc, net)) return e;
  if (!flat_dev || !packed_dev) return pob_fail(where, "NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  POB_LAUNCH(where, POB_PH_OPTIM, st,
             pob::launch_pack_vanilla(flat_dev, pob::posenc_width(net.pe), static_cast<uint8_t*>(packed_dev), st));
  return 0;
}

int pob_eval_points_vanilla(const void* packed_dev, const pob_posenc* posenc, const pob_view_branch* view, int mlp,
                            const float* points_dev, const float* viewdirs_dev, int64_t m, float* table_dev,
                            float* raw_rgb_dev, float* raw_sigma_dev, float* out_rgbs_dev, int sigma_activation,
                            void* stream) {
  const char* where = "pob_eval_points_vanilla";
  pob::NetDesc net;
  if (!packed_dev) return pob_fail(where, "packed weights pointer is NULL");
  if (int e = pob_check_posenc(where, posenc, net)) return e;
  if (mlp != 0 && mlp != 1) return pob_fail(where, "mlp must be 0 or 1");
  if (int e = pob_check_view(where, view, mlp + 1)) return e;
  if (int e = pob_check_sigma_activation(where, sigma_activation)) return e;
  if (m < 0) return pob_fail(where, "negative point count");
  if (!points_dev || !viewdirs_dev || !table_dev || (!out_rgbs_dev && (!raw_rgb_dev || !raw_sigma_dev)))
    return pob_fail(where, "NULL pointer");
  if (reinterpret_cast<uintptr_t>(table_dev) & 7) return pob_fail(where, "table_dev must be 8-byte aligned");
  const int sms = pob_sms_or_fail(where);
  if (!sms) return 1;
  if (m == 0) return 0;
  pob::FwdParams p = pob_vanilla_params(packed_dev, net, *view, mlp, table_dev);
  p.src_mode = pob::SRC_POINTS;
  p.M = m;
  p.points = points_dev;
  p.out_rgbs = reinterpret_cast<float4*>(out_rgbs_dev);
  p.out_rgb = raw_rgb_dev;
  p.out_sigma = raw_sigma_dev;
  p.sigma_act = sigma_activation;
  cudaStream_t st = (cudaStream_t)stream;
  POB_LAUNCH(where, POB_PH_FWD, st,
             pob::launch_view_table(viewdirs_dev, m, view->deg_view, net.pe.legacy, view->mlp[mlp].w10e_dev,
                                    view->mlp[mlp].c_dev, table_dev, st));
  POB_LAUNCH(where, POB_PH_FWD, st, pob::launch_mlp_fwd_vanilla(p, sms, st));
  return 0;
}

int pob_sample_coarse(const float* z_base_dev, const float* t_rand_dev, int n_rays, int n_samples,
                      float* z_out_dev, void* stream) {
  if (!z_base_dev || !z_out_dev) return pob_fail("pob_sample_coarse", "NULL pointer");
  if (n_rays < 0 || n_samples < 1) return pob_fail("pob_sample_coarse", "bad sizes");
  pob_count_launch();
  POB_CUDA("pob_sample_coarse",
           pob::launch_sample_coarse(z_base_dev, t_rand_dev, n_rays, n_samples, z_out_dev, (cudaStream_t)stream));
  return 0;
}

int pob_draw_uniforms(uint64_t seed, float step, const float* step_dev, float* t_rand_dev, int64_t n_t,
                      float* u_dev, int64_t n_u, float* sp_points_dev, int64_t n_sp, float sp_radius, void* stream) {
  if (n_t < 0 || n_u < 0 || n_sp < 0) return pob_fail("pob_draw_uniforms", "negative size");
  if ((n_t && !t_rand_dev) || (n_u && !u_dev) || (n_sp && !sp_points_dev))
    return pob_fail("pob_draw_uniforms", "NULL pointer");
  if (!pob_sms_or_fail("pob_draw_uniforms")) return 1;
  pob_count_launch();
  POB_CUDA("pob_draw_uniforms", pob::launch_draw_uniforms(seed, step, step_dev, t_rand_dev, n_t, u_dev, n_u,
                                                          sp_points_dev, n_sp, sp_radius, (cudaStream_t)stream));
  return 0;
}

int pob_composite(const float* rgbs_dev, const float* z_dev, const float* dirs_dev, int n_rays, int n_samples,
                  int white_bkgd, float* out_rgb_dev, float* out_disp_dev, float* out_acc_dev,
                  float* out_weights_dev, void* stream) {
  if (!rgbs_dev || !z_dev || !dirs_dev || !out_rgb_dev) return pob_fail("pob_composite", "NULL pointer");
  if (n_rays < 0 || n_samples < 1 || n_samples > pob::MAX_RAY_SAMPLES)
    return pob_fail("pob_composite", "n_samples must be in [1,1024]");
  pob_count_launch();
  POB_CUDA("pob_composite",
           pob::launch_composite_fwd(reinterpret_cast<const float4*>(rgbs_dev), z_dev, dirs_dev, n_rays, n_samples,
                                     white_bkgd, out_rgb_dev, out_disp_dev, out_acc_dev, out_weights_dev,
                                     (cudaStream_t)stream));
  return 0;
}

int pob_composite_bwd(const float* rgbs_dev, const float* z_dev, const float* dirs_dev, const float* comp_rgb_dev,
                      const float* pixels_dev, int n_rays, int n_samples, int white_bkgd, float gscale,
                      float* g_out_dev, float* sq_err_sum_dev, void* stream) {
  if (!rgbs_dev || !z_dev || !dirs_dev || !comp_rgb_dev || !pixels_dev || !g_out_dev)
    return pob_fail("pob_composite_bwd", "NULL pointer");
  if (n_rays < 0 || n_samples < 1 || n_samples > pob::MAX_RAY_SAMPLES)
    return pob_fail("pob_composite_bwd", "n_samples must be in [1,1024]");
  pob_count_launch();
  POB_CUDA("pob_composite_bwd",
           pob::launch_composite_bwd(reinterpret_cast<const float4*>(rgbs_dev), z_dev, dirs_dev, comp_rgb_dev,
                                     pixels_dev, n_rays, n_samples, white_bkgd, gscale, pob::SIGMA_RELU,
                                     reinterpret_cast<float4*>(g_out_dev), sq_err_sum_dev, (cudaStream_t)stream));
  return 0;
}

int pob_sample_pdf(const float* z_coarse_dev, const float* weights_dev, const float* u_dev, int u_per_ray,
                   int n_rays, int n_coarse, int n_fine, float* z_out_dev, void* stream) {
  if (!z_coarse_dev || !weights_dev || !u_dev || !z_out_dev) return pob_fail("pob_sample_pdf", "NULL pointer");
  if (n_coarse < 3 || n_fine < 1 || n_coarse + n_fine > pob::MAX_RAY_SAMPLES)
    return pob_fail("pob_sample_pdf", "need n_coarse >= 3 and n_coarse + n_fine <= 1024");
  pob_count_launch();
  POB_CUDA("pob_sample_pdf", pob::launch_sample_pdf(z_coarse_dev, weights_dev, u_dev, u_per_ray, n_rays, n_coarse,
                                                    n_fine, z_out_dev, (cudaStream_t)stream));
  return 0;
}


int64_t pob_quantize_workspace_bytes(int64_t n_basis, int64_t n, int weighted) {
  if (n_basis < 1 || n < 0 || n > INT32_MAX || n_basis * n >= (int64_t(1) << 40)) return -1;
  return int64_t(pob::quant_layout(n_basis, n, weighted != 0).bytes);
}

int pob_quantize_median_cut(const float* points_dev, const double* weights_dev, int64_t n_basis, int64_t n, int bits,
                            float* palette_dev, uint16_t* map_dev, void* workspace_dev, int64_t workspace_bytes,
                            void* stream) {
  const char* W = "pob_quantize_median_cut";
  if (bits < 0 || bits > pob::QUANT_MAX_BITS) return pob_fail(W, "bits must be in [0, 16] (the map is uint16)");
  if (n_basis < 1 || n < 0 || n > INT32_MAX || n_basis * n >= (int64_t(1) << 40))
    return pob_fail(W, "need n_basis >= 1, 0 <= n < 2^31 (uint32 point indices) and n_basis * n < 2^40");
  if (!palette_dev || (n > 0 && (!points_dev || !map_dev || !workspace_dev)))
    return pob_fail(W, "NULL pointer");
  if (reinterpret_cast<uintptr_t>(workspace_dev) % 256 != 0) return pob_fail(W, "workspace is not 256-byte aligned");
  if (n > 0 && workspace_bytes < pob_quantize_workspace_bytes(n_basis, n, weights_dev != nullptr))
    return pob_fail(W, "workspace is smaller than pob_quantize_workspace_bytes");
  const int sms = pob_sms_or_fail(W);
  if (!sms) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {   // median_cut of no points: an all-zero palette, an empty map
    POB_CUDA(W, cudaMemsetAsync(palette_dev, 0, size_t(n_basis) * (size_t(1) << bits) * 3 * sizeof(float), st));
    return 0;
  }
  return pob::launch_quantize(points_dev, weights_dev, n, int(n_basis), bits, palette_dev, map_dev, workspace_dev,
                              sms, st);
}

}  // extern "C"
