// C-ABI of the batched MAPDN voltage-control env (include/mapdn_b200.h): handle management,
// one-off Ybus assembly + symbolic analysis of the radial network, kernel launches.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "../../include/mapdn_b200.h"
#include "env_kernel.cuh"

// kernel<<<grid, block, smem, stream>>>(args...); under MAPDN_HOST_EMU (tests/emu: the library compiled with g++ for the
// CPU SIMT emulation, test infrastructure) the same launch runs on OS threads
#ifdef MAPDN_HOST_EMU
#define MAPDN_LAUNCH(kernel, grid, block, smem, stream, ...) emu::launch(kernel, grid, block, smem, stream, __VA_ARGS__)
#else
#define MAPDN_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<grid, block, smem, stream>>>(__VA_ARGS__)
#endif

namespace mapdn {

static thread_local std::string g_last_error;

static mapdn_status fail(mapdn_status st, const std::string& msg) {
  g_last_error = msg;
  return st;
}

#define MAPDN_CUDA(expr)                                                                        \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess)                                                                      \
      return fail(MAPDN_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));          \
  } while (0)
#define MAPDN_TRY(expr)                                                                         \
  do {                                                                                          \
    const mapdn_status _s = (expr);                                                             \
    if (_s != MAPDN_OK) return _s;                                                              \
  } while (0)

// Every entry point runs on the handle's device and leaves the calling thread's current device as it found it
// (the caller -- PyTorch, CuPy -- tracks the current device through the CUDA runtime).
struct DeviceGuard {
  int prev = -1, dev = -1;
  cudaError_t err = cudaSuccess;
  explicit DeviceGuard(int device) : dev(device) {
    err = cudaGetDevice(&prev);
    if (err == cudaSuccess && prev != dev) err = cudaSetDevice(dev);
  }
  ~DeviceGuard() { if (prev >= 0 && prev != dev) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};
#define MAPDN_ON_DEVICE(device)          \
  DeviceGuard _device_guard(device);     \
  MAPDN_CUDA(_device_guard.err)

// ------------------------------------------------------------------------------------------------
// Ybus assembly on the device (PYPOWER makeYbus, SURVEY Appendix A.3). Runs once per handle: the
// topology never changes between env steps (the reference rebuilds Ybus inside every pp.runpp).
// ------------------------------------------------------------------------------------------------
__global__ void ybus_branch_kernel(int n_br, const double* __restrict__ r, const double* __restrict__ x,
                                   const double* __restrict__ b, const double* __restrict__ g,
                                   const double* __restrict__ tap, const double* __restrict__ shift_deg,
                                   const unsigned char* __restrict__ status, double* __restrict__ ybr /*[n_br,8]*/) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_br) return;
  const double st = status[k] ? 1.0 : 0.0;
  const double den = r[k] * r[k] + x[k] * x[k];
  // Ys = stat / (r + jx); an out-of-service branch contributes exactly zero (also when r = x = 0)
  const double ys_g = status[k] ? r[k] / den : 0.0, ys_b = status[k] ? -x[k] / den : 0.0;
  const double ytt_g = ys_g + 0.5 * st * g[k], ytt_b = ys_b + 0.5 * st * b[k];   // Ys + j*Bc/2, Bc = b - jg
  const double t = (tap[k] == 0.0) ? 1.0 : tap[k];
  double sn, cs;
  sincos(shift_deg[k] * (3.14159265358979323846 / 180.0), &sn, &cs);
  const double tr = t * cs, ti = t * sn;                                  // tau = tap * exp(j*shift)
  const double t2 = tr * tr + ti * ti;
  // Yff = Ytt / (tau conj(tau)); Yft = -Ys / conj(tau); Ytf = -Ys / tau
  double* o = ybr + 8 * k;
  o[0] = ytt_g / t2; o[1] = ytt_b / t2;
  // -Ys/conj(tau) = -Ys * tau / |tau|^2
  o[2] = -(ys_g * tr - ys_b * ti) / t2; o[3] = -(ys_g * ti + ys_b * tr) / t2;
  // -Ys/tau = -Ys * conj(tau) / |tau|^2
  o[4] = -(ys_g * tr + ys_b * ti) / t2; o[5] = -(-ys_g * ti + ys_b * tr) / t2;
  o[6] = ytt_g; o[7] = ytt_b;
}

__global__ void ybus_diag_kernel(int n_bus, int n_br, const int* __restrict__ from, const int* __restrict__ to,
                                 const double* __restrict__ ybr, const double* __restrict__ gs,
                                 const double* __restrict__ bs, double inv_base, double* __restrict__ ydiag /*[n_bus,2]*/) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_bus) return;
  double g = gs[i] * inv_base, b = bs[i] * inv_base;                      // Ysh = (GS + jBS)/baseMVA
  for (int k = 0; k < n_br; ++k) {
    if (from[k] == i) { g += ybr[8 * k + 0]; b += ybr[8 * k + 1]; }
    if (to[k] == i) { g += ybr[8 * k + 6]; b += ybr[8 * k + 7]; }
  }
  ydiag[2 * i] = g; ydiag[2 * i + 1] = b;
}

// ---- small gather kernels over the env state kept in HBM ----
__global__ void scale_copy_kernel(long long n, const double* __restrict__ in, double scale, double* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = in[i] * scale;
}
__global__ void int_to_double_kernel(long long n, const int* __restrict__ in, double* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = static_cast<double>(in[i]);
}
__global__ void i64_to_double_kernel(long long n, const long long* __restrict__ in, double* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = static_cast<double>(in[i]);
}

__global__ void get_obs_kernel(const __grid_constant__ Params p) {
  const int tot = p.n_sgen * p.obs_dim;
  const long long gid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (gid >= static_cast<long long>(p.nb) * tot) return;
  const int env = static_cast<int>(gid / tot), idx = static_cast<int>(gid - static_cast<long long>(env) * tot);
  p.obs[gid] = obs_entry(p, env, idx);
}

// history > 1, after a reset launch: frame 0 of the new episode of every reset env (mask) into ring slot 0
__global__ void reset_frame_kernel(const __grid_constant__ Params p) {
  const int tot = p.n_sgen * p.obs_dim;
  const long long gid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (gid >= static_cast<long long>(p.nb) * tot) return;
  const int env = static_cast<int>(gid / tot), idx = static_cast<int>(gid - static_cast<long long>(env) * tot);
  if (p.mask != nullptr && !p.mask[env]) return;
  // one thread per entry: lane idx of tot lanes, so write_frame0's loop runs once
  write_frame0(p, env, idx, tot, [&](int i) { return obs_entry(p, env, i); });
}

// mapdn_get_obs_stacked: the stacked rows from the ring and the step counters - the rule the step kernel applies in its
// epilogue, one 16-byte piece (even obs_dim) or one entry per thread
__global__ void obs_stacked_kernel(const __grid_constant__ Params p) {
  const int per = (p.obs_dim & 1) == 0 ? 2 : 1;
  const int row = p.n_sgen * p.history * p.obs_dim / per;                  // pieces per env
  const long long gid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (gid >= static_cast<long long>(p.nb) * row) return;
  const int env = static_cast<int>(gid / row), c = static_cast<int>(gid - static_cast<long long>(env) * row);
  const double* ring = p.hist + static_cast<size_t>(env) * p.history * p.n_sgen * p.obs_dim;
  // the newest frame is in the ring too: write_stacked_row reads it there, restricted to this thread's piece
  write_stacked_row(p, p.obs_stacked, env, p.steps[env] - 1, c, row, [&](int i) {
    return ring[static_cast<size_t>((p.steps[env] - 1) % p.history) * p.n_sgen * p.obs_dim + i];
  });
}

// get_state() (reference :213-230): [P_bus | Q_bus | pv | q | vm | va(deg)] restricted to state_space
__global__ void get_state_kernel(const __grid_constant__ Params p) {
  const long long gid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (gid >= static_cast<long long>(p.nb) * p.state_dim) return;
  const int env = static_cast<int>(gid / p.state_dim), idx = static_cast<int>(gid - static_cast<long long>(env) * p.state_dim);
  const size_t eN = static_cast<size_t>(env) * p.n_bus, eG = static_cast<size_t>(env) * p.n_sgen;
  const unsigned src = __ldg(p.state_src + idx);
  const int kind = static_cast<int>(src >> 28), ix = static_cast<int>(src & 0x0FFFFFFFu);
  double v = 0.0;
  if (kind == OBS_PBUS) v = p.res_p[eN + ix];
  else if (kind == OBS_QBUS) v = p.res_q[eN + ix];
  else if (kind == OBS_PV) v = p.cur_pv[eG + ix];
  else if (kind == OBS_QSG) v = p.cur_q[eG + ix];
  else if (kind == OBS_VM) v = p.res_vm[eN + ix];
  else if (kind == OBS_VA_DEG) v = p.res_va[eN + ix] * 57.295779513082320876798;
  p.state[gid] = v;
}

// mapdn_record: the tester record row of every env from the state in HBM (the six get_field columns side by side)
__global__ void record_kernel(const __grid_constant__ Params p) {
  const int ng = p.n_sgen, n = p.n_bus, row = 2 * ng + 3 * n + p.n_line;
  const long long gid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (gid >= static_cast<long long>(p.nb) * row) return;
  const int env = static_cast<int>(gid / row), k = static_cast<int>(gid - static_cast<long long>(env) * row);
  const size_t eN = static_cast<size_t>(env) * n, eG = static_cast<size_t>(env) * ng;
  double v;
  if (k < ng) v = p.cur_pv[eG + k];
  else if (k < 2 * ng) v = p.cur_q[eG + k - ng];
  else if (k < 2 * ng + n) v = p.res_p[eN + k - 2 * ng];
  else if (k < 2 * ng + 2 * n) v = p.res_q[eN + k - 2 * ng - n];
  else if (k < 2 * ng + 3 * n) v = p.res_vm[eN + k - 2 * ng - 2 * n];
  else v = p.res_pl[static_cast<size_t>(env) * p.n_line + k - 2 * ng - 3 * n];
  p.record[static_cast<size_t>(env) * p.record_stride + k] = v;
}

// ---- env state snapshots (mapdn_snapshot / mapdn_restore) ----
// Segment s of the state: env b's bytes[s] bytes at base[s] + b * bytes[s]. A snapshot row packs the segments in the
// order of the header's list, segment s at row offset off[s] (16-byte aligned); off[MAPDN_N_SNAPSHOT] is the row size.
struct SnapLayout {
  unsigned char* base[MAPDN_N_SNAPSHOT];
  int bytes[MAPDN_N_SNAPSHOT];
  long long off[MAPDN_N_SNAPSHOT + 1];
};

// One segment of one row by one warp, in T-wide pieces (bytes and the padded length are multiples of sizeof(T)). The
// snapshot direction also zeroes the padding, so that equal states give equal rows.
template <class T, bool RESTORE>
__device__ __forceinline__ void copy_segment(unsigned char* state, unsigned char* row, int bytes, int padded, int lane) {
  T* __restrict__ st = reinterpret_cast<T*>(state);      // a row never overlaps the state: loads may run ahead of stores
  T* __restrict__ rw = reinterpret_cast<T*>(row);
  const int n = bytes / static_cast<int>(sizeof(T));
  if (RESTORE) {
    for (int i = lane; i < n; i += 32) st[i] = rw[i];
  } else {
    for (int i = lane; i < n; i += 32) rw[i] = st[i];
    for (int i = n + lane; i < padded / static_cast<int>(sizeof(T)); i += 32) rw[i] = T{};
  }
}

// Gather (state -> rows) or scatter (RESTORE: rows -> state). Warp w moves segment w mod MAPDN_N_SNAPSHOT of row
// k = w / MAPDN_N_SNAPSHOT between env idx[k] (env k without a list) and buf + k * off[MAPDN_N_SNAPSHOT]: 16-byte accesses
// when the segment's size per env is a multiple of 16 (its start in the state array is then 16-byte aligned too), else
// 8- or 4-byte ones. A row whose env is outside [0, nb) is skipped.
template <bool RESTORE>
__global__ void snapshot_kernel(const __grid_constant__ SnapLayout sl, const int* __restrict__ idx, int n, int nb,
                                unsigned char* __restrict__ buf) {
  const long long w = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = static_cast<int>(threadIdx.x & 31);
  if (w >= static_cast<long long>(n) * MAPDN_N_SNAPSHOT) return;
  const int k = static_cast<int>(w / MAPDN_N_SNAPSHOT), s = static_cast<int>(w - static_cast<long long>(k) * MAPDN_N_SNAPSHOT);
  const int env = idx ? __ldg(idx + k) : k;
  if (env < 0 || env >= nb) return;
  const int bytes = sl.bytes[s], padded = static_cast<int>(sl.off[s + 1] - sl.off[s]);
  unsigned char* state = sl.base[s] + static_cast<size_t>(env) * bytes;
  unsigned char* row = buf + static_cast<size_t>(k) * sl.off[MAPDN_N_SNAPSHOT] + sl.off[s];
  if (bytes % 16 == 0) copy_segment<int4, RESTORE>(state, row, bytes, padded, lane);
  else if (bytes % 8 == 0) copy_segment<long long, RESTORE>(state, row, bytes, padded, lane);
  else copy_segment<int, RESTORE>(state, row, bytes, padded, lane);
}

}  // namespace mapdn

using namespace mapdn;

// ------------------------------------------------------------------------------------------------
struct mapdn_env {
  int device = 0;
  mapdn_cfg cfg{};
  mapdn_dims dims{};
  Params base{};                       // static + state pointers; io fields filled per call
  std::vector<void*> allocs;           // everything cudaMalloc'ed
  int G = 8, threads = 128, epb = 16, smem = 0, helper_threads = 32;
  int max_blocks_step[2][2][2] = {};   // persistent grid of the MODE_STEP instantiations [auto-reset][observation history][tester records]
  bool dense = false;                  // meshed net: dense-LU fallback solver
  long long launches = 0;
  // Ybus pieces kept for the test hook
  std::vector<double> ybr, ydiag;
  std::vector<int> br_from, br_to;
  // device-side staging buffers of the *_host entry points
  double *d_stage_actions = nullptr, *d_stage_reward = nullptr, *d_stage_info = nullptr, *d_stage_obs = nullptr;
  unsigned char* d_stage_term = nullptr;
  int obs_zero_off = 0;                // slab offset of the constant-zero slot the obs padding reads
  std::vector<int> agent_len, agent_off;   // compact observation rows: true length / offset of every agent's block
  int compact_row = 0;                 // entries per compact row (sum of agent_len, rounded up to a multiple of 4)
  std::vector<const void*> pinned_ok;  // host buffers already verified as pinned (mapdn_step_host_pinned)
};

namespace {

template <class T>
mapdn_status dev_upload(mapdn_env* e, const std::vector<T>& v, const T** out) {
  void* d = nullptr;
  const size_t bytes = std::max<size_t>(v.size() * sizeof(T), 16);
  MAPDN_CUDA(cudaMalloc(&d, bytes));
  e->allocs.push_back(d);
  if (!v.empty()) MAPDN_CUDA(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  *out = static_cast<const T*>(d);
  return MAPDN_OK;
}

template <class T>
mapdn_status dev_alloc(mapdn_env* e, size_t count, T** out) {
  void* d = nullptr;
  const size_t bytes = std::max<size_t>(count * sizeof(T), 16);
  MAPDN_CUDA(cudaMalloc(&d, bytes));
  MAPDN_CUDA(cudaMemset(d, 0, bytes));
  e->allocs.push_back(d);
  *out = static_cast<T*>(d);
  return MAPDN_OK;
}

template <class T>
std::vector<T> vec_or(const T* p, size_t n, T fill) {
  return p ? std::vector<T>(p, p + n) : std::vector<T>(n, fill);
}

using KernelFn = void (*)(const Params);
constexpr int kHelperPairsPerWarp = 256;   // Box-Muller pairs of a CTA round per helper warp

template <int G, bool DENSE>
KernelFn kernel_for_mode(int mode, bool record, bool hist, bool autoreset) {
  switch (mode) {
    case MODE_SOLVE: return env_kernel<G, MODE_SOLVE, DENSE>;
    case MODE_STEP:
      if (autoreset) return hist ? env_kernel<G, MODE_STEP, DENSE, false, true, true> : env_kernel<G, MODE_STEP, DENSE, false, false, true>;
      if (hist) return record ? env_kernel<G, MODE_STEP, DENSE, true, true> : env_kernel<G, MODE_STEP, DENSE, false, true>;
      return record ? env_kernel<G, MODE_STEP, DENSE, true> : env_kernel<G, MODE_STEP, DENSE>;
    case MODE_DROOP: return env_kernel<G, MODE_DROOP, DENSE>;
    default: return env_kernel<G, MODE_RESET, DENSE>;
  }
}

// record: the MODE_STEP instantiation that also writes the tester record rows (mapdn_step_record); hist: the one that
// also records observation frames (handles with history); autoreset: the one that also resets the envs that terminated
// (mapdn_step_autoreset, never with record)
KernelFn kernel_for(int G, int mode, bool dense = false, bool record = false, bool hist = false, bool autoreset = false) {
  if (dense) return kernel_for_mode<32, true>(mode, record, hist, autoreset);
  switch (G) {
    case 4: return kernel_for_mode<4, false>(mode, record, hist, autoreset);
    case 8: return kernel_for_mode<8, false>(mode, record, hist, autoreset);
    case 16: return kernel_for_mode<16, false>(mode, record, hist, autoreset);
    case 64: return kernel_for_mode<64, false>(mode, record, hist, autoreset);
    case 128: return kernel_for_mode<128, false>(mode, record, hist, autoreset);
    default: return kernel_for_mode<32, false>(mode, record, hist, autoreset);
  }
}

// smem per env in double2 units: (npq + 1) node records of 9 double2, sgen p/q, scratch of ng + 2 nl
// doubles. For G = 4 two envs share a quarter-warp of a 128-bit access, so their slabs must start
// 64 B apart modulo 128 B.
// The prologue stages 2 n_load scaled load values per env. They fit the Newton fields of the node records (12 dead
// doubles per record, see env_kernel.cuh) unless the net has very many loads per bus.
bool stage_fits_records(int npq, int nl) { return 2 * nl <= 12 * (npq + 2); }

// scratch doubles per env: next pv row / droop voltages [n_sgen], the partial sums per warp of the multi-warp group
// reductions, and the staged loads when they do not fit the records
int scratch_doubles_for(int ng, int nl, int G, bool stage_rec) {
  return ng + (G > 32 ? 10 * (G / 32) : 0) + (stage_rec ? 0 : 2 * nl);
}

int env_stride2_for(int npq, int ng, int nl, int G, bool stage_rec) {
  int stride = kNodeArrays2 * (npq + 2) + ng + (scratch_doubles_for(ng, nl, G, stage_rec) + 1) / 2;
  if (G == 4) while ((stride * 16) % 128 != 64) ++stride;
  return stride;
}

mapdn_status launch_env_kernel(mapdn_env* e, int mode, Params& p, cudaStream_t st, bool autoreset = false) {
  const bool record = mode == MODE_STEP && p.record != nullptr;
  const bool hist = mode == MODE_STEP && p.history > 1;      // every step of a handle with history records its frame
  KernelFn fn = kernel_for(e->G, mode, e->dense, record, hist, autoreset);
  const int needed = (p.nb + e->epb - 1) / e->epb;
  int grid = std::min(needed, std::max(1, e->max_blocks_step[autoreset][hist][record]));
  const int rounds = (needed + grid - 1) / grid;
  grid = (needed + rounds - 1) / rounds;       // balance the persistent loop
#ifdef MAPDN_PROFILE
  static long long* d_prof = nullptr;
  if (!d_prof) cudaMalloc(&d_prof, 16 * sizeof(long long));
  cudaMemset(d_prof, 0, 16 * sizeof(long long));
  p.prof = d_prof;
#endif
  p.helper_threads = e->helper_threads;
  MAPDN_LAUNCH(fn, grid, e->threads + (mode == MODE_STEP ? e->helper_threads : 0), e->smem, st, p);   // MODE_STEP: + helper warps
  MAPDN_CUDA(cudaGetLastError());
  e->launches++;
#ifdef MAPDN_PROFILE
  {
    long long hp[16];
    cudaDeviceSynchronize();
    cudaMemcpy(hp, d_prof, sizeof(hp), cudaMemcpyDeviceToHost);
    static const char* nm[12] = {"-", "setup+prologue", "init/update", "edges", "F/diag", "elim", "backsub", "reload+slack",
                                 "q+nextrow", "BP/OP+bus+lines", "reward/info", "obs/state"};
    long long tot = 0;
    for (int k = 0; k < 12; ++k) tot += hp[k];
    fprintf(stderr, "[prof mode=%d nb=%d] total %lld cyc:", mode, p.nb, tot);
    for (int k = 1; k < 12; ++k) fprintf(stderr, " %s=%lld", nm[k], hp[k]);
    if (hp[14] > 0)
      fprintf(stderr, " | forward-sweep step: %lld executions in %lld solves, load wait %lld + arithmetic %lld cyc per step",
              hp[14], hp[15], hp[12] / hp[14], hp[13] / hp[14]);
    fprintf(stderr, "\n");
  }
#endif
  return MAPDN_OK;
}

constexpr auto nothing = [](cudaStream_t) { return MAPDN_OK; };   // before / after of a step that needs neither

// Outputs of the reset that mapdn_step_autoreset runs after the step (any may be NULL)
struct AutoReset { double* obs; double* obs_stacked; uint8_t* ok; };

// The MODE_STEP launch behind the eight mapdn_step* entry points, after each has checked its own pointers: refuses a
// handle without a profile store, then runs on the handle's device. The kernel reads the actions from and writes its
// outputs to the given buffers (info / obs / record may be NULL; obs holds floats when obs_f32). before(st) runs ahead of
// the launch and may refuse the call or enqueue what the kernel reads; after(st) enqueues what follows the kernel. With
// `autoreset`, the launch also resets the envs that terminate in the step.
template <class Before, class After>
mapdn_status step(mapdn_env* e, const double* actions, int32_t add_noise, double* reward, uint8_t* term, double* info,
                  void* obs, bool obs_f32, void* stream, Before before, After after, int obs_skip_off = -1,
                  int obs_compact_len = 0, double* record = nullptr, int64_t record_stride = 0,
                  double* obs_stacked = nullptr, const AutoReset* autoreset = nullptr) {
  if (!e->base.prof_pv) return fail(MAPDN_ERR_INVALID, "handle was created without a profile store");
  MAPDN_ON_DEVICE(e->device);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  mapdn_status s = before(st);
  if (s != MAPDN_OK) return s;
  Params p = e->base;
  p.actions = actions; p.add_noise = add_noise; p.reward = reward; p.term = term; p.info = info;
  p.obs = obs_f32 ? nullptr : static_cast<double*>(obs); p.obs32 = obs_f32 ? static_cast<float*>(obs) : nullptr;
  p.obs_skip_off = obs_skip_off; p.obs_compact_len = obs_compact_len; p.record = record; p.record_stride = record_stride;
  p.obs_stacked = obs_stacked;
  if (autoreset) { p.reset_obs = autoreset->obs; p.reset_obs_stacked = autoreset->obs_stacked; p.reset_ok = autoreset->ok; }
  s = launch_env_kernel(e, MODE_STEP, p, st, autoreset != nullptr);
  return s != MAPDN_OK ? s : after(st);
}

// mapdn_step_host / mapdn_step_host_f32obs: H2D of the actions, the step into the staging buffers, D2H of the outputs
// asked for, stream synchronisation. The fp64 staging buffer of the observations also holds them as floats.
mapdn_status step_staged(mapdn_env* e, const double* actions_host, int32_t add_noise, double* reward_host,
                         uint8_t* terminated_host, double* info_host, void* obs_host, bool obs_f32, void* stream) {
  if (!e || !actions_host || !reward_host || !terminated_host) return fail(MAPDN_ERR_INVALID, "null argument");
  const size_t B = e->dims.batch, ng = e->dims.n_sgen;
  const size_t obs_bytes = B * ng * e->dims.obs_dim * (obs_f32 ? sizeof(float) : sizeof(double));
  auto h2d = [&](cudaStream_t st) {
    MAPDN_CUDA(cudaMemcpyAsync(e->d_stage_actions, actions_host, B * ng * sizeof(double), cudaMemcpyHostToDevice, st));
    return MAPDN_OK;
  };
  auto d2h = [&](cudaStream_t st) {
    MAPDN_CUDA(cudaMemcpyAsync(reward_host, e->d_stage_reward, B * sizeof(double), cudaMemcpyDeviceToHost, st));
    MAPDN_CUDA(cudaMemcpyAsync(terminated_host, e->d_stage_term, B, cudaMemcpyDeviceToHost, st));
    if (info_host) MAPDN_CUDA(cudaMemcpyAsync(info_host, e->d_stage_info, B * MAPDN_N_INFO * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (obs_host) MAPDN_CUDA(cudaMemcpyAsync(obs_host, e->d_stage_obs, obs_bytes, cudaMemcpyDeviceToHost, st));
    MAPDN_CUDA(cudaStreamSynchronize(st));
    return MAPDN_OK;
  };
  return step(e, e->d_stage_actions, add_noise, e->d_stage_reward, e->d_stage_term, info_host ? e->d_stage_info : nullptr,
              obs_host ? e->d_stage_obs : nullptr, obs_f32, stream, h2d, d2h);
}

// The kernel of the pinned and compact paths reads and writes the host buffers themselves: each must be page-locked host
// memory with unified addressing (device address = host address). Buffers that passed are remembered.
mapdn_status check_pinned(mapdn_env* e, const void* const (&host)[5]) {
  static const char* const what[5] = {"actions_host", "reward_host", "terminated_host", "info_host", "obs_host"};
  for (int k = 0; k < 5; ++k) {
    if (!host[k] || std::find(e->pinned_ok.begin(), e->pinned_ok.end(), host[k]) != e->pinned_ok.end()) continue;
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, host[k]) != cudaSuccess || at.type != cudaMemoryTypeHost || at.devicePointer != host[k]) {
      cudaGetLastError();
      return fail(MAPDN_ERR_INVALID, std::string(what[k]) + ": not page-locked host memory with unified addressing "
                                     "(cudaHostAlloc / cudaHostRegister it, or use mapdn_step_host)");
    }
    if (e->pinned_ok.size() < 64) e->pinned_ok.push_back(host[k]);
  }
  return MAPDN_OK;
}

// One flat gather launch over n items in 256-thread blocks, on the handle's device, counted with its launches
template <class Kernel, class... Args>
mapdn_status gather(mapdn_env* e, Kernel kernel, long long n, void* stream, Args... args) {
  if (n == 0) return MAPDN_OK;
  MAPDN_ON_DEVICE(e->device);
  MAPDN_LAUNCH(kernel, static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream), args...);
  MAPDN_CUDA(cudaGetLastError());
  e->launches++;
  return MAPDN_OK;
}

// The snapshot segments of the handle's state arrays, in the header's order (MAPDN_N_SNAPSHOT): the ring only with history
SnapLayout snapshot_layout(const mapdn_env* e) {
  const Params& p = e->base;
  const long long n = p.n_bus, ng = p.n_sgen, nl = p.n_load;
  void* const base[MAPDN_N_SNAPSHOT] = {p.cur_pl, p.cur_ql, p.cur_pv, p.cur_q, p.res_vm, p.res_va, p.res_p, p.res_q,
                                        p.res_pl, p.sum_rewards, p.start_row, p.steps, p.episode, p.nr_iters, p.hist};
  const long long bytes[MAPDN_N_SNAPSHOT] = {8 * nl, 8 * nl, 8 * ng, 8 * ng, 8 * n, 8 * n, 8 * n, 8 * n, 8LL * p.n_line,
                                             8, 8, 4, 4, 4, p.history > 1 ? 8LL * p.history * ng * p.obs_dim : 0};
  SnapLayout sl{};
  for (int s = 0; s < MAPDN_N_SNAPSHOT; ++s) {
    sl.base[s] = static_cast<unsigned char*>(base[s]);
    sl.bytes[s] = static_cast<int>(bytes[s]);
    sl.off[s + 1] = sl.off[s] + (bytes[s] + 15) / 16 * 16;
  }
  return sl;
}

// mapdn_snapshot / mapdn_restore: the argument checks of both, then one snapshot_kernel launch (one warp per row and
// segment)
mapdn_status snapshot_copy(mapdn_env* e, const int32_t* idx, int32_t n, const void* buf, void* stream, bool restore) {
  if (!e || !buf) return fail(MAPDN_ERR_INVALID, "null argument");
  if (!e->base.prof_pv) return fail(MAPDN_ERR_INVALID, "handle was created without a profile store");
  if (n <= 0 || n > e->base.nb) return fail(MAPDN_ERR_INVALID, "n must be in [1, batch]");
  if (!idx && n != e->base.nb) return fail(MAPDN_ERR_INVALID, "without an index list n must equal the batch");
  if (reinterpret_cast<uintptr_t>(buf) % 16 != 0) return fail(MAPDN_ERR_INVALID, "snapshot buffer not 16-byte aligned");
  const SnapLayout sl = snapshot_layout(e);
  unsigned char* rows = static_cast<unsigned char*>(const_cast<void*>(buf));
  const long long threads = 32LL * MAPDN_N_SNAPSHOT * n;
  return restore ? gather(e, snapshot_kernel<true>, threads, stream, sl, idx, n, e->base.nb, rows)
                 : gather(e, snapshot_kernel<false>, threads, stream, sl, idx, n, e->base.nb, rows);
}

// ------------------------------------------------------------------------------------------------
// mapdn_create, stage by stage. Between the Ybus assembly and the kernel attributes every stage is host arithmetic on
// plain structs: no CUDA call, no handle. Each takes what it reads by const reference, so the order of the calls in
// mapdn_create is the only order dependency.
// ------------------------------------------------------------------------------------------------
mapdn_status validate_create_args(const mapdn_net_desc* net, const mapdn_profile_desc* prof, const mapdn_cfg* cfg) {
  const int n = net->n_bus, nbr = net->n_branch, nl = net->n_load, ng = net->n_sgen;
  if (n < 2 || n > 65000) return fail(MAPDN_ERR_INVALID, "n_bus must be in [2, 65000]");
  if (nbr < 1 || nl < 0 || ng < 1) return fail(MAPDN_ERR_INVALID, "need >=1 branch and >=1 sgen");
  if (cfg->batch < 1) return fail(MAPDN_ERR_INVALID, "batch must be >= 1");
  if (!net->br_from || !net->br_to || !net->br_r || !net->br_x || !net->sgen_bus || !net->sgen_zone ||
      !net->bus_zone || (nl > 0 && !net->load_bus))
    return fail(MAPDN_ERR_INVALID, "missing required network array");
  if (net->slack_bus < 0 || net->slack_bus >= n) return fail(MAPDN_ERR_INVALID, "slack_bus out of range");
  if (!(net->base_mva > 0)) return fail(MAPDN_ERR_INVALID, "base_mva must be positive");
  if (cfg->barrier < 0 || cfg->barrier > 4) return fail(MAPDN_ERR_INVALID, "unknown voltage barrier");
  if (cfg->lanes_per_env != 0 && cfg->lanes_per_env != 4 && cfg->lanes_per_env != 8 && cfg->lanes_per_env != 16 &&
      cfg->lanes_per_env != 32 && cfg->lanes_per_env != 64 && cfg->lanes_per_env != 128)
    return fail(MAPDN_ERR_INVALID, "lanes_per_env must be 0, 4, 8, 16, 32, 64 or 128");
  for (int k = 0; k < nbr; ++k)
    if (net->br_from[k] < 0 || net->br_from[k] >= n || net->br_to[k] < 0 || net->br_to[k] >= n ||
        net->br_from[k] == net->br_to[k])
      return fail(MAPDN_ERR_INVALID, "branch endpoint out of range");
  for (int l = 0; l < nl; ++l)
    if (net->load_bus[l] < 0 || net->load_bus[l] >= n) return fail(MAPDN_ERR_INVALID, "load_bus out of range");
  for (int j = 0; j < ng; ++j)
    if (net->sgen_bus[j] < 0 || net->sgen_bus[j] >= n) return fail(MAPDN_ERR_INVALID, "sgen_bus out of range");
  if (prof) {
    if (!prof->pv || !prof->load_p || !prof->load_q || !prof->pv_std || !prof->load_p_std ||
        !prof->load_q_std || !prof->s_max || prof->n_rows < 2 || prof->steps_per_hour < 1)
      return fail(MAPDN_ERR_INVALID, "incomplete profile description");
  }
  return MAPDN_OK;
}

// The branch and shunt arrays with the optional ones filled in, and the Ybus pieces the device computed from them
struct Ybus {
  std::vector<int> from, to;
  std::vector<unsigned char> st, line;       // in service; counts as a line (line-loss table)
  std::vector<double> gs, bs;                // bus shunts
  std::vector<double> ybr, ydiag;            // [n_branch, 8] Yff Yft Ytf Ytt, [n_bus, 2]
};

// ---- 1. Ybus on the device ----
mapdn_status ybus_on_device(mapdn_env* e, const mapdn_net_desc& net, Ybus& y) {
  const int n = net.n_bus, nbr = net.n_branch;
  std::vector<double> br_r(net.br_r, net.br_r + nbr), br_x(net.br_x, net.br_x + nbr);
  std::vector<double> br_b = vec_or(net.br_b, nbr, 0.0), br_g = vec_or(net.br_g, nbr, 0.0);
  std::vector<double> br_tap = vec_or(net.br_tap, nbr, 1.0), br_sh = vec_or(net.br_shift_deg, nbr, 0.0);
  y.st = vec_or<unsigned char>(net.br_status, nbr, 1);
  y.line = vec_or<unsigned char>(net.br_is_line, nbr, 1);
  y.gs = vec_or(net.bus_gs_mw, n, 0.0); y.bs = vec_or(net.bus_bs_mvar, n, 0.0);
  y.from.assign(net.br_from, net.br_from + nbr);
  y.to.assign(net.br_to, net.br_to + nbr);
  for (int k = 0; k < nbr; ++k)
    if (y.st[k] && br_r[k] == 0.0 && br_x[k] == 0.0) return fail(MAPDN_ERR_INVALID, "zero-impedance branch");
  const double *d_r, *d_x, *d_b, *d_g, *d_tap, *d_sh, *d_gs, *d_bs;
  const unsigned char* d_st;
  const int *d_f, *d_t;
  double *d_ybr, *d_ydiag;
  MAPDN_TRY(dev_upload(e, br_r, &d_r)); MAPDN_TRY(dev_upload(e, br_x, &d_x)); MAPDN_TRY(dev_upload(e, br_b, &d_b));
  MAPDN_TRY(dev_upload(e, br_g, &d_g)); MAPDN_TRY(dev_upload(e, br_tap, &d_tap)); MAPDN_TRY(dev_upload(e, br_sh, &d_sh));
  MAPDN_TRY(dev_upload(e, y.st, &d_st)); MAPDN_TRY(dev_upload(e, y.from, &d_f)); MAPDN_TRY(dev_upload(e, y.to, &d_t));
  MAPDN_TRY(dev_upload(e, y.gs, &d_gs)); MAPDN_TRY(dev_upload(e, y.bs, &d_bs));
  MAPDN_TRY(dev_alloc(e, static_cast<size_t>(8) * nbr, &d_ybr)); MAPDN_TRY(dev_alloc(e, static_cast<size_t>(2) * n, &d_ydiag));
  MAPDN_LAUNCH(ybus_branch_kernel, (nbr + 127) / 128, 128, 0, 0, nbr, d_r, d_x, d_b, d_g, d_tap, d_sh, d_st, d_ybr);
  MAPDN_LAUNCH(ybus_diag_kernel, (n + 127) / 128, 128, 0, 0, n, nbr, d_f, d_t, d_ybr, d_gs, d_bs, 1.0 / net.base_mva, d_ydiag);
  MAPDN_CUDA(cudaGetLastError());
  e->launches += 2;
  y.ybr.resize(static_cast<size_t>(8) * nbr);
  y.ydiag.resize(static_cast<size_t>(2) * n);
  MAPDN_CUDA(cudaMemcpy(y.ybr.data(), d_ybr, y.ybr.size() * sizeof(double), cudaMemcpyDeviceToHost));
  MAPDN_CUDA(cudaMemcpy(y.ydiag.data(), d_ydiag, y.ydiag.size() * sizeof(double), cudaMemcpyDeviceToHost));
  e->br_from = y.from; e->br_to = y.to; e->ybr = y.ybr; e->ydiag = y.ydiag;      // kept for the test hook
  return MAPDN_OK;
}

struct Pair { double gab = 0, bab = 0, gba = 0, bba = 0; };   // Y[a,b], Y[b,a] with a < b
using Pairs = std::map<std::pair<int, int>, Pair>;            // the in-service branches, parallel ones merged

// Ybus[a,b] of two different buses; zero when no branch joins them
void yoff(const Pairs& pairs, int a, int b, double& g, double& bb) {
  const auto it = pairs.find({std::min(a, b), std::max(a, b)});
  if (it == pairs.end()) { g = bb = 0.0; return; }
  const Pair& pr = it->second;
  if (a < b) { g = pr.gab; bb = pr.bab; } else { g = pr.gba; bb = pr.bba; }
}

// The forest of PQ buses. Nodes are numbered breadth first (roots, then level by level) until relabel_nodes permutes them:
// it rewrites order, node_of_bus, parent, nchild, kid0 and kid1; cfirst, height, eorder, elev and dlev describe the
// breadth-first numbering, which the sweep schedules are planned on.
struct Forest {
  int n = 0, npq = 0, slack = 0;
  Pairs pairs;
  std::vector<std::vector<int>> adj;         // by bus, sorted
  bool meshed = false;
  std::vector<int> order, node_of_bus, parent_bus;    // node -> bus; bus -> node (slack -> npq); bus -> parent bus (-1: root)
  std::vector<int> parent, nchild, cfirst, height;    // by node; the children of i are cfirst[i] .. cfirst[i] + nchild[i] - 1
  std::vector<int> kid0, kid1;               // first and second child (npq = none); further children follow kid1 contiguously
  std::vector<int> eorder;                   // nodes by height
  std::vector<uint16_t> elev, dlev;          // [n_lev + 1] level starts: in eorder by height, in node ids by depth
  int n_lev = 0, max_children = 0;
};

// ---- 2. symbolic analysis: merge parallel branches, check the net is radial, build the forest
//         of PQ buses (slack removed) and re-root every tree at its centre ----
mapdn_status build_forest(const Ybus& y, int n, int slack, Forest& f) {
  const int npq = n - 1;
  f.n = n; f.npq = npq; f.slack = slack;
  Pairs& pairs = f.pairs;
  for (size_t k = 0; k < y.from.size(); ++k) {
    if (!y.st[k]) continue;
    const int fr = y.from[k], t = y.to[k];
    const double* yk = &y.ybr[8 * k];
    Pair& pr = pairs[{std::min(fr, t), std::max(fr, t)}];
    if (fr < t) { pr.gab += yk[2]; pr.bab += yk[3]; pr.gba += yk[4]; pr.bba += yk[5]; }   // Ybus[f,t]+=Yft, [t,f]+=Ytf
    else        { pr.gba += yk[2]; pr.bba += yk[3]; pr.gab += yk[4]; pr.bab += yk[5]; }
  }
  std::vector<std::vector<int>>& adj = f.adj;
  adj.resize(n);
  for (auto& kv : pairs) { adj[kv.first.first].push_back(kv.first.second); adj[kv.first.second].push_back(kv.first.first); }
  for (auto& a : adj) std::sort(a.begin(), a.end());
  {   // connectivity + radiality on the full graph
    std::vector<char> seen(n, 0);
    std::vector<int> q{slack};
    seen[slack] = 1;
    for (size_t qh = 0; qh < q.size(); ++qh)
      for (int v : adj[q[qh]]) if (!seen[v]) { seen[v] = 1; q.push_back(v); }
    if (static_cast<int>(q.size()) != n)
      return fail(MAPDN_ERR_TOPOLOGY, "network is not connected to the slack bus (" +
                                          std::to_string(n - q.size()) + " unreachable buses)");
  }
  // A radial net (|edges| = n - 1) takes the zero-fill tree solver; a meshed one the dense-LU fallback.
  const bool meshed = f.meshed = static_cast<int>(pairs.size()) != n - 1;
  if (meshed && n - 1 > 256)
    return fail(MAPDN_ERR_TOPOLOGY, "network is meshed (" + std::to_string(pairs.size() - (n - 1)) +
                                        " loop-closing branches) and has more than 256 PQ buses: the dense "
                                        "fallback solver only covers small meshed feeders");
  // BFS inside the PQ forest (never crossing the slack bus)
  auto bfs = [&](int src, std::vector<int>& dist, std::vector<int>& from) {
    std::vector<int> q{src};
    dist[src] = 0; from[src] = -1;
    for (size_t qh = 0; qh < q.size(); ++qh)
      for (int v : adj[q[qh]]) if (v != slack && dist[v] < 0) { dist[v] = dist[q[qh]] + 1; from[v] = q[qh]; q.push_back(v); }
    return q;
  };
  std::vector<int> roots;
  {
    std::vector<int> d0(n, -1), f0(n, -1);
    for (int s0 : adj[slack]) {                        // one tree per slack neighbour
      if (d0[s0] >= 0) continue;
      std::vector<int> comp = bfs(s0, d0, f0);
      int u = comp.back();                             // farthest from s0
      std::vector<int> d1(n, -1), f1(n, -1);
      std::vector<int> c1 = bfs(u, d1, f1);
      int v = c1.back();                               // farthest from u: u..v is a diameter
      int c = v;
      for (int k = 0; k < d1[v] / 2; ++k) c = f1[c];   // walk half-way back: the centre
      roots.push_back(c);
    }
  }
  std::vector<int>&order = f.order, &node_of_bus = f.node_of_bus, &parent_bus = f.parent_bus;
  std::vector<int> depth(n, 0);
  node_of_bus.assign(n, -1); parent_bus.assign(n, -1);
  order.reserve(npq);
  for (int r : roots) { node_of_bus[r] = static_cast<int>(order.size()); order.push_back(r); }
  for (size_t qh = 0; qh < order.size(); ++qh) {
    const int u = order[qh];
    for (int v : adj[u]) {
      if (v == slack || node_of_bus[v] >= 0) continue;
      node_of_bus[v] = static_cast<int>(order.size());
      parent_bus[v] = u;
      depth[v] = depth[u] + 1;
      order.push_back(v);
    }
  }
  node_of_bus[slack] = npq;
  std::vector<int>&parent = f.parent, &nchild = f.nchild, &height = f.height, &cfirst = f.cfirst;
  parent.assign(npq, -1); nchild.assign(npq, 0); height.assign(npq, 0);
  for (int i = 0; i < npq; ++i)
    if (parent_bus[order[i]] >= 0) { parent[i] = node_of_bus[parent_bus[order[i]]]; nchild[parent[i]]++; }
  if (meshed) {   // no elimination forest: every bus is its own root, the sweeps are not used
    std::fill(parent.begin(), parent.end(), -1);
    std::fill(nchild.begin(), nchild.end(), 0);
    for (int b = 0; b < n; ++b) depth[b] = 0;
  }
  for (int i = npq - 1; i >= 0; --i)
    if (parent[i] >= 0) height[parent[i]] = std::max(height[parent[i]], height[i] + 1);
  cfirst.resize(npq + 1);
  cfirst[0] = static_cast<int>(roots.size());
  for (int i = 0; i < npq; ++i) cfirst[i + 1] = cfirst[i] + nchild[i];
  int max_h = 0;
  for (int i = 0; i < npq; ++i) max_h = std::max(max_h, height[i]);
  const int n_lev = f.n_lev = max_h + 1;                // = max depth + 1
  f.elev.resize(n_lev + 1); f.dlev.resize(n_lev + 1);
  for (int hgt = 0; hgt <= max_h; ++hgt) {
    f.elev[hgt] = static_cast<uint16_t>(f.eorder.size());
    for (int i = 0; i < npq; ++i) if (height[i] == hgt) f.eorder.push_back(i);
  }
  f.elev[n_lev] = static_cast<uint16_t>(f.eorder.size());
  {
    int d = 0;
    f.dlev[0] = 0;
    for (int i = 0; i < npq; ++i) while (depth[order[i]] > d) f.dlev[++d] = static_cast<uint16_t>(i);
    while (d < n_lev) f.dlev[++d] = static_cast<uint16_t>(npq);
  }
  f.kid0.assign(npq, npq); f.kid1.assign(npq, npq);
  for (int i = 0; i < npq; ++i) {
    f.max_children = std::max(f.max_children, nchild[i]);
    if (nchild[i] > 0) f.kid0[i] = cfirst[i];
    if (nchild[i] > 1) f.kid1[i] = cfirst[i] + 1;
  }
  return MAPDN_OK;
}

// Idle lanes of a sweep step work on the trash record npq + 1 and reach for the zero slot npq
uint64_t esched_idle(int npq) {
  return static_cast<uint64_t>(npq + 1) | (static_cast<uint64_t>(npq) << 16) | (static_cast<uint64_t>(npq) << 32) |
         (static_cast<uint64_t>(kEschedReg0 | kEschedIdle) << 48);
}
uint64_t bsched_idle(int npq) {
  return static_cast<uint64_t>(npq + 1) | (static_cast<uint64_t>(npq) << 16) |
         (static_cast<uint64_t>(kBschedRegParent | kBschedIdle) << 32);
}

struct Sweeps {
  int G = 0;                                 // lanes per env
  std::vector<uint64_t> esched, bsched;      // [steps * G] forward elimination / back substitution, see kernel_params.h
  int n_wide_e = 0, n_narrow_b = 0;          // G > 32: forward steps [n_wide_e, end) and back steps [0, n_narrow_b) use warp 0 only
  int n_esteps() const { return static_cast<int>(esched.size()) / G; }
  int n_bsteps() const { return static_cast<int>(bsched.size()) / G; }
};

// ---- 2a. lanes per env and the two sweep schedules ----
mapdn_status plan_sweeps(const Forest& f, int lanes_per_env, Sweeps& s) {
  const int npq = f.npq, n_lev = f.n_lev;
  const std::vector<int>&nchild = f.nchild, &cfirst = f.cfirst, &height = f.height, &parent = f.parent;
  int G = lanes_per_env;
  if (G == 0) G = (npq <= 64) ? 8 : (npq <= 256 ? 32 : 64);      // fastest on H100 at every BASELINE size (DESIGN.md §4)
  if (f.meshed) G = 32;                  // the dense fallback works one warp per env
  s.G = G;
  // Flat schedules for this G: a level wider than G takes several steps; idle lanes get the trash record.
  // Lanes follow chains: a bus is placed on the lane that handled its child (forward sweep) / its parent
  // (back sweep) in the immediately preceding step whenever that lane is free, so the dependent value can
  // stay in registers.
  const uint64_t trash = npq + 1;
  std::vector<uint64_t>&esched = s.esched, &bsched = s.bsched;
  std::vector<int> lane_of(npq, -1), step_of(npq, -1), reg_child(npq, -1), epos(npq, -1);
  int cur = 0;
  // Multi-warp groups (G > 32): the levels near the roots hold a handful of buses. From the first level on after which no
  // level is wider than a warp ("narrow suffix" of the forward sweep / "narrow prefix" of the back sweep) only warp 0 of
  // the group works: those steps are packed into lanes 0..31 and synchronise with __syncwarp instead of a named barrier.
  int first_narrow_lev = n_lev;
  if (G > 32) { while (first_narrow_lev > 0 && f.elev[first_narrow_lev] - f.elev[first_narrow_lev - 1] <= 32) --first_narrow_lev; }
  s.n_wide_e = -1;
  for (int l = 0; l < n_lev; ++l) {
    const int w = f.elev[l + 1] - f.elev[l], nst = (w + G - 1) / G;
    const bool narrow = G > 32 && l >= first_narrow_lev;
    if (narrow && s.n_wide_e < 0) s.n_wide_e = cur;
    std::vector<int> slot(static_cast<size_t>(nst) * G, -1), inh(npq, -1);
    std::vector<int> rest;
    for (int k = f.elev[l]; k < f.elev[l + 1]; ++k) {
      const int i = f.eorder[k];
      int pick = -1;
      if (nchild[i] >= 1 && nchild[i] <= 2)
        for (int c = cfirst[i]; c < cfirst[i] + nchild[i]; ++c)
          if (step_of[c] == cur - 1 && slot[lane_of[c]] < 0 && (!narrow || lane_of[c] < 32) &&
              (pick < 0 || height[c] > height[pick])) pick = c;
      if (pick >= 0) { slot[lane_of[pick]] = i; inh[i] = pick; }
      else rest.push_back(i);
    }
    size_t pos = 0;
    for (int i : rest) { while (slot[pos] >= 0) ++pos; slot[pos] = i; }
    for (int sidx = 0; sidx < nst * G; ++sidx) {
      const int i = slot[sidx];
      if (i < 0) { esched.push_back(esched_idle(npq)); continue; }
      lane_of[i] = sidx % G; step_of[i] = cur + sidx / G;
      uint64_t c0 = npq, c1 = npq, fl = kEschedLeaf;       // no child: zero update, nothing to fetch
      if (nchild[i] > 2) {
        c0 = cfirst[i]; c1 = cfirst[i] + 1; fl = static_cast<uint64_t>(std::min(nchild[i] - 2, 255)) | kEschedLoad0 | kEschedLoad1;
        if (nchild[i] - 2 > 255) return fail(MAPDN_ERR_UNSUPPORTED, "a bus with more than 257 children");
      } else if (nchild[i] >= 1) {
        const int a0 = inh[i] >= 0 ? inh[i] : cfirst[i];
        c0 = a0; fl = (inh[i] >= 0 && sidx / G == 0) ? kEschedReg0 : kEschedLoad0;
        if (fl & kEschedReg0) reg_child[i] = a0;
        if (nchild[i] == 2) { c1 = (a0 == cfirst[i]) ? cfirst[i] + 1 : cfirst[i]; fl |= kEschedLoad1; }
      }
      epos[i] = static_cast<int>(esched.size());
      esched.push_back(static_cast<uint64_t>(i) | (c0 << 16) | (c1 << 32) | (fl << 48));
    }
    cur += nst;
  }
  // a bus stores its Schur update only if its parent will fetch it from shared memory
  for (int i = 0; i < npq; ++i)
    if (parent[i] >= 0 && reg_child[parent[i]] != i) esched[epos[i]] |= static_cast<uint64_t>(kEschedStore) << 48;
  if (s.n_wide_e < 0) s.n_wide_e = cur;           // no narrow suffix
  // back sweep by depth: children inherit the lane of their parent (the child with the tallest subtree first)
  std::fill(lane_of.begin(), lane_of.end(), -1); std::fill(step_of.begin(), step_of.end(), -1);
  cur = 0;
  const int first_back_level = 1;      // the roots' dx = D^-1 r is already in place
  int last_narrow_dlev = first_back_level - 1;  // depth levels first_back_level .. last_narrow_dlev are narrow (prefix)
  if (G > 32) { while (last_narrow_dlev + 1 < n_lev && f.dlev[last_narrow_dlev + 2] - f.dlev[last_narrow_dlev + 1] <= 32) ++last_narrow_dlev; }
  s.n_narrow_b = 0;
  for (int l = first_back_level; l < n_lev; ++l) {
    const int w = f.dlev[l + 1] - f.dlev[l], nst = (w + G - 1) / G;
    if (G > 32 && l <= last_narrow_dlev) s.n_narrow_b = cur + nst;
    std::vector<int> slot(static_cast<size_t>(nst) * G, -1);
    std::vector<char> reg(npq, 0);
    std::vector<int> nodes;
    for (int i = f.dlev[l]; i < f.dlev[l + 1]; ++i) nodes.push_back(i);
    std::stable_sort(nodes.begin(), nodes.end(), [&](int a, int b) { return height[a] > height[b]; });
    std::vector<int> rest;
    for (int i : nodes) {
      const int pa = parent[i];
      if (pa >= 0 && step_of[pa] == cur - 1 && lane_of[pa] >= 0 && slot[lane_of[pa]] < 0) { slot[lane_of[pa]] = i; reg[i] = 1; }
      else rest.push_back(i);
    }
    size_t pos = 0;
    for (int i : rest) { while (slot[pos] >= 0) ++pos; slot[pos] = i; }
    for (int sidx = 0; sidx < nst * G; ++sidx) {
      const int i = slot[sidx];
      if (i < 0) { bsched.push_back(bsched_idle(npq)); continue; }
      lane_of[i] = sidx % G; step_of[i] = cur + sidx / G;
      bsched.push_back(static_cast<uint64_t>(i) | (static_cast<uint64_t>(parent[i] >= 0 ? parent[i] : npq) << 16) |
                       (static_cast<uint64_t>((reg[i] && sidx / G == 0) ? kBschedRegParent : 0u) << 32));
    }
    cur += nst;
  }
  if (getenv("MAPDN_DEBUG_SCHED")) {
    int nreg = 0, nl0 = 0, nl1 = 0, nreal = 0;
    for (uint64_t e2 : esched) { if ((e2 & 0xFFFF) == trash) continue; ++nreal; unsigned fl = e2 >> 48; nreg += !!(fl & kEschedReg0); nl0 += !!(fl & kEschedLoad0); nl1 += !!(fl & kEschedLoad1); }
    int breg = 0, breal = 0;
    for (uint64_t b2 : bsched) { if ((b2 & 0xFFFF) == trash) continue; ++breal; breg += (b2 >> 32) & 1; }
    fprintf(stderr, "[sched] G=%d levels=%d esteps=%zu real=%d reg0=%d load0=%d load1=%d | bsteps=%zu real=%d regp=%d\n", G, n_lev,
            esched.size() / G, nreal, nreg, nl0, nl1, bsched.size() / G, breal, breg);
  }
  if (bsched.empty()) bsched.assign(G, bsched_idle(npq));      // a forest of single buses: one all-idle step
  return MAPDN_OK;
}

// ---- 2b. bank-conflict-aware relabelling of the node records ----
// A node record is 144 B = 9 x 16 B, so the 16-byte bank group of field f of node i is (i + f) mod 8: the eight lanes of a
// quarter-warp (one 128-bit access wavefront) are conflict free iff their node ids differ mod 8. The passes own nodes
// by id (conflict free by construction) but reach parents / children by pointer, and the sweeps touch whatever the
// schedules say; ncu counted 25 % of the shared-load wavefronts as conflicts with the breadth-first ids. The ids are
// free to choose, so pick a permutation that minimises the weighted number of extra wavefronts over every access group
// of the kernel (simulated annealing on pairwise swaps, deterministic; identity when it does not apply).
// Permutes the forest and both schedules together, or leaves them as they are.
void relabel_nodes(const Ybus& y, Forest& f, Sweeps& s) {
  const int n = f.n, npq = f.npq, G = s.G;
  std::vector<int>&order = f.order, &node_of_bus = f.node_of_bus, &parent = f.parent, &nchild = f.nchild, &kid0 = f.kid0, &kid1 = f.kid1;
  std::vector<uint64_t>&esched = s.esched, &bsched = s.bsched;
  if (f.meshed || f.max_children > 2 || G < 8 || npq < 8 || getenv("MAPDN_NO_RELABEL")) return;
  struct Grp { std::vector<int> nodes; double w; };
  std::vector<Grp> groups;                                  // groups whose members do not depend on the labelling
  const double w_iter = 4.5;                                // Newton iterations per step (sweeps and passes run that often)
  auto add_quarters = [&](const std::vector<int>& per_lane, double w) {      // per_lane: node per lane of the group (-1: no access)
    for (int q = 0; q < G / 8; ++q) {
      Grp g; g.w = w;
      for (int l = 8 * q; l < 8 * q + 8; ++l) if (per_lane[l] >= 0) g.nodes.push_back(per_lane[l]);
      std::sort(g.nodes.begin(), g.nodes.end());
      g.nodes.erase(std::unique(g.nodes.begin(), g.nodes.end()), g.nodes.end());      // same address = broadcast
      if (g.nodes.size() > 1) groups.push_back(std::move(g));
    }
  };
  std::vector<int> own(G), c0v(G), c1v(G);
  for (size_t st = 0; st < esched.size() / G; ++st) {
    for (int l = 0; l < G; ++l) {
      const uint64_t ed = esched[st * G + l];
      const unsigned fl = static_cast<unsigned>(ed >> 48);
      own[l] = static_cast<int>(ed & 0xFFFFu);
      c0v[l] = (fl & kEschedLoad0) ? static_cast<int>((ed >> 16) & 0xFFFFu) : -1;
      c1v[l] = (fl & kEschedLoad1) ? static_cast<int>((ed >> 32) & 0xFFFFu) : -1;
    }
    add_quarters(own, 2.0 * w_iter);                        // own blocks: loaded (prefetch) and stored
    add_quarters(c0v, w_iter); add_quarters(c1v, w_iter);
  }
  for (size_t st = 0; st < bsched.size() / G; ++st) {
    for (int l = 0; l < G; ++l) {
      const uint64_t bd = bsched[st * G + l];
      const unsigned bfl = static_cast<unsigned>(bd >> 32);
      own[l] = static_cast<int>(bd & 0xFFFFu);
      c0v[l] = (bfl & (kBschedRegParent | kBschedIdle)) ? -1 : static_cast<int>((bd >> 16) & 0xFFFFu);
    }
    add_quarters(own, 2.0 * w_iter); add_quarters(c0v, w_iter);
  }
  for (int b0 = 0; b0 < n; b0 += G) {                       // epilogue: per-bus loop, buses b0 + lane
    for (int l = 0; l < G; ++l) own[l] = (b0 + l < n) ? node_of_bus[b0 + l] : -1;
    add_quarters(own, 1.0);
  }
  {
    std::vector<int> lf, lt;
    for (size_t k = 0; k < y.from.size(); ++k) if (y.line[k]) { lf.push_back(node_of_bus[y.from[k]]); lt.push_back(node_of_bus[y.to[k]]); }
    for (size_t k0 = 0; k0 < lf.size(); k0 += G) {
      for (int l = 0; l < G; ++l) { own[l] = (k0 + l < lf.size()) ? lf[k0 + l] : -1; c0v[l] = (k0 + l < lt.size()) ? lt[k0 + l] : -1; }
      add_quarters(own, 1.0); add_quarters(c0v, 1.0);
    }
  }
  // lab[base id] = label; sentinel / trash keep their ids
  std::vector<int> lab(npq + 2), inv(npq + 2);
  for (int i = 0; i < npq + 2; ++i) lab[i] = inv[i] = i;
  auto extra = [&](const int* ids, int cnt) {               // extra wavefronts of one access: max multiplicity - 1
    int c[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int mx = 0;
    for (int k = 0; k < cnt; ++k) mx = std::max(mx, ++c[ids[k] & 7]);
    return std::max(0, mx - 1);
  };
  auto cost = [&]() {
    double tot = 0.0;
    int ids[8];
    for (const Grp& g : groups) {
      int cnt = 0;
      for (int v : g.nodes) ids[cnt++] = lab[v];
      tot += g.w * extra(ids, cnt);
    }
    // passes: label L is handled by lane L % G in round L / G; neighbours reached by pointer
    for (int L0 = 0; L0 < npq; L0 += 8) {
      int pa[8], k0[8], k1[8], np = 0, n0 = 0, n1 = 0;
      auto push_unique = [](int* a, int& cnt, int v) { for (int k = 0; k < cnt; ++k) if (a[k] == v) return; a[cnt++] = v; };
      for (int L = L0; L < std::min(npq, L0 + 8); ++L) {
        const int i = inv[L];
        push_unique(pa, np, parent[i] >= 0 ? lab[parent[i]] : npq);
        push_unique(k0, n0, lab[kid0[i]]); push_unique(k1, n1, lab[kid1[i]]);
      }
      tot += w_iter * (extra(pa, np) + extra(k0, n0) + extra(k1, n1));
    }
    return tot;
  };
  const double cost0 = cost();
  double cur = cost0, best = cur;
  std::vector<int> best_lab = lab;
  uint64_t rng = 0x9E3779B97F4A7C15ull;
  auto rnd = [&]() { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return rng; };
  const int iters = std::min(400 * npq, 30000);
  double T = std::max(1.0, 0.02 * cur);
  const double cool = std::pow(1e-3, 1.0 / std::max(1, iters));
  for (int it = 0; it < iters && best > 0.0; ++it, T *= cool) {
    const int a = static_cast<int>(rnd() % npq), b = static_cast<int>(rnd() % npq);
    if (a == b || ((lab[a] ^ lab[b]) & 7) == 0) continue;  // same residue: no effect on any group
    std::swap(lab[a], lab[b]); inv[lab[a]] = a; inv[lab[b]] = b;
    const double c2 = cost();
    const double u = static_cast<double>(rnd() >> 11) * (1.0 / 9007199254740992.0);
    if (c2 <= cur || u < std::exp((cur - c2) / T)) {
      cur = c2;
      if (cur < best) { best = cur; best_lab = lab; }
    } else {
      std::swap(lab[a], lab[b]); inv[lab[a]] = a; inv[lab[b]] = b;
    }
  }
  lab = best_lab;
  if (best < cost0) {
    // apply: new id of base node i is lab[i]
    std::vector<int> order2(npq), parent2(npq), nchild2(npq), k0b(npq), k1b(npq);
    for (int i = 0; i < npq; ++i) {
      const int L = lab[i];
      order2[L] = order[i];
      parent2[L] = parent[i] >= 0 ? lab[parent[i]] : -1;
      nchild2[L] = nchild[i];
      k0b[L] = lab[kid0[i]]; k1b[L] = lab[kid1[i]];
    }
    order = order2; parent = parent2; nchild = nchild2; kid0 = k0b; kid1 = k1b;
    for (int i = 0; i < npq; ++i) node_of_bus[order[i]] = i;
    auto map16 = [&](uint64_t v) { return static_cast<uint64_t>(lab[static_cast<int>(v & 0xFFFFu)]); };
    for (uint64_t& ed : esched)
      ed = (ed & 0xFFFF000000000000ull) | map16(ed) | (map16(ed >> 16) << 16) | (map16(ed >> 32) << 32);
    for (uint64_t& bd : bsched)
      bd = (bd & 0xFFFFFFFF00000000ull) | map16(bd) | (map16(bd >> 16) << 16);
  }
  if (getenv("MAPDN_DEBUG_SCHED"))
    fprintf(stderr, "[relabel] weighted extra shared-memory wavefronts per env-step: %.1f -> %.1f (%d swaps tried)\n",
            cost0, best, iters);
}

struct ElementMaps { std::vector<uint16_t> lptr, lidx, sptr, sidx, xptr, xidx; };   // node -> loads / sgens / sgens of the node's zone (CSR)

// ---- 3. element -> node maps (needed by the hot blob) ----
ElementMaps element_maps(const mapdn_net_desc& net, const Forest& f) {
  const int npq = f.npq, nl = net.n_load, ng = net.n_sgen;
  ElementMaps m;
  m.lptr.assign(npq + 2, 0); m.lidx.resize(std::max(1, nl)); m.sptr.assign(npq + 2, 0); m.sidx.resize(ng); m.xptr.assign(npq + 2, 0);
  std::vector<std::vector<int>> ln(npq + 1), sn(npq + 1);
  for (int l = 0; l < nl; ++l) ln[f.node_of_bus[net.load_bus[l]]].push_back(l);
  for (int j = 0; j < ng; ++j) sn[f.node_of_bus[net.sgen_bus[j]]].push_back(j);
  int a = 0, b = 0;
  for (int i = 0; i <= npq; ++i) {
    m.lptr[i] = static_cast<uint16_t>(a); m.sptr[i] = static_cast<uint16_t>(b);
    m.xptr[i] = static_cast<uint16_t>(m.xidx.size());
    for (int l : ln[i]) m.lidx[a++] = static_cast<uint16_t>(l);
    const int bus = (i == npq) ? f.slack : f.order[i];
    for (int j : sn[i]) {
      m.sidx[b++] = static_cast<uint16_t>(j);
      if (net.sgen_zone[j] == net.bus_zone[bus]) m.xidx.push_back(static_cast<uint16_t>(j));   // reference :238-244
    }
  }
  m.lptr[npq + 1] = static_cast<uint16_t>(a); m.sptr[npq + 1] = static_cast<uint16_t>(b);
  m.xptr[npq + 1] = static_cast<uint16_t>(m.xidx.size());
  return m;
}

// Slab offset (in doubles) of the sentinel record's UP.x: constant zero. The obs padding reads it.
int zero_slot(int npq) { return 2 * (npq * kNodeArrays2 + A_UP); }

struct ObsPrograms {
  int obs_dim = 0, pvq_off2 = 0, scratch_off2 = 0;
  std::vector<uint16_t> obs_off, obs_compact;          // hot copies: padded rows, rows without the padding
  std::vector<unsigned> obs_src, state_src;            // cold copies: kind | node, kind | bus or sgen
  std::vector<int> obs_xptr, obs_xidx;                 // sgens to add back per obs entry (CSR)
  std::vector<int> agent_len, agent_off;               // compact rows: true length / offset of every agent's block
};

// obs program (reference get_obs :232-274): per agent [P_zone | Q_zone | pv | q | vm_zone | va_zone | 0...].
// Hot copy: double offset of the source inside the env slab. Cold copy (get_obs_kernel): kind | node.
mapdn_status obs_programs(const mapdn_net_desc& net, const Forest& f, int G, int state_space_mask, ObsPrograms& o) {
  const int n = f.n, npq = f.npq, nl = net.n_load, ng = net.n_sgen;
  const std::vector<int>& node_of_bus = f.node_of_bus;
  const int ssm = (state_space_mask & 31) ? (state_space_mask & 31) : 31;
  const bool ss_dem = ssm & 1, ss_pv = ssm & 2, ss_q = ssm & 4, ss_vm = ssm & 8, ss_va = ssm & 16;
  int obs_dim = 0;
  std::vector<std::vector<int>> zb(ng);
  for (int a = 0; a < ng; ++a) {
    for (int b = 0; b < n; ++b) if (net.bus_zone[b] == net.sgen_zone[a]) zb[a].push_back(b);
    const int nz = static_cast<int>(zb[a].size());
    obs_dim = std::max(obs_dim, nz * (2 * ss_dem + ss_vm + ss_va) + ss_pv + ss_q);
  }
  const int pvq_off2 = kNodeArrays2 * (npq + 2), scratch_off2 = pvq_off2 + ng;      // + sentinel + trash records
  if (2 * (scratch_off2 + (scratch_doubles_for(ng, nl, G, false) + 1) / 2) >= 65535)
    return fail(MAPDN_ERR_UNSUPPORTED, "network too large for 16-bit slab offsets");
  o.obs_dim = obs_dim; o.pvq_off2 = pvq_off2; o.scratch_off2 = scratch_off2;
  o.obs_off.resize(static_cast<size_t>(ng) * obs_dim);
  o.obs_src.assign(static_cast<size_t>(ng) * obs_dim, 0u);
  o.obs_xptr.assign(static_cast<size_t>(ng) * obs_dim + 1, 0);
  o.agent_len.assign(ng, 0);
  auto src = [](ObsKind kind, int ix) { return (static_cast<unsigned>(kind) << 28) | static_cast<unsigned>(ix); };
  for (int a = 0; a < ng; ++a) {
    // entry list of this agent in the reference's order (:254-266), then zero padding (:270-274)
    std::vector<std::pair<ObsKind, int>> ent;            // (kind, bus or sgen)
    if (ss_dem) { for (int b : zb[a]) ent.push_back({OBS_P, b}); for (int b : zb[a]) ent.push_back({OBS_Q, b}); }
    if (ss_pv) ent.push_back({OBS_PV, a});
    if (ss_q) ent.push_back({OBS_QSG, a});
    if (ss_vm) for (int b : zb[a]) ent.push_back({OBS_VM, b});
    if (ss_va) for (int b : zb[a]) ent.push_back({OBS_VA, b});
    o.agent_len[a] = static_cast<int>(ent.size());
    for (int k = 0; k < obs_dim; ++k) {
      const size_t idx = static_cast<size_t>(a) * obs_dim + k;
      o.obs_xptr[idx] = static_cast<int>(o.obs_xidx.size());
      ObsKind kind = OBS_ZERO;
      int ix = 0, off = zero_slot(npq);
      if (k < static_cast<int>(ent.size())) {
        kind = ent[k].first;
        const int t2 = ent[k].second;
        if (kind == OBS_P || kind == OBS_Q) {
          ix = node_of_bus[t2];
          off = 2 * (node_of_bus[t2] * kNodeArrays2 + A_OP) + (kind == OBS_P ? 0 : 1);
          for (int j = 0; j < ng; ++j)
            if (net.sgen_zone[j] == net.sgen_zone[a] && net.sgen_bus[j] == t2) o.obs_xidx.push_back(j);
        } else if (kind == OBS_PV) { ix = t2; off = 2 * pvq_off2 + t2; }
        else if (kind == OBS_QSG) { ix = t2; off = 2 * pvq_off2 + ng + t2; }
        else { ix = node_of_bus[t2]; off = 2 * (node_of_bus[t2] * kNodeArrays2 + A_VV) + (kind == OBS_VM ? 0 : 1); }
      }
      o.obs_src[idx] = src(kind, ix);
      o.obs_off[idx] = static_cast<uint16_t>(off);
    }
  }
  o.obs_xptr[static_cast<size_t>(ng) * obs_dim] = static_cast<int>(o.obs_xidx.size());
  // the same program without the padding: agent blocks back to back, the row rounded up to 4 entries (16-byte pieces of
  // fp32 rows) with reads of the zero slot
  o.agent_off.assign(ng, 0);
  for (int a = 0; a < ng; ++a) {
    o.agent_off[a] = static_cast<int>(o.obs_compact.size());
    for (int k = 0; k < o.agent_len[a]; ++k) o.obs_compact.push_back(o.obs_off[static_cast<size_t>(a) * obs_dim + k]);
  }
  while (o.obs_compact.size() % 4) o.obs_compact.push_back(static_cast<uint16_t>(zero_slot(npq)));
  // state program (reference get_state :213-230), bus-indexed
  std::vector<unsigned>& state_src = o.state_src;
  if (ss_dem) { for (int b = 0; b < n; ++b) state_src.push_back(src(OBS_PBUS, b)); for (int b = 0; b < n; ++b) state_src.push_back(src(OBS_QBUS, b)); }
  if (ss_pv) for (int j = 0; j < ng; ++j) state_src.push_back(src(OBS_PV, j));
  if (ss_q) for (int j = 0; j < ng; ++j) state_src.push_back(src(OBS_QSG, j));
  if (ss_vm) for (int b = 0; b < n; ++b) state_src.push_back(src(OBS_VM, b));
  if (ss_va) for (int b = 0; b < n; ++b) state_src.push_back(src(OBS_VA_DEG, b));
  return MAPDN_OK;
}

struct BranchTables {
  int n_line = 0;
  std::vector<uint16_t> line_nodes;          // [2 * n_line] from / to node; never empty, see below
  std::vector<double> line_c;                // [4 * n_line] loss coefficients
  std::vector<uint16_t> nbr_ptr, nbr_idx;    // meshed nets: CSR of the PQ-PQ Ybus pattern
  std::vector<double> nbr_y;
};

// ---- 3a. line-loss table, and the PQ-PQ Ybus pattern (CSR) for the dense fallback ----
BranchTables branch_tables(const Ybus& y, const Forest& f, double base_mva) {
  BranchTables t;
  for (size_t k = 0; k < y.from.size(); ++k) {
    if (!y.line[k]) continue;
    const double* yk = &y.ybr[8 * k];
    t.line_nodes.push_back(static_cast<uint16_t>(f.node_of_bus[y.from[k]]));
    t.line_nodes.push_back(static_cast<uint16_t>(f.node_of_bus[y.to[k]]));
    // pl = Re(Sf + St) = Gff|Vf|^2 + Gtt|Vt|^2 + (Gft+Gtf) Re(Vf Vt*) + (Bft-Btf) Im(Vf Vt*)   [x baseMVA]
    t.line_c.push_back(yk[0] * base_mva); t.line_c.push_back(yk[6] * base_mva);
    t.line_c.push_back((yk[2] + yk[4]) * base_mva); t.line_c.push_back((yk[3] - yk[5]) * base_mva);
  }
  t.n_line = static_cast<int>(t.line_nodes.size() / 2);
  // a net without lines keeps one all-zero entry in the hot blob and in the cold copies: n_line stays 0
  if (t.line_nodes.empty()) { t.line_nodes.assign(2, 0); t.line_c.assign(4, 0.0); }
  t.nbr_ptr.assign(1, 0);
  if (f.meshed) {
    t.nbr_ptr.assign(f.npq + 1, 0);
    for (int i = 0; i < f.npq; ++i) {
      const int b = f.order[i];
      for (int v : f.adj[b]) {
        if (v == f.slack) continue;
        double g, bb;
        yoff(f.pairs, b, v, g, bb);
        t.nbr_idx.push_back(static_cast<uint16_t>(f.node_of_bus[v])); t.nbr_y.push_back(g); t.nbr_y.push_back(bb);
      }
      t.nbr_ptr[i + 1] = static_cast<uint16_t>(t.nbr_idx.size());
    }
  }
  return t;
}

struct HotBlob {
  HotLayout hl{};                            // offsets only: bytes / tables_in_blob follow from the launch geometry
  std::vector<unsigned char> blob;           // bytes_full bytes
  int bytes_core = 0, bytes_full = 0;        // without / with the once-per-step tables
  std::vector<double> ysl_cold;              // Y[i,slack]: cold table, non-zero for a few buses
  std::vector<int> sl_node;                  // the slack-adjacent nodes and their Y[slack,i]
  std::vector<double> sl_y;
};

// Appends a table to the blob at the next 16-byte boundary and returns its byte offset. The slot holds at least min_count
// entries (zeros beyond the table's own): the kernel addresses some tables that can be empty.
template <class T>
int blob_put(std::vector<unsigned char>& blob, const std::vector<T>& v, size_t min_count = 0) {
  const size_t off = blob.size();
  blob.resize(off + (std::max(v.size(), min_count) * sizeof(T) + 15) / 16 * 16, 0);
  if (!v.empty()) std::memcpy(blob.data() + off, v.data(), v.size() * sizeof(T));
  return static_cast<int>(off);
}

// ---- 3b. hot static blob ----
HotBlob build_hot_blob(const Ybus& y, const Forest& f, const Sweeps& s, const ElementMaps& m, const ObsPrograms& o,
                       const BranchTables& t) {
  const int npq = f.npq, slack = f.slack;
  HotBlob h;
  std::vector<double> yup(2 * static_cast<size_t>(npq), 0.0), ydn(2 * static_cast<size_t>(npq + 1), 0.0), yii(2 * static_cast<size_t>(npq));
  std::vector<uint64_t> ndesc(npq);
  h.ysl_cold.assign(2 * static_cast<size_t>(npq), 0.0);
  double* ysl = h.ysl_cold.data();
  for (int i = 0; i < npq; ++i) {
    const int b = f.order[i];
    yii[2 * i] = y.ydiag[2 * b]; yii[2 * i + 1] = y.ydiag[2 * b + 1];
    if (f.parent[i] >= 0) {
      yoff(f.pairs, b, f.parent_bus[b], yup[2 * i], yup[2 * i + 1]);       // Y[i,parent]
      yoff(f.pairs, f.parent_bus[b], b, ydn[2 * i], ydn[2 * i + 1]);       // Y[parent,i]
    }
    const uint64_t sl_adj = f.pairs.count({std::min(b, slack), std::max(b, slack)}) ? 1 : 0;
    if (sl_adj) {
      yoff(f.pairs, b, slack, ysl[2 * i], ysl[2 * i + 1]);               // Y[i,slack]
      double g, bb;
      yoff(f.pairs, slack, b, g, bb);                                    // Y[slack,i]
      h.sl_node.push_back(i); h.sl_y.push_back(g); h.sl_y.push_back(bb);
    }
    // parent | child0 | child1 | number of further children (contiguous after child1); npq = zero slot
    const uint64_t pa = f.parent[i] >= 0 ? static_cast<uint64_t>(f.parent[i]) : npq;   // roots: sentinel, Y = 0
    const uint64_t c0 = static_cast<uint64_t>(f.kid0[i]), c1 = static_cast<uint64_t>(f.kid1[i]);   // npq = none
    const uint64_t nx = f.nchild[i] > 2 ? f.nchild[i] - 2 : 0;
    ndesc[i] = pa | (c0 << 16) | (c1 << 32) | (nx << 48) | (sl_adj << 63);
  }
  const std::vector<uint16_t> nob(f.node_of_bus.begin(), f.node_of_bus.end());
  HotLayout& hl = h.hl;
  hl.yup = blob_put(h.blob, yup); hl.ydn = blob_put(h.blob, ydn); hl.yii = blob_put(h.blob, yii);
  hl.ndesc = blob_put(h.blob, ndesc); hl.esched = blob_put(h.blob, s.esched); hl.bsched = blob_put(h.blob, s.bsched);
  hl.lptr = blob_put(h.blob, m.lptr); hl.lidx = blob_put(h.blob, m.lidx);
  hl.sptr = blob_put(h.blob, m.sptr); hl.sidx = blob_put(h.blob, m.sidx);
  hl.xptr = blob_put(h.blob, m.xptr); hl.xidx = blob_put(h.blob, m.xidx, 1);
  hl.node_of_bus = blob_put(h.blob, nob);
  hl.nbr_ptr = blob_put(h.blob, t.nbr_ptr); hl.nbr_idx = blob_put(h.blob, t.nbr_idx, 1); hl.nbr_y = blob_put(h.blob, t.nbr_y, 2);
  h.bytes_core = static_cast<int>(h.blob.size());
  // the once-per-step tables go last: the TMA copy either includes them (hl.bytes = bytes_full) or stops before them
  hl.ysl = blob_put(h.blob, h.ysl_cold); hl.obs_off = blob_put(h.blob, o.obs_off);
  hl.line_nodes = blob_put(h.blob, t.line_nodes); hl.line_c = blob_put(h.blob, t.line_c);
  h.bytes_full = static_cast<int>(h.blob.size());
  return h;
}

struct Geometry {
  bool cold_tables = false, stage_rec = false;   // the two ways to buy shared memory, see below
  int stride2 = 0, epb = 0, smem = 0, helper_threads = 32;
  int smem_needed = 0;                           // set on a refusal: the bytes of the smallest plan (one group of envs)
};

// ---- 5. launch geometry ----
// envs per CTA: sub-warp groups pack 32/G envs into each of 1..4 solver warps; multi-warp groups (G = 64 / 128)
// put 1..4 envs of G threads in a CTA. Fewer envs per CTA when that spreads the batch over all SMs.
mapdn_status plan_geometry(int npq, int ng, int nl, int G, int batch, int bytes_core, int bytes_full, size_t max_smem,
                           int n_sm, Geometry& geo) {
  const int unit = (G <= 32) ? 32 / G : 1;               // envs added per step of the search
  // Two ways to buy shared memory when it limits the envs per SM, both with a price: (a) the four
  // once-per-step tables (Y[i,slack], obs program, line tables) stay in global memory instead of the staged blob - their
  // first touch after an L2 flush is an HBM round trip at the start of the epilogue, softened by an L2 prefetch at kernel
  // start; (b) the prologue stages the scaled loads inside the node records - index arithmetic in every step of
  // case33. Each is used only if it lets the batch finish in fewer rounds (case322 x 1024: 4 envs per SM and 2 rounds
  // instead of 3 and 3).
  struct Plan { bool cold, rec, ok; int st2, epb; long long rounds; };
  auto smem_with = [&](bool cold, int st2, int c) {
    return static_cast<size_t>(cold ? bytes_core : bytes_full) + static_cast<size_t>(c) * (st2 * 16 + 16);   // + helper scalars
  };
  auto make_plan = [&](bool cold, bool rec) {
    Plan pl{cold, rec, false, 0, 0, 0};
    if (rec && !stage_fits_records(npq, nl)) return pl;
    pl.st2 = env_stride2_for(npq, ng, nl, G, rec);
    // two solver warps per CTA for small sub-warp groups, four for one-warp envs,
    // as many multi-warp envs as fit (<= 512 solver threads)
    int c_epb = (G <= 16) ? 2 * unit : 4 * unit;
    if (G > 32) while (c_epb > 1 && c_epb * G > 512) --c_epb;
    // Few-round batches (the BASELINE.json configs): one CTA per SM holding ceil(B / (SMs * rounds)) envs balances the
    // SMs exactly (case33 x 4096 on 132 SMs: 128 CTAs of 32 envs). Many-round batches keep several small CTAs per SM.
    auto fits = [&](int c) { return smem_with(cold, pl.st2, c) <= max_smem && c * G <= (G <= 32 ? 256 : 512); };
    for (int r = 1; r <= 3; ++r) {
      int c = (batch + n_sm * r - 1) / (n_sm * r);
      c = (c + unit - 1) / unit * unit;
      if (fits(c)) { c_epb = std::max(c_epb, c); break; }
    }
    if (const char* ov = getenv("MAPDN_EPB")) c_epb = std::max(unit, atoi(ov) / unit * unit);   // tuning override
    // the override obeys the search's caps too: 256 / 512 solver threads (launch bounds, named-barrier ids 3 + gidx <= 15)
    while (c_epb > unit && (smem_with(cold, pl.st2, c_epb) > max_smem || c_epb * G > (G <= 32 ? 256 : 512))) c_epb -= unit;
    pl.epb = c_epb;
    pl.ok = smem_with(cold, pl.st2, c_epb) <= max_smem;
    pl.rounds = (batch + static_cast<long long>(c_epb) * n_sm - 1) / (static_cast<long long>(c_epb) * n_sm);
    return pl;
  };
  const Plan plans[4] = {make_plan(false, false), make_plan(false, true), make_plan(true, false), make_plan(true, true)};   // cheapest first
  const Plan* best = nullptr;
  for (const Plan& pl : plans) if (pl.ok && (!best || pl.rounds < best->rounds)) best = &pl;
  if (const char* ov = getenv("MAPDN_PLAN")) {             // tuning override: 0..3 = index into the list above
    const int k = atoi(ov);
    if (k >= 0 && k < 4 && plans[k].ok) best = &plans[k];
  }
  if (!best) {       // every plan that could be built needs more than max_smem with a single group of envs
    size_t need = SIZE_MAX;
    for (const Plan& pl : plans) if (pl.st2 > 0) need = std::min(need, smem_with(pl.cold, pl.st2, unit));
    geo.smem_needed = static_cast<int>(need);
    return fail(MAPDN_ERR_UNSUPPORTED, "network too large for the shared-memory resident solver (" + std::to_string(need) +
                                           " B needed at " + std::to_string(G) + " lanes per env, " +
                                           std::to_string(max_smem) + " B available)");
  }
  geo.stride2 = best->st2; geo.epb = best->epb; geo.stage_rec = best->rec; geo.cold_tables = best->cold;
  geo.smem = static_cast<int>(smem_with(geo.cold_tables, geo.stride2, geo.epb));
  // helper warps (next profile rows + noise, concurrent with the Newton iteration): one per 256 Box-Muller pairs of a
  // CTA round, at most 4 -- a single warp can be the critical path of case322
  const int n_pair = (ng + 2 * nl + 1) / 2;
  geo.helper_threads = 32 * std::min(4, std::max(1, (geo.epb * n_pair + kHelperPairsPerWarp - 1) / kHelperPairsPerWarp));
  if (const char* ov = getenv("MAPDN_HELPERS")) geo.helper_threads = 32 * std::min(4, std::max(1, atoi(ov)));   // tuning override
  return MAPDN_OK;
}

// Everything sections 2a to 5 plan for one lane count. relabel_nodes permutes the forest, so each plan owns a copy.
struct LanePlan {
  Forest f;
  Sweeps s;
  ObsPrograms o;
  BranchTables t;
  HotBlob hot;
  Geometry geo;
};

mapdn_status plan_for_lanes(const Ybus& y, const Forest& forest, const mapdn_net_desc& net, const mapdn_cfg& cfg, int lanes,
                            const cudaDeviceProp& dp, LanePlan& p) {
  p.f = forest;
  MAPDN_TRY(plan_sweeps(p.f, lanes, p.s));
  relabel_nodes(y, p.f, p.s);
  const ElementMaps m = element_maps(net, p.f);
  MAPDN_TRY(obs_programs(net, p.f, p.s.G, cfg.state_space_mask, p.o));
  p.t = branch_tables(y, p.f, net.base_mva);
  p.hot = build_hot_blob(y, p.f, p.s, m, p.o, p.t);
  return plan_geometry(net.n_bus - 1, net.n_sgen, net.n_load, p.s.G, cfg.batch, p.hot.bytes_core, p.hot.bytes_full,
                       dp.sharedMemPerBlockOptin, dp.multiProcessorCount, p.geo);
}

// The lane count of the handle. An explicit lanes_per_env is planned as asked. With lanes_per_env = 0 the default of
// plan_sweeps comes first; the schedules grow as depth x lanes, so a deep feeder (a 400-bus chain at 64 lanes) can miss
// shared memory at the default and fit at fewer lanes. Then the other lane counts are tried in a fixed order - one warp
// per env, narrower groups, multi-warp groups last - and the first that fits is taken. The dense fallback of a meshed
// net always works one warp per env.
mapdn_status plan_lanes(const Ybus& y, const Forest& forest, const mapdn_net_desc& net, const mapdn_cfg& cfg,
                        const cudaDeviceProp& dp, LanePlan& p) {
  const mapdn_status st = plan_for_lanes(y, forest, net, cfg, cfg.lanes_per_env, dp, p);
  if (st != MAPDN_ERR_UNSUPPORTED || p.geo.smem_needed == 0 || cfg.lanes_per_env != 0 || forest.meshed) return st;
  int need = p.geo.smem_needed, need_lanes = p.s.G;
  for (const int lanes : {32, 16, 8, 4, 64, 128}) {
    if (lanes == p.s.G) continue;
    LanePlan q;
    const mapdn_status sq = plan_for_lanes(y, forest, net, cfg, lanes, dp, q);
    if (sq == MAPDN_OK) { p = std::move(q); return MAPDN_OK; }
    if (sq != MAPDN_ERR_UNSUPPORTED || q.geo.smem_needed == 0) return sq;
    if (q.geo.smem_needed < need) { need = q.geo.smem_needed; need_lanes = lanes; }
  }
  return fail(MAPDN_ERR_UNSUPPORTED, "network too large for the shared-memory resident solver at every lane count (" +
                                         std::to_string(need) + " B needed at " + std::to_string(need_lanes) + " lanes per env, " +
                                         std::to_string(dp.sharedMemPerBlockOptin) + " B available)");
}

// The flat start of the first Newton iteration: every PQ bus at vm_init, angle 0; the slack at vm0, va0 = e0 + j f0
struct FlatStart { double vm_init, vm0, va0, e0, f0; };

FlatStart flat_start(const mapdn_net_desc& net) {
  FlatStart v{};
  v.vm_init = (net.vm_init > 0) ? net.vm_init : net.slack_vm;
  v.vm0 = net.slack_vm; v.va0 = net.slack_va_deg * (3.14159265358979323846 / 180.0);
  v.e0 = v.vm0 * std::cos(v.va0); v.f0 = v.vm0 * std::sin(v.va0);
  return v;
}

// The first Newton iteration starts from the flat start, where S_calc and the Jacobian depend on the network only:
// factorise J(V0) once, leaf -> root on the elimination forest, with the formulas of the kernel's edge / mismatch pass
// and elimination step (env_kernel.cuh: nr_solve). Per node six double2: S_calc = (P, Q); M = D'^-1 J[i,parent] rows
// 0 / 1 (what the back sweep multiplies dx_parent with); D'^-1 rows 0 / 1; J[parent,i] = (a, b).
std::vector<double> first_iteration_factors(const Forest& f, const HotBlob& hot, const FlatStart& v0) {
  const int npq = f.npq;
  std::vector<double> ft(static_cast<size_t>(12) * std::max(1, npq), 0.0);
  if (f.meshed) return ft;
  const double* yup = reinterpret_cast<const double*>(hot.blob.data() + hot.hl.yup);
  const double* ydn = reinterpret_cast<const double*>(hot.blob.data() + hot.hl.ydn);
  const double* yii = reinterpret_cast<const double*>(hot.blob.data() + hot.hl.yii);
  const std::vector<double>& ysl_cold = hot.ysl_cold;
  // children in a labelling-independent order (first child, second child, then the contiguous extras): the node
  // relabelling of section 2b must not change a single bit of the results
  std::vector<std::vector<int>> kids(npq);
  for (int i = 0; i < npq; ++i) {
    if (f.kid0[i] != npq) kids[i].push_back(f.kid0[i]);
    if (f.kid1[i] != npq) kids[i].push_back(f.kid1[i]);
    for (int c = 2; c < f.nchild[i]; ++c) kids[i].push_back(f.kid1[i] + c - 1);      // extras follow child 1 contiguously
  }
  std::vector<int> topo;                               // parents before children
  for (int i = 0; i < npq; ++i) if (f.parent[i] < 0) topo.push_back(i);
  for (size_t qh = 0; qh < topo.size(); ++qh) for (int c : kids[topo[qh]]) topo.push_back(c);
  const double vi_x = v0.vm_init, vi_y = 0.0;            // every PQ bus
  std::vector<double> upx(npq), upy(npq), dnx(npq), dny(npq), d01x(npq), d01y(npq), d23x(npq), d23y(npq);
  std::vector<double> s00(npq, 0.0), s01(npq, 0.0), s10(npq, 0.0), s11(npq, 0.0);     // Schur update a bus hands to its parent
  for (int i = 0; i < npq; ++i) {                      // edge terms of (i, parent); roots: Y = 0
    const double vp_x = v0.vm_init, vp_y = 0.0;
    const double cc = vi_x * vp_x + vi_y * vp_y, ss = vi_y * vp_x - vi_x * vp_y;
    upx[i] = yup[2 * i] * ss - yup[2 * i + 1] * cc; upy[i] = yup[2 * i] * cc + yup[2 * i + 1] * ss;
    dnx[i] = -ydn[2 * i] * ss - ydn[2 * i + 1] * cc; dny[i] = ydn[2 * i] * cc - ydn[2 * i + 1] * ss;
  }
  for (int i = 0; i < npq; ++i) {                      // S_calc and the diagonal blocks
    const double cs0 = vi_x * v0.e0 + vi_y * v0.f0, sn0 = vi_y * v0.e0 - vi_x * v0.f0;
    double sa = ysl_cold[2 * i] * sn0 - ysl_cold[2 * i + 1] * cs0 + upx[i];
    double sb = ysl_cold[2 * i] * cs0 + ysl_cold[2 * i + 1] * sn0 + upy[i];
    for (int c : kids[i]) { sa += dnx[c]; sb += dny[c]; }
    const double vv = vi_x * vi_x + vi_y * vi_y;
    const double gv = yii[2 * i] * vv, bv = yii[2 * i + 1] * vv;
    const double Pc = gv + sb, Qc = sa - bv;
    ft[12 * i + 0] = Pc; ft[12 * i + 1] = Qc;
    d01x[i] = -Qc - bv; d01y[i] = Pc + gv; d23x[i] = Pc - gv; d23y[i] = Qc - bv;
  }
  for (size_t k = topo.size(); k-- > 0;) {              // children before parents
    const int i = topo[k];
    for (int c : kids[i]) { d01x[i] -= s00[c]; d01y[i] -= s01[c]; d23x[i] -= s10[c]; d23y[i] -= s11[c]; }
    const double idet = 1.0 / (d01x[i] * d23y[i] - d01y[i] * d23x[i]);
    const double ux = upx[i], uy = upy[i], dx = dnx[i], dy = dny[i];
    const double ma00 = d23y[i] * ux + d01y[i] * uy, ma01 = d23y[i] * uy - d01y[i] * ux;      // adj(D') J[i,parent]
    const double ma10 = -d23x[i] * ux - d01x[i] * uy, ma11 = d01x[i] * ux - d23x[i] * uy;
    ft[12 * i + 2] = ma00 * idet; ft[12 * i + 3] = ma01 * idet; ft[12 * i + 4] = ma10 * idet; ft[12 * i + 5] = ma11 * idet;
    ft[12 * i + 6] = d23y[i] * idet; ft[12 * i + 7] = -d01y[i] * idet;                         // D'^-1
    ft[12 * i + 8] = -d23x[i] * idet; ft[12 * i + 9] = d01x[i] * idet;
    ft[12 * i + 10] = dx; ft[12 * i + 11] = dy;
    s00[i] = (dx * ma00 + dy * ma10) * idet; s01[i] = (dx * ma01 + dy * ma11) * idet;         // J[parent,i] D'^-1 J[i,parent]
    s10[i] = (dx * ma10 - dy * ma00) * idet; s11[i] = (dx * ma11 - dy * ma01) * idet;
  }
  return ft;
}

// The shared-memory attribute of the nine kernel instantiations the handle launches, and the persistent grid of the six
// step variants (needs G, threads, helper_threads, smem and dense of the handle)
mapdn_status size_kernels(mapdn_env* e, const cudaDeviceProp& dp) {
  struct Variant { int mode; bool record, hist, autoreset; };
  const Variant variants[9] = {{MODE_STEP, false, false, false}, {MODE_STEP, true, false, false}, {MODE_STEP, false, true, false},
                               {MODE_STEP, true, true, false}, {MODE_STEP, false, false, true}, {MODE_STEP, false, true, true},
                               {MODE_SOLVE, false, false, false}, {MODE_RESET, false, false, false}, {MODE_DROOP, false, false, false}};
  for (const Variant& v : variants) {       // the plain step first: it bounds the grids of the other five
    KernelFn fn = kernel_for(e->G, v.mode, e->dense, v.record, v.hist, v.autoreset);
    // the attribute belongs to the function, not to the handle: always allow the device maximum, so that creating a
    // second handle with a smaller footprint cannot break the launches of the first
    cudaFuncAttributes fa{};
    MAPDN_CUDA(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(fn)));
    const int dyn_max = static_cast<int>(dp.sharedMemPerBlockOptin - fa.sharedSizeBytes);        // opt-in limit minus the static part
    if (e->smem > dyn_max) return fail(MAPDN_ERR_UNSUPPORTED, "network too large for the shared-memory resident solver");
    MAPDN_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_max));
    if (v.mode != MODE_STEP) continue;
    int per_sm = 0;
    MAPDN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, e->threads + e->helper_threads, e->smem));
    int blocks = std::max(1, per_sm) * dp.multiProcessorCount;
    if (e->dense) blocks = std::min(blocks, 2 * dp.multiProcessorCount);   // bounds the dense workspace
    // the record, history and auto-reset instantiations hold more registers: each persistent grid is sized by its own
    // occupancy (never larger than the plain step's)
    if (v.record || v.hist || v.autoreset) blocks = std::min(blocks, e->max_blocks_step[0][0][0]);
    e->max_blocks_step[v.autoreset][v.hist][v.record] = blocks;
  }
  return MAPDN_OK;
}

// ---- 6. upload + env state ----
// Fills e->base from the plan, uploads every table and allocates the env state. Needs the handle's launch geometry and
// the grid of the plain step (size_kernels): a meshed net's dense workspace has one slice per resident env group.
mapdn_status upload_plan(mapdn_env* e, const mapdn_net_desc& net, const mapdn_profile_desc* prof, const Ybus& y,
                         const Forest& f, const Sweeps& s, const ObsPrograms& o, const BranchTables& t, const HotBlob& hot,
                         const Geometry& geo, const FlatStart& v0, const std::vector<double>& ft) {
  const mapdn_cfg& cfg = e->cfg;
  const int n = f.n, npq = f.npq, nl = net.n_load, ng = net.n_sgen, slack = f.slack;
  Params& P = e->base;
  P.n_bus = n; P.npq = npq; P.n_load = nl; P.n_sgen = ng; P.n_line = t.n_line; P.n_lev = f.n_lev;
  P.obs_dim = o.obs_dim; P.state_dim = static_cast<int>(o.state_src.size()); P.n_slack_adj = static_cast<int>(hot.sl_node.size());
  P.n_esteps = s.n_esteps(); P.n_bsteps = s.n_bsteps(); P.has_extra_children = f.max_children > 2;
  P.n_wide_e = std::min(s.n_wide_e, P.n_esteps); P.n_narrow_b = std::min(s.n_narrow_b, P.n_bsteps);
  P.slack_bus = slack;
  P.nb = cfg.batch; P.env_stride2 = geo.stride2; P.pvq_off2 = o.pvq_off2; P.scratch_off2 = o.scratch_off2;
  P.hot_layout = hot.hl;
  P.hot_layout.tables_in_blob = geo.cold_tables ? 0 : 1;
  P.hot_layout.bytes = geo.cold_tables ? hot.bytes_core : hot.bytes_full;
  P.helper_off = P.hot_layout.bytes + e->epb * geo.stride2 * 16;
  P.stage_in_records = geo.stage_rec ? 1 : 0;
  P.obs_skip_off = -1;
  P.history = 1;
  e->obs_zero_off = zero_slot(npq);
  MAPDN_TRY(dev_upload(e, o.obs_compact, &P.obs_compact_prog));
  P.obs_compact_len = 0;
  e->agent_len = o.agent_len; e->agent_off = o.agent_off; e->compact_row = static_cast<int>(o.obs_compact.size());
  {   // bus shunts by node (res_bus p/q carry the shunt power, pandapower _get_shunt_results)
    std::vector<double> sh_g(npq + 1), sh_b(npq + 1);
    bool any = false;
    for (int i = 0; i <= npq; ++i) {
      const int b = (i == npq) ? slack : f.order[i];
      sh_g[i] = y.gs[b]; sh_b[i] = y.bs[b];
      any = any || y.gs[b] != 0.0 || y.bs[b] != 0.0;
    }
    P.has_shunt = any;
    MAPDN_TRY(dev_upload(e, sh_g, &P.sh_g)); MAPDN_TRY(dev_upload(e, sh_b, &P.sh_b));
  }
  MAPDN_TRY(dev_upload(e, hot.blob, &P.hot));
  MAPDN_TRY(dev_upload(e, f.order, &P.bus_of_node));
  MAPDN_TRY(dev_upload(e, vec_or(net.load_scaling, nl, 1.0), &P.lscale));
  MAPDN_TRY(dev_upload(e, vec_or(net.sgen_scaling, ng, 1.0), &P.sscale));
  MAPDN_TRY(dev_upload(e, hot.sl_node, &P.sl_node)); MAPDN_TRY(dev_upload(e, hot.sl_y, &P.sl_y));
  {
    const double *d_ysl = nullptr, *d_ft = nullptr;
    MAPDN_TRY(dev_upload(e, hot.ysl_cold, &d_ysl));
    P.ysl = reinterpret_cast<const double2*>(d_ysl);
    MAPDN_TRY(dev_upload(e, ft, &d_ft));
    P.first_tab = reinterpret_cast<const double2*>(d_ft);
  }
  MAPDN_TRY(dev_upload(e, o.obs_off, &P.obs_off));
  MAPDN_TRY(dev_upload(e, t.line_nodes, &P.line_nodes)); MAPDN_TRY(dev_upload(e, t.line_c, &P.line_c));
  {
    std::vector<int> sgen_node(ng);
    for (int j = 0; j < ng; ++j) sgen_node[j] = f.node_of_bus[net.sgen_bus[j]];
    MAPDN_TRY(dev_upload(e, sgen_node, &P.sgen_node));
  }
  MAPDN_TRY(dev_upload(e, o.state_src, &P.state_src)); MAPDN_TRY(dev_upload(e, o.obs_src, &P.obs_src));
  MAPDN_TRY(dev_upload(e, o.obs_xptr, &P.obs_xptr)); MAPDN_TRY(dev_upload(e, o.obs_xidx, &P.obs_xidx));
  const size_t B = static_cast<size_t>(cfg.batch);
  if (prof) {
    const size_t T = static_cast<size_t>(prof->n_rows);
    MAPDN_TRY(dev_upload(e, std::vector<double>(prof->s_max, prof->s_max + ng), &P.s_max));
    MAPDN_TRY(dev_upload(e, std::vector<double>(prof->pv_std, prof->pv_std + ng), &P.pv_std));
    MAPDN_TRY(dev_upload(e, std::vector<double>(prof->load_p_std, prof->load_p_std + nl), &P.lp_std));
    MAPDN_TRY(dev_upload(e, std::vector<double>(prof->load_q_std, prof->load_q_std + nl), &P.lq_std));
    double *dpv, *dlp, *dlq;
    MAPDN_TRY(dev_alloc(e, T * ng, &dpv)); MAPDN_TRY(dev_alloc(e, T * nl, &dlp)); MAPDN_TRY(dev_alloc(e, T * nl, &dlq));
    MAPDN_CUDA(cudaMemcpy(dpv, prof->pv, T * ng * sizeof(double), cudaMemcpyHostToDevice));
    if (nl) {
      MAPDN_CUDA(cudaMemcpy(dlp, prof->load_p, T * nl * sizeof(double), cudaMemcpyHostToDevice));
      MAPDN_CUDA(cudaMemcpy(dlq, prof->load_q, T * nl * sizeof(double), cudaMemcpyHostToDevice));
    }
    P.prof_pv = dpv; P.prof_lp = dlp; P.prof_lq = dlq;
    P.n_rows = prof->n_rows; P.steps_per_hour = prof->steps_per_hour;
    const int episode_days = cfg.episode_limit / (24 * prof->steps_per_hour) + 1;     // reference :397
    P.n_day_choices = prof->n_days - episode_days;                                    // reference :398
    if (P.n_day_choices < 1) return fail(MAPDN_ERR_INVALID, "profile store shorter than one episode");
    // the latest sampled window must fit: start_max + episode_limit rows
    const long long last = (static_cast<long long>(P.n_day_choices - 1) * 24 + 23) * prof->steps_per_hour +
                           (prof->steps_per_hour - 1) + cfg.episode_limit;
    if (last > prof->n_rows - 1) return fail(MAPDN_ERR_INVALID, "profile store shorter than n_days claims");
  }
  P.base_mva = net.base_mva; P.inv_base = 1.0 / net.base_mva;
  P.vm_init = v0.vm_init; P.vm0 = v0.vm0; P.va0 = v0.va0; P.e0 = v0.e0; P.f0 = v0.f0;
  P.ysl_g0 = y.ydiag[2 * slack]; P.ysl_b0 = y.ydiag[2 * slack + 1];
  P.tol = (cfg.tol > 0) ? cfg.tol : 1e-8;
  P.max_iter = (cfg.max_iter > 0) ? cfg.max_iter : 10;
  P.barrier = cfg.barrier; P.voltage_weight = cfg.voltage_weight; P.q_weight = cfg.q_weight;
  P.line_weight = cfg.line_weight; P.use_line_weight = cfg.use_line_weight;
  P.v_upper = cfg.v_upper; P.v_lower = cfg.v_lower; P.episode_limit = cfg.episode_limit;
  P.action_low = cfg.action_low; P.action_high = cfg.action_high; P.reset_action = cfg.reset_action;
  P.seed = cfg.seed; P.env_id_offset = cfg.env_id_offset;
  MAPDN_TRY(dev_alloc(e, B * nl, &P.cur_pl)); MAPDN_TRY(dev_alloc(e, B * nl, &P.cur_ql));
  MAPDN_TRY(dev_alloc(e, B * ng, &P.cur_pv)); MAPDN_TRY(dev_alloc(e, B * ng, &P.cur_q));
  MAPDN_TRY(dev_alloc(e, B * n, &P.res_vm)); MAPDN_TRY(dev_alloc(e, B * n, &P.res_va));
  MAPDN_TRY(dev_alloc(e, B * n, &P.res_p)); MAPDN_TRY(dev_alloc(e, B * n, &P.res_q));
  MAPDN_TRY(dev_alloc(e, B * std::max(1, t.n_line), &P.res_pl));
  MAPDN_TRY(dev_alloc(e, B, &P.steps)); MAPDN_TRY(dev_alloc(e, B, &P.sum_rewards));
  MAPDN_TRY(dev_alloc(e, B, &P.start_row)); MAPDN_TRY(dev_alloc(e, B, &P.episode)); MAPDN_TRY(dev_alloc(e, B, &P.nr_iters));
  if (f.meshed) {
    const size_t m = 2 * static_cast<size_t>(npq);
    P.dense_stride = static_cast<int>(m * (m + 1));
    const size_t groups = static_cast<size_t>(e->max_blocks_step[0][0][0]) * e->epb;       // one slice per resident env group
    MAPDN_TRY(dev_alloc(e, groups * P.dense_stride, &P.dense_ws));
  }
  // staging for the *_host entry points
  MAPDN_TRY(dev_alloc(e, B * ng, &e->d_stage_actions)); MAPDN_TRY(dev_alloc(e, B, &e->d_stage_reward)); MAPDN_TRY(dev_alloc(e, B, &e->d_stage_term));
  MAPDN_TRY(dev_alloc(e, B * MAPDN_N_INFO, &e->d_stage_info));
  MAPDN_TRY(dev_alloc(e, B * std::max<size_t>(ng * o.obs_dim, e->compact_row), &e->d_stage_obs));   // compact rows round up to 4 entries

  mapdn_dims& d = e->dims;
  d.batch = cfg.batch; d.n_bus = n; d.n_branch = net.n_branch; d.n_line = t.n_line; d.n_load = nl; d.n_sgen = ng;
  d.n_agents = ng; d.n_actions = 1; d.obs_dim = o.obs_dim; d.state_dim = P.state_dim; d.n_info = MAPDN_N_INFO;
  d.lanes_per_env = e->G; d.envs_per_block = e->epb; d.smem_bytes = e->smem; d.n_levels = f.n_lev;
  // SURVEY §8d: read p_load,q_load,p_pv,a ; write vm,va ; write obs ; reward+done+11 info
  d.algorithmic_bytes_per_env_step = 8LL * (2 * nl + 2 * ng) + 8LL * 2 * n + 8LL * ng * o.obs_dim + 8LL * 13;
  return MAPDN_OK;
}

}  // namespace

extern "C" {

int32_t mapdn_abi_version(void) { return MAPDN_ABI_VERSION; }
const char* mapdn_last_error(void) { return g_last_error.c_str(); }

mapdn_status mapdn_destroy(mapdn_env* e) {
  if (!e) return MAPDN_OK;
  DeviceGuard guard(e->device);
  for (void* d : e->allocs) cudaFree(d);
  delete e;
  return MAPDN_OK;
}

mapdn_status mapdn_create(const mapdn_net_desc* net, const mapdn_profile_desc* prof, const mapdn_cfg* cfg,
                          int32_t device, mapdn_env** out) {
  if (!net || !cfg || !out) return fail(MAPDN_ERR_INVALID, "null argument");
  *out = nullptr;
  MAPDN_TRY(validate_create_args(net, prof, cfg));
  MAPDN_ON_DEVICE(device);
  // owns the half-built handle: every refusal below frees it and its device memory
  std::unique_ptr<mapdn_env, decltype(&mapdn_destroy)> e(new (std::nothrow) mapdn_env(), &mapdn_destroy);
  if (!e) return fail(MAPDN_ERR_NOMEM, "out of host memory");
  e->device = device;
  e->cfg = *cfg;
  const int n = net->n_bus;

  Ybus y;
  MAPDN_TRY(ybus_on_device(e.get(), *net, y));
  Forest forest;
  MAPDN_TRY(build_forest(y, n, net->slack_bus, forest));
  cudaDeviceProp dp{};
  MAPDN_CUDA(cudaGetDeviceProperties(&dp, device));
  LanePlan p;
  MAPDN_TRY(plan_lanes(y, forest, *net, *cfg, dp, p));
  const FlatStart v0 = flat_start(*net);
  const std::vector<double> ft = first_iteration_factors(p.f, p.hot, v0);

  e->dense = p.f.meshed;
  e->G = p.s.G; e->threads = p.geo.epb * p.s.G; e->epb = p.geo.epb; e->smem = p.geo.smem; e->helper_threads = p.geo.helper_threads;
  MAPDN_TRY(size_kernels(e.get(), dp));
  MAPDN_TRY(upload_plan(e.get(), *net, prof, y, p.f, p.s, p.o, p.t, p.hot, p.geo, v0, ft));
  // the memsets / uploads above ran on the legacy default stream: order them before any launch of the caller's
  // (possibly non-blocking) streams
  MAPDN_CUDA(cudaDeviceSynchronize());
  *out = e.release();
  return MAPDN_OK;
}

mapdn_status mapdn_get_dims(const mapdn_env* e, mapdn_dims* out) {
  if (!e || !out) return fail(MAPDN_ERR_INVALID, "null argument");
  *out = e->dims;
  return MAPDN_OK;
}

int64_t mapdn_launch_count(const mapdn_env* e) { return e ? e->launches : 0; }

mapdn_status mapdn_reset(mapdn_env* e, const int32_t* start_dhi_dev, const uint8_t* mask_dev, int32_t add_noise,
                         double* obs_dev, double* state_dev, uint8_t* converged_dev, void* stream) {
  if (!e) return fail(MAPDN_ERR_INVALID, "null handle");
  if (!e->base.prof_pv) return fail(MAPDN_ERR_INVALID, "handle was created without a profile store");
  MAPDN_ON_DEVICE(e->device);
  Params p = e->base;
  p.start_dhi = start_dhi_dev; p.mask = mask_dev; p.add_noise = add_noise; p.obs = obs_dev; p.state = state_dev;
  p.reset_ok = converged_dev;
  mapdn_status s = launch_env_kernel(e, MODE_RESET, p, static_cast<cudaStream_t>(stream));
  if (s != MAPDN_OK || p.history <= 1) return s;
  // frame 0 of the new episodes into ring slot 0 (the reset kernel itself has no history instantiation)
  return gather(e, reset_frame_kernel, static_cast<long long>(p.nb) * p.n_sgen * p.obs_dim, stream, p);
}

mapdn_status mapdn_set_history(mapdn_env* e, int32_t history) {
  if (!e) return fail(MAPDN_ERR_INVALID, "null handle");
  if (history < 1) return fail(MAPDN_ERR_INVALID, "history must be >= 1");
  MAPDN_ON_DEVICE(e->device);
  Params& P = e->base;
  if (P.hist) {                 // cudaFree waits for the launches still reading the ring
    MAPDN_CUDA(cudaFree(P.hist));
    e->allocs.erase(std::find(e->allocs.begin(), e->allocs.end(), static_cast<void*>(P.hist)));
    P.hist = nullptr;
  }
  P.history = 1;
  if (history == 1) return MAPDN_OK;
  const mapdn_status s = dev_alloc(e, static_cast<size_t>(P.nb) * history * P.n_sgen * P.obs_dim, &P.hist);
  if (s != MAPDN_OK) return s;
  MAPDN_CUDA(cudaDeviceSynchronize());     // the zero fill ran on the legacy default stream: order it before any launch
  P.history = history;
  return MAPDN_OK;
}

mapdn_status mapdn_step(mapdn_env* e, const double* actions_dev, int32_t add_noise, double* reward_dev,
                        uint8_t* terminated_dev, double* info_dev, double* obs_dev, void* stream) {
  if (!e || !actions_dev || !reward_dev || !terminated_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  return step(e, actions_dev, add_noise, reward_dev, terminated_dev, info_dev, obs_dev, false, stream, nothing, nothing);
}

static int record_row_len(const mapdn_env* e) { return 2 * e->dims.n_sgen + 3 * e->dims.n_bus + e->dims.n_line; }

mapdn_status mapdn_record_layout(const mapdn_env* e, int32_t* off, int32_t* row_len) {
  if (!e) return fail(MAPDN_ERR_INVALID, "null handle");
  const int ng = e->dims.n_sgen, n = e->dims.n_bus;
  const int32_t o[MAPDN_N_RECORD] = {0, ng, 2 * ng, 2 * ng + n, 2 * ng + 2 * n, 2 * ng + 3 * n};
  if (off) for (int k = 0; k < MAPDN_N_RECORD; ++k) off[k] = o[k];
  if (row_len) *row_len = record_row_len(e);
  return MAPDN_OK;
}

mapdn_status mapdn_record(mapdn_env* e, double* record_dev, int64_t record_stride, void* stream) {
  if (!e || !record_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  if (record_stride < record_row_len(e)) return fail(MAPDN_ERR_INVALID, "record_stride shorter than a record row");
  Params p = e->base;
  p.record = record_dev; p.record_stride = record_stride;
  return gather(e, record_kernel, static_cast<long long>(p.nb) * record_row_len(e), stream, p);
}

mapdn_status mapdn_step_record(mapdn_env* e, const double* actions_dev, int32_t add_noise, double* reward_dev,
                               uint8_t* terminated_dev, double* info_dev, double* obs_dev, double* record_dev,
                               int64_t record_stride, void* stream) {
  if (!e || !actions_dev || !reward_dev || !terminated_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  auto check_stride = [&](cudaStream_t) {
    if (record_dev && record_stride < record_row_len(e)) return fail(MAPDN_ERR_INVALID, "record_stride shorter than a record row");
    return MAPDN_OK;
  };
  return step(e, actions_dev, add_noise, reward_dev, terminated_dev, info_dev, obs_dev, false, stream, check_stride, nothing,
              -1, 0, record_dev, record_stride);
}

static int stacked_row_len(const mapdn_env* e) { return e->base.history * e->dims.n_sgen * e->dims.obs_dim; }

mapdn_status mapdn_step_stacked(mapdn_env* e, const double* actions_dev, int32_t add_noise, double* reward_dev,
                                uint8_t* terminated_dev, double* info_dev, double* obs_dev, double* obs_stacked_dev,
                                double* record_dev, int64_t record_stride, void* stream) {
  if (!e || !actions_dev || !reward_dev || !terminated_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  if (e->base.history <= 1) return fail(MAPDN_ERR_INVALID, "handle has no observation history (mapdn_set_history)");
  if (record_dev && record_stride < record_row_len(e)) return fail(MAPDN_ERR_INVALID, "record_stride shorter than a record row");
  return step(e, actions_dev, add_noise, reward_dev, terminated_dev, info_dev, obs_dev, false, stream, nothing, nothing,
              -1, 0, record_dev, record_stride, obs_stacked_dev);
}

mapdn_status mapdn_step_autoreset(mapdn_env* e, const double* actions_dev, int32_t add_noise, double* reward_dev,
                                  uint8_t* terminated_dev, double* info_dev, double* obs_dev, double* obs_stacked_dev,
                                  double* reset_obs_dev, double* reset_obs_stacked_dev, uint8_t* reset_ok_dev, void* stream) {
  if (!e || !actions_dev || !reward_dev || !terminated_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  if (e->base.history <= 1 && (obs_stacked_dev || reset_obs_stacked_dev))
    return fail(MAPDN_ERR_INVALID, "handle has no observation history (mapdn_set_history)");
  const AutoReset ar{reset_obs_dev, reset_obs_stacked_dev, reset_ok_dev};
  return step(e, actions_dev, add_noise, reward_dev, terminated_dev, info_dev, obs_dev, false, stream, nothing, nothing,
              -1, 0, nullptr, 0, obs_stacked_dev, &ar);
}

mapdn_status mapdn_get_obs_stacked(mapdn_env* e, double* obs_stacked_dev, void* stream) {
  if (!e || !obs_stacked_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  if (e->base.history <= 1) return fail(MAPDN_ERR_INVALID, "handle has no observation history (mapdn_set_history)");
  Params p = e->base;
  p.obs_stacked = obs_stacked_dev;
  const long long pieces = static_cast<long long>(p.nb) * stacked_row_len(e) / ((p.obs_dim & 1) == 0 ? 2 : 1);
  return gather(e, obs_stacked_kernel, pieces, stream, p);
}

mapdn_status mapdn_snapshot_layout(const mapdn_env* e, int64_t* off) {
  if (!e || !off) return fail(MAPDN_ERR_INVALID, "null argument");
  const SnapLayout sl = snapshot_layout(e);
  for (int s = 0; s <= MAPDN_N_SNAPSHOT; ++s) off[s] = sl.off[s];
  return MAPDN_OK;
}

mapdn_status mapdn_snapshot(mapdn_env* e, const int32_t* idx_dev, int32_t n, void* buf_dev, void* stream) {
  return snapshot_copy(e, idx_dev, n, buf_dev, stream, false);
}

mapdn_status mapdn_restore(mapdn_env* e, const int32_t* idx_dev, int32_t n, const void* buf_dev, void* stream) {
  return snapshot_copy(e, idx_dev, n, buf_dev, stream, true);
}

mapdn_status mapdn_step_host(mapdn_env* e, const double* actions_host, int32_t add_noise, double* reward_host,
                             uint8_t* terminated_host, double* info_host, double* obs_host, void* stream) {
  return step_staged(e, actions_host, add_noise, reward_host, terminated_host, info_host, obs_host, false, stream);
}

mapdn_status mapdn_step_host_pinned(mapdn_env* e, const double* actions_host, int32_t add_noise, double* reward_host,
                                    uint8_t* terminated_host, double* info_host, void* obs_host, int32_t obs_is_f32,
                                    int32_t skip_padding, int32_t sync, void* stream) {
  if (!e || !actions_host || !reward_host || !terminated_host) return fail(MAPDN_ERR_INVALID, "null argument");
  auto pinned = [&](cudaStream_t) { return check_pinned(e, {actions_host, reward_host, terminated_host, info_host, obs_host}); };
  auto finish = [&](cudaStream_t st) {
    if (sync) MAPDN_CUDA(cudaStreamSynchronize(st));
    return MAPDN_OK;
  };
  return step(e, actions_host, add_noise, reward_host, terminated_host, info_host, obs_host, obs_is_f32, stream, pinned, finish,
              skip_padding ? e->obs_zero_off : -1);
}

mapdn_status mapdn_obs_compact_layout(const mapdn_env* e, int32_t* agent_off, int32_t* agent_len, int32_t* row_len) {
  if (!e) return fail(MAPDN_ERR_INVALID, "null handle");
  for (int a = 0; a < e->dims.n_agents; ++a) {
    if (agent_off) agent_off[a] = e->agent_off[a];
    if (agent_len) agent_len[a] = e->agent_len[a];
  }
  if (row_len) *row_len = e->compact_row;
  return MAPDN_OK;
}

mapdn_status mapdn_step_host_compact(mapdn_env* e, const double* actions_host, int32_t add_noise, double* reward_host,
                                     uint8_t* terminated_host, double* info_host, void* obs_host, int32_t obs_is_f32,
                                     int32_t direct, int32_t sync, void* stream) {
  if (!e || !actions_host || !reward_host || !terminated_host || !obs_host) return fail(MAPDN_ERR_INVALID, "null argument");
  // obs_host is checked also when the rows go through the staging buffer: a copy to pageable memory would be synchronous
  auto pinned = [&](cudaStream_t) { return check_pinned(e, {actions_host, reward_host, terminated_host, info_host, obs_host}); };
  auto finish = [&](cudaStream_t st) {
    const size_t bytes = static_cast<size_t>(e->dims.batch) * e->compact_row * (obs_is_f32 ? sizeof(float) : sizeof(double));
    if (!direct) MAPDN_CUDA(cudaMemcpyAsync(obs_host, e->d_stage_obs, bytes, cudaMemcpyDeviceToHost, st));
    if (sync) MAPDN_CUDA(cudaStreamSynchronize(st));
    return MAPDN_OK;
  };
  return step(e, actions_host, add_noise, reward_host, terminated_host, info_host, direct ? obs_host : e->d_stage_obs,
              obs_is_f32, stream, pinned, finish, -1, e->compact_row);
}

mapdn_status mapdn_wait(mapdn_env* e, void* stream) {
  if (!e) return fail(MAPDN_ERR_INVALID, "null handle");
  MAPDN_ON_DEVICE(e->device);
  MAPDN_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  return MAPDN_OK;
}

mapdn_status mapdn_step_f32obs(mapdn_env* e, const double* actions_dev, int32_t add_noise, double* reward_dev,
                               uint8_t* terminated_dev, double* info_dev, float* obs_dev, void* stream) {
  if (!e || !actions_dev || !reward_dev || !terminated_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  return step(e, actions_dev, add_noise, reward_dev, terminated_dev, info_dev, obs_dev, true, stream, nothing, nothing);
}

mapdn_status mapdn_step_host_f32obs(mapdn_env* e, const double* actions_host, int32_t add_noise, double* reward_host,
                                    uint8_t* terminated_host, double* info_host, float* obs_host, void* stream) {
  return step_staged(e, actions_host, add_noise, reward_host, terminated_host, info_host, obs_host, true, stream);
}

mapdn_status mapdn_get_obs(mapdn_env* e, double* obs_dev, void* stream) {
  if (!e || !obs_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  Params p = e->base;
  p.obs = obs_dev;
  return gather(e, get_obs_kernel, static_cast<long long>(p.nb) * p.n_sgen * p.obs_dim, stream, p);
}

mapdn_status mapdn_get_state(mapdn_env* e, double* state_dev, void* stream) {
  if (!e || !state_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  Params p = e->base;
  p.state = state_dev;
  return gather(e, get_state_kernel, static_cast<long long>(p.nb) * p.state_dim, stream, p);
}

mapdn_status mapdn_get_field(mapdn_env* e, int32_t field, double* out_dev, void* stream) {
  if (!e || !out_dev) return fail(MAPDN_ERR_INVALID, "null argument");
  const Params& p = e->base;
  const long long B = p.nb;
  const double* src = nullptr;
  long long cnt = 0;
  double scale = 1.0;
  switch (field) {
    case MAPDN_FIELD_VM: src = p.res_vm; cnt = B * p.n_bus; break;
    case MAPDN_FIELD_VA_DEG: src = p.res_va; cnt = B * p.n_bus; scale = 57.295779513082320876798; break;
    case MAPDN_FIELD_P_BUS: src = p.res_p; cnt = B * p.n_bus; break;
    case MAPDN_FIELD_Q_BUS: src = p.res_q; cnt = B * p.n_bus; break;
    case MAPDN_FIELD_P_SGEN: src = p.cur_pv; cnt = B * p.n_sgen; break;
    case MAPDN_FIELD_Q_SGEN: src = p.cur_q; cnt = B * p.n_sgen; break;
    case MAPDN_FIELD_LINE_LOSS: src = p.res_pl; cnt = B * p.n_line; break;
    case MAPDN_FIELD_P_LOAD: src = p.cur_pl; cnt = B * p.n_load; break;
    case MAPDN_FIELD_Q_LOAD: src = p.cur_ql; cnt = B * p.n_load; break;
    case MAPDN_FIELD_SUM_REWARDS: src = p.sum_rewards; cnt = B; break;
    case MAPDN_FIELD_STEPS: return gather(e, int_to_double_kernel, B, stream, B, p.steps, out_dev);
    case MAPDN_FIELD_NR_ITERS: return gather(e, int_to_double_kernel, B, stream, B, p.nr_iters, out_dev);
    case MAPDN_FIELD_START_ROW: return gather(e, i64_to_double_kernel, B, stream, B, p.start_row, out_dev);
    default: return fail(MAPDN_ERR_INVALID, "unknown field");
  }
  return gather(e, scale_copy_kernel, cnt, stream, cnt, src, scale, out_dev);
}

mapdn_status mapdn_solve(mapdn_env* e, int32_t nb, const double* p_load, const double* q_load, const double* p_sgen,
                         const double* q_sgen, double* vm, double* va_deg, double* p_bus, double* q_bus, double* pl,
                         int32_t* iters, uint8_t* converged, void* stream) {
  if (!e || nb < 1 || !p_sgen || !q_sgen || (e->dims.n_load > 0 && (!p_load || !q_load)))
    return fail(MAPDN_ERR_INVALID, "null argument");
  MAPDN_ON_DEVICE(e->device);
  Params p = e->base;
  p.nb = nb;
  p.in_pl = p_load; p.in_ql = q_load; p.in_pv = p_sgen; p.in_q = q_sgen;
  p.out_vm = vm; p.out_va = va_deg; p.out_p = p_bus; p.out_q = q_bus; p.out_pl = pl;
  p.out_iters = iters; p.out_conv = converged;
  return launch_env_kernel(e, MODE_SOLVE, p, static_cast<cudaStream_t>(stream));
}

mapdn_status mapdn_droop(mapdn_env* e, int32_t nb, const double* p_load, const double* q_load, const double* p_sgen,
                         const double* s_rated, const double* q_max_manual, double gain, double tol, int32_t max_ite,
                         double* vm, double* q_sgen, double* loss, int32_t* iterations, void* stream) {
  if (!e || nb < 1 || !p_sgen || !s_rated || !q_max_manual || !q_sgen || !loss || !iterations ||
      (e->dims.n_load > 0 && (!p_load || !q_load)))
    return fail(MAPDN_ERR_INVALID, "null argument");
  if (max_ite < 1 || !(gain > 0.0)) return fail(MAPDN_ERR_INVALID, "droop: need max_ite >= 1 and gain > 0");
  MAPDN_ON_DEVICE(e->device);
  Params p = e->base;
  p.nb = nb;
  p.in_pl = p_load; p.in_ql = q_load; p.in_pv = p_sgen; p.in_q = nullptr;
  p.droop_s = s_rated; p.droop_qmm = q_max_manual; p.droop_gain = gain; p.droop_tol = tol; p.droop_max_ite = max_ite;
  p.out_vm = vm; p.out_va = nullptr; p.out_p = nullptr; p.out_q = nullptr; p.out_pl = nullptr;
  p.out_iters = iterations; p.out_conv = nullptr; p.droop_q_out = q_sgen; p.droop_loss_out = loss;
  return launch_env_kernel(e, MODE_DROOP, p, static_cast<cudaStream_t>(stream));
}

mapdn_status mapdn_get_ybus_dense(mapdn_env* e, double* g_host, double* b_host) {
  if (!e || !g_host || !b_host) return fail(MAPDN_ERR_INVALID, "null argument");
  const int n = e->dims.n_bus;
  std::fill(g_host, g_host + static_cast<size_t>(n) * n, 0.0);
  std::fill(b_host, b_host + static_cast<size_t>(n) * n, 0.0);
  for (int i = 0; i < n; ++i) { g_host[static_cast<size_t>(i) * n + i] = e->ydiag[2 * i]; b_host[static_cast<size_t>(i) * n + i] = e->ydiag[2 * i + 1]; }
  for (size_t k = 0; k < e->br_from.size(); ++k) {
    const size_t f = e->br_from[k], t = e->br_to[k];
    g_host[f * n + t] += e->ybr[8 * k + 2]; b_host[f * n + t] += e->ybr[8 * k + 3];
    g_host[t * n + f] += e->ybr[8 * k + 4]; b_host[t * n + f] += e->ybr[8 * k + 5];
  }
  return MAPDN_OK;
}

}  // extern "C"
