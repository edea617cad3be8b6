// hmpc_capi.cu — host side of libhector_mpc_b200.so: the C-ABI declared in include/hector_mpc_b200.h.
//
// Part 1 re-exports the reference's boundary (convexMPC_interface.h:39-43) on top of a one-robot
// context; part 2 is the batched interface.  There is no CPU solve path in this library.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <condition_variable>
#include <cstring>
#include <ctime>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/hector_mpc_b200.h"
#include "hmpc_device.cuh"
#include "hmpc_chain.h"

static_assert(sizeof(update_data_t) == 3016, "update_data_t must match convexMPC_interface.h:19-37");
static_assert(sizeof(problem_setup) == 16, "problem_setup must match convexMPC_interface.h:11-17");

namespace {

thread_local std::string g_err;

bool cuda_fail(cudaError_t e, const char* what)
{
  if (e == cudaSuccess) return false;
  g_err = std::string(what) + ": " + cudaGetErrorString(e);
  return true;
}
#define CK(call)                          \
  do {                                    \
    if (cuda_fail((call), #call)) return HMPC_ERR_CUDA; \
  } while (0)

// Small host worker pool for the byte-shuffling around the GPU call (packing records, widening results).
// Workers spin briefly after a job (a control loop calling at 200 Hz+ keeps them hot), then sleep.
class HostPool {
 public:
  explicit HostPool(int nworkers)
  {
    for (int i = 0; i < nworkers; i++) workers_.emplace_back([this, i] { run(i); });
  }
  ~HostPool()
  {
    {
      std::lock_guard<std::mutex> lk(m_);
      stop_ = true;
      gen_++;
    }
    cv_.notify_all();
    for (auto& t : workers_) t.join();
  }
  int size() const { return (int)workers_.size() + 1; }
  // run fn(part, nparts) on nparts = size() threads (the caller takes part 0); returns when all are done
  void parallel(const std::function<void(int, int)>& fn)
  {
    const int np = size();
    if (np == 1) { fn(0, 1); return; }
    fn_ = &fn;
    pending_.store(np - 1, std::memory_order_release);
    {
      std::lock_guard<std::mutex> lk(m_);
      gen_++;
    }
    cv_.notify_all();
    fn(0, np);
    while (pending_.load(std::memory_order_acquire) != 0) std::this_thread::yield();  // the parts are equal-sized: a short wait
  }

 private:
  void run(int idx)
  {
    unsigned seen = 0;
    for (;;) {
      // spin ~50 us for the next generation, then block
      bool got = false;
      const auto t0 = std::chrono::steady_clock::now();
      while (std::chrono::steady_clock::now() - t0 < std::chrono::microseconds(50)) {
        if (gen_relaxed() != seen) { got = true; break; }
      }
      if (!got) {
        std::unique_lock<std::mutex> lk(m_);
        cv_.wait(lk, [&] { return gen_ != seen; });
      }
      {
        std::lock_guard<std::mutex> lk(m_);
        seen = gen_;
        if (stop_) return;
      }
      (*fn_)(idx + 1, size());
      pending_.fetch_sub(1, std::memory_order_acq_rel);
    }
  }
  unsigned gen_relaxed()
  {
    std::lock_guard<std::mutex> lk(m_);
    return gen_;
  }
  std::vector<std::thread> workers_;
  std::mutex m_;
  std::condition_variable cv_;
  unsigned gen_ = 0;
  bool stop_ = false;
  const std::function<void(int, int)>* fn_ = nullptr;
  std::atomic<int> pending_{0};
};

constexpr int NCHUNK = 4;  // the host-buffer path pipelines pack / H2D / solve / D2H over this many chunks at most

// The slots of d_cls: eager device-resident chains use one, chains recorded into a CUDA graph the other (enqueue_solve).
constexpr int EAGER_SLOT = 0, CAPTURE_SLOT = 1, CLS_SLOTS = 2;
static_assert(CAPTURE_SLOT < CLS_SLOTS, "d_cls holds CLS_SLOTS slots");

// A view of rows [b0, b0 + nb) of the context's result staging (d_out, h_out).  The chunk of those rows starts at byte
// b0 * hmpc_ctx::row_bytes() and holds [nb][12N] float wrenches, then [nb] status words, then [nb][10] float torques.
// tau is null in a view without torques; bytes counts wrenches, status words and (if in the view) torques.
struct ResultRows { float* wrench; int* status; float* tau; size_t bytes; };

using hmpc::ClassCfg;

}  // namespace

struct hmpc_ctx {
  int device = 0, max_batch = 0, horizon = 0, rec_stride = 0, sm_count = 0;
  hmpc::SolverSettings cfg;
  ClassCfg cls[3];
  int ncls = 0;
  // refinement class (hmpc_set_refinement): instances beyond the conditioning limit are solved again with iterative
  // refinement against the stored Hessian instead of ending with code 4
  ClassCfg ref{};
  // the multi-query instantiations of the same classes (hmpc_solve_device_multi) and their scratch: d_mq + mq_off[c] for
  // class c (3: the refinement class), one row of hmpc::mq_scratch_floats per CTA
  ClassCfg mcls[3], mref{};
  float* d_mq = nullptr;
  size_t mq_off[4] = {};
  unsigned char* h_multi = nullptr;  // pinned, max_batch x (row, traj, wrench, status, cost) of a staged hmpc_solve_batch_multi
  // hmpc_solve_batch_states_multi (allocated by the first one): the candidates' trajectories [max_batch][12N], and pinned
  // max_batch x (state, command, wrench, status, cost, best) of a staged call
  float* d_smtraj = nullptr;
  unsigned char* h_smulti = nullptr;
  int* d_ref = nullptr;            // host-buffer path: [NCHUNK][1 + max_batch] refinement list length + list
  unsigned char* d_rec = nullptr;
  unsigned char* d_out = nullptr;  // host-buffer path: result staging (rows())
  int* d_status = nullptr;         // scratch status (assembly hook)
  int* d_counts = nullptr;         // [4] class list lengths (assembly hook)
  int* d_lists = nullptr;          // [NCHUNK][host_lists_ints] class lists (host-built, host-buffer path)
  int* d_cls = nullptr;            // [CLS_SLOTS][ClassSlot::cls_slot_ints] class-list lengths and lists (device-resident path)
  unsigned char* h_mask = nullptr; // pinned [max_batch]: the mask of hmpc_solve_batch_masked, read mapped by the in-place mode
  unsigned eager_calls = 0;        // eager device-resident chains so far: parity of the list lengths in use
  unsigned char* h_rec = nullptr;  // pinned
  unsigned char* h_out = nullptr;  // pinned mirror of d_out
  unsigned char* d_states = nullptr;  // hmpc_state_t staging of hmpc_solve_batch_states (row f-1)
  unsigned char* h_states = nullptr;  // pinned
  int* h_cls = nullptr;            // pinned [NCHUNK][host_lists_ints]: host-built class counts + lists (host-buffer path)
  cudaStream_t stream = nullptr;   // chunk 0 / single-robot stream
  cudaStream_t xstream[3] = {nullptr, nullptr, nullptr};  // further chunks of the pipelined host path
  HostPool* pool = nullptr;        // helper threads for packing / widening (large batches only)
  // multi-GPU (one process per GPU, batch sharded): NCCL communicator + double-buffered float results for the gather
  void* nccl = nullptr;            // ncclComm_t
  int shard_rank = 0, shard_world = 1;
  // [max_batch][12N] this rank's results of tick t / t+1.  Every sharded call leaves each robot's latest row in
  // shard_buf[(shard_tick - 1) & 1] (zeros before its first solve), gathering or not.
  float* shard_buf[2] = {nullptr, nullptr};
  unsigned shard_tick = 0;         // sharded calls that completed their buffer
  cudaStream_t gstream = nullptr;  // the gather runs here, behind `solved`, beside the next tick
  cudaEvent_t solved = nullptr, gathered[2] = {nullptr, nullptr};
  int* d_ws = nullptr;             // [max_batch][WS_STATE_INTS] working sets of the previous tick (closed-loop warm start)
  int warm_start = 1;              // the warm calls propose them to the next tick (HMPC_WARM_START=0: cold start every tick)
  int* d_shift = nullptr;          // [max_batch] per-robot shifts of hmpc_solve_batch_warm (staged copy)
  int* h_shift = nullptr;          // pinned [max_batch] the same, also read mapped by the zero-copy and in-place modes
  double* h_pred = nullptr;        // pinned [2][max_batch][12N]: wrenches in and plans out of a staged hmpc_predict_batch
                                   // (allocated by the first one)
  unsigned char* h_cert = nullptr; // pinned, max_batch x (row, wrench, certificate, multipliers) of a staged
                                   // hmpc_certify_batch (allocated by the first one)
  // caller-owned host buffers registered with hmpc_pin_host_buffer: hmpc_solve_batch lets the kernels read the
  // reference records from them and write results to them in place (no packing, no staging copies, no widening)
  struct Pin { char* base; size_t bytes; };   // what the caller asked for
  struct Run { uintptr_t lo, hi; };           // page runs actually registered with CUDA (arrays may share pages)
  std::vector<Pin> pins;
  std::vector<Run> runs;
  bool pinned(const void* p, size_t bytes) const
  {
    const char* q = static_cast<const char*>(p);
    for (const Pin& r : pins)
      if (q >= r.base && q + bytes <= r.base + r.bytes) return true;
    return false;
  }
  size_t row_bytes() const { return (size_t)12 * horizon * 4 + 4 + 40; }  // one robot's results in d_out / h_out
  ResultRows rows(unsigned char* base, int b0, int nb, bool tau = true) const
  {
    const size_t nw = (size_t)12 * horizon;
    unsigned char* p = base + (size_t)b0 * row_bytes();
    return {reinterpret_cast<float*>(p), reinterpret_cast<int*>(p + (size_t)nb * nw * 4),
            tau ? reinterpret_cast<float*>(p + (size_t)nb * (nw * 4 + 4)) : nullptr, (size_t)nb * (nw * 4 + 4 + (tau ? 40 : 0))};
  }
};

namespace {

cudaError_t prep_class(const ClassCfg& c, int* occ)
{
  cudaError_t e = cudaErrorInvalidDeviceFunction;
  // The attribute is per kernel instantiation and process-wide, and several contexts (other horizons, the
  // reference-style global context) share the runtime-horizon instantiations: always raise it to the device's opt-in
  // maximum instead of this context's carve-up, so no context can lower it under another's launches.
#define HMPC_PREP(ID, NT, MB, NF, CL) HMPC_PREP_K(ID, (hmpc::hmpc_solve_kernel<NT, MB, NF, CL>), NT)
#define HMPC_PREP_MQ(ID, NT, MB, NF, CL) HMPC_PREP_K(ID, (hmpc::hmpc_solve_kernel<NT, MB, NF, CL, true>), NT)
#define HMPC_PREP_K(ID, KERNEL, NT)                                                                    \
  case ID: {                                                                                           \
    auto k = KERNEL;                                                                                   \
    e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);              \
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, k, NT, c.smem);       \
    break;                                                                                             \
  }
  switch (c.variant) { HMPC_VARIANTS(HMPC_PREP) HMPC_MQ_VARIANTS(HMPC_PREP_MQ) }
#undef HMPC_PREP
#undef HMPC_PREP_MQ
#undef HMPC_PREP_K
  return e;
}

// programmatic dependent launch for the device-resident chain (classification -> class 0 -> class 1 -> class 2):
// every kernel of the chain may become resident while its predecessor drains and waits (griddepcontrol.wait) before it
// reads what the predecessor wrote.  HMPC_PDL=0 switches back to plain stream order.
bool pdl_enabled()
{
  static const bool on = !(getenv("HMPC_PDL") && atoi(getenv("HMPC_PDL")) == 0);
  return on;
}

template <typename... KArgs, typename... Args>
cudaError_t launch_chain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args... args)
{
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

// the shapes of the context's classes (hmpc::plan_classes) and what the device makes of them: resident CTAs per class;
// the same for the multi-query classes, and their scratch
int build_classes(hmpc_ctx* c)
{
  c->ncls = hmpc::plan_classes(c->horizon, c->cls, c->ref);
  if (c->ncls == 0 || hmpc::plan_classes(c->horizon, c->mcls, c->mref, true) != c->ncls) {
    g_err = "horizon too long for the built kernel variants";
    return HMPC_ERR_ARG;
  }
  size_t mq_rows = 0;
  for (int i = 0; i <= 2 * c->ncls + 1; i++) {
    const bool mq = i > c->ncls;
    const int j = mq ? i - c->ncls - 1 : i;
    ClassCfg& k = mq ? (j < c->ncls ? c->mcls[j] : c->mref) : (j < c->ncls ? c->cls[j] : c->ref);
    int occ = 0;
    if (cuda_fail(prep_class(k, &occ), "kernel attribute/occupancy (is this an sm_90a device?)")) return HMPC_ERR_CUDA;
    if (occ < 1) { g_err = "kernel does not fit on this device"; return HMPC_ERR_CUDA; }
    k.grid_cap = occ * c->sm_count;
    if (mq) {
      c->mq_off[j < c->ncls ? j : 3] = mq_rows * hmpc::mq_scratch_floats(c->horizon);
      mq_rows += hmpc::mq_scratch_ctas(k, c->max_batch);
    }
  }
  if (cuda_fail(cudaMalloc(&c->d_mq, mq_rows * hmpc::mq_scratch_floats(c->horizon) * sizeof(float)), "cudaMalloc multi-query scratch"))
    return HMPC_ERR_CUDA;
  return HMPC_OK;
}

long long* g_dbg_clk = nullptr;  // profiling hook (hmpc_debug_set_clock_buffer)

// one launch of class `cls` (0-2, or hmpc::REFINE_CLASS) over `count` instances, as many CTAs as are resident at most;
// with `mq` the class's multi-query instantiation
int launch_class(const hmpc_ctx* c, int cls, const hmpc::SolveIO& io, const hmpc::ChainLists& lists, int count, cudaStream_t st,
                 bool pdl = false, const hmpc::MultiIO* mq = nullptr)
{
  const ClassCfg& k = cls == hmpc::REFINE_CLASS ? (mq ? c->mref : c->ref) : (mq ? c->mcls[cls] : c->cls[cls]);
  hmpc::KernelArgs ka = mq ? hmpc::multi_launch_args(c->cfg, c->horizon, c->ncls, cls, k, io, lists, *mq)
                           : hmpc::launch_args(c->cfg, c->horizon, c->ncls, cls, k, io, lists);
  ka.dbg_clk = ka.dbg_H ? nullptr : g_dbg_clk;  // (the assembly dump is not stamped)
  const int grid = count < k.grid_cap ? count : k.grid_cap;
  cudaError_t e = cudaErrorInvalidDeviceFunction;
#define HMPC_LAUNCH(ID, NT, MB, NF, CL) \
  case ID: e = launch_chain(hmpc::hmpc_solve_kernel<NT, MB, NF, CL>, dim3(grid), dim3(NT), (size_t)k.smem, st, pdl, ka); break;
#define HMPC_LAUNCH_MQ(ID, NT, MB, NF, CL) \
  case ID: e = launch_chain(hmpc::hmpc_solve_kernel<NT, MB, NF, CL, true>, dim3(grid), dim3(NT), (size_t)k.smem, st, pdl, ka); break;
  switch (k.variant) { HMPC_VARIANTS(HMPC_LAUNCH) HMPC_MQ_VARIANTS(HMPC_LAUNCH_MQ) }
#undef HMPC_LAUNCH
#undef HMPC_LAUNCH_MQ
  CK(e);
  CK(cudaGetLastError());
  return HMPC_OK;
}

// the preparation kernel (hmpc_chain.h: prepare_args) on one thread per robot or list entry at most
int launch_prepare(const hmpc::PrepareArgs& pa, cudaStream_t st, bool pdl)
{
  CK(launch_chain(hmpc::hmpc_prepare_kernel, dim3(hmpc::prepare_grid(pa.batch)), dim3(hmpc::PREPARE_THREADS), 0, st, pdl,
                  pa.states, pa.batch, pa.N, pa.dtMPC, pa.records, pa.rec_stride, pa.list, pa.count));
  CK(cudaGetLastError());
  return HMPC_OK;
}

// the trajectory preparation of a multi-command states call (hmpc_chain.h: prepare_traj_args) on one thread per (robot or
// list entry, candidate) at most
int launch_prepare_traj(const hmpc::PrepareTrajArgs& pa, cudaStream_t st, bool pdl)
{
  CK(launch_chain(hmpc::hmpc_prepare_traj_kernel, dim3(hmpc::prepare_grid(pa.batch * pa.K)), dim3(hmpc::PREPARE_THREADS), 0, st,
                  pdl, pa.states, pa.batch, pa.K, pa.cmd, pa.N, pa.dtMPC, pa.traj, pa.list, pa.count));
  CK(cudaGetLastError());
  return HMPC_OK;
}

// the carry kernel (hmpc_chain.h: carry_grid): rows of `cur` the mask does not list get their bytes from `prev`
int launch_carry(const unsigned char* mask, int batch, int N, const float* prev, float* cur, cudaStream_t st)
{
  hmpc::hmpc_carry_kernel<<<hmpc::carry_grid(batch, N), hmpc::CARRY_THREADS, 0, st>>>(
      mask, batch, hmpc::carry_row_vecs(N), reinterpret_cast<const float4*>(prev), reinterpret_cast<float4*>(cur));
  CK(cudaGetLastError());
  return HMPC_OK;
}

// the prediction kernel (hmpc_chain.h: predict_grid) over B rows of `rows`, row_stride bytes apart
template <typename T>
int launch_predict(const hmpc_ctx* c, const void* rows, int row_stride, int B, const unsigned char* mask, const T* wrench,
                   T* pred, cudaStream_t st)
{
  hmpc::hmpc_predict_kernel<T><<<hmpc::predict_grid(B), hmpc::PREDICT_THREADS, 0, st>>>(
      static_cast<const unsigned char*>(rows), row_stride, B, c->horizon, c->cfg.dt, mask, wrench, pred);
  CK(cudaGetLastError());
  return HMPC_OK;
}

// the certificate kernel (hmpc_chain.h: certify_grid) over B rows of `rows` in layout `lay`
template <typename T>
int launch_certify(const hmpc_ctx* c, const void* rows, hmpc::RowLayout lay, int B, const unsigned char* mask, const T* wrench,
                   hmpc_certificate_t* cert, T* lambda, cudaStream_t st)
{
  hmpc::hmpc_certify_kernel<T><<<hmpc::certify_grid(B), hmpc::CERT_THREADS, 0, st>>>(
      static_cast<const unsigned char*>(rows), lay, B, c->horizon, c->cfg.dt, c->cfg.f_max, mask, wrench,
      reinterpret_cast<hmpc::CertOut*>(cert), lambda, nullptr);
  CK(cudaGetLastError());
  return HMPC_OK;
}

// the multi-query call's cost kernel (hmpc_chain.h: multi_cost_grid) over the B x K rows
template <typename T>
int launch_multi_cost(const hmpc_ctx* c, const void* rows, hmpc::RowLayout lay, int B, int K, const unsigned char* mask,
                      const float* traj, const T* wrench, double* cost, cudaStream_t st)
{
  hmpc::hmpc_multi_cost_kernel<T><<<hmpc::multi_cost_grid((long long)B * K), hmpc::PREDICT_THREADS, 0, st>>>(
      static_cast<const unsigned char*>(rows), lay, B, K, c->horizon, c->cfg.dt, mask, traj, wrench, cost);
  CK(cudaGetLastError());
  return HMPC_OK;
}

// the pick kernel of a multi-command states call (hmpc_chain.h: pick_grid) over the B robots
template <typename T>
int launch_pick(const hmpc_ctx* c, void* records, int B, int K, const unsigned char* mask, const float* traj, const T* wrench,
                const int* status, const double* cost, int* best, float* tau, cudaStream_t st)
{
  hmpc::hmpc_pick_kernel<T><<<hmpc::pick_grid(B), hmpc::PREDICT_THREADS, 0, st>>>(
      static_cast<unsigned char*>(records), c->rec_stride, B, K, c->horizon, c->cfg.f_max, mask, traj, wrench, status, cost, best,
      tau);
  CK(cudaGetLastError());
  return HMPC_OK;
}

}  // namespace

static_assert(sizeof(hmpc_certificate_t) == sizeof(hmpc::CertOut) && offsetof(hmpc_certificate_t, flags) ==
              offsetof(hmpc::CertOut, flags), "hmpc_certificate_t is the kernel's CertOut");
static_assert(HMPC_CERT_PASS == hmpc::CERT_PASS && HMPC_CERT_NONFINITE == hmpc::CERT_NONFINITE &&
              HMPC_CERT_SWING == hmpc::CERT_SWING && HMPC_CERT_STATIONARITY == hmpc::CERT_STATIONARITY &&
              HMPC_CERT_PRIMAL == hmpc::CERT_PRIMAL && HMPC_CERT_COMPLEMENTARITY == hmpc::CERT_COMPL,
              "certificate flag bits");
static_assert(HMPC_CERT_STATIONARITY_TOL == hmpc::CERT_STAT_TOL && HMPC_CERT_PRIMAL_TOL == hmpc::CERT_PRIMAL_TOL &&
              HMPC_CERT_COMPLEMENTARITY_TOL == hmpc::CERT_COMPL_TOL, "certificate thresholds");
static_assert(sizeof(update_data_t) == 3016 && offsetof(update_data_t, Alpha_K) == 1896 && offsetof(update_data_t, traj) == 168 &&
              offsetof(update_data_t, gait) == 1944, "hmpc_chain.h: update_rows");

// ---------------------------------------------------------------------------------------------------
// records
// ---------------------------------------------------------------------------------------------------
HMPC_EXTERNC size_t hmpc_record_bytes(int horizon)
{
  if (horizon < 1 || horizon > 18) return 0;
  size_t b = (size_t)(54 + 12 * horizon) * 4 + (size_t)2 * horizon;
  return (b + 15) / 16 * 16;
}

HMPC_EXTERNC int hmpc_pack_records(const update_data_t* in, int n, int horizon, void* out)
{
  const size_t stride = hmpc_record_bytes(horizon);
  if (!in || !out || n < 0 || stride == 0) { g_err = "hmpc_pack_records: bad argument"; return HMPC_ERR_ARG; }
  unsigned char* o = static_cast<unsigned char*>(out);
  for (int i = 0; i < n; i++, o += stride) {
    const update_data_t& u = in[i];
    if (i + 2 < n) {  // the live bytes of a record are ~11 scattered cache lines of 47: fetch ahead
      const char* nx = reinterpret_cast<const char*>(&in[i + 2]);
      for (int off = 0; off < (42 + 12 * horizon) * 4; off += 64) __builtin_prefetch(nx + off);
      __builtin_prefetch(nx + offsetof(update_data_t, Alpha_K));
      __builtin_prefetch(nx + offsetof(update_data_t, gait));
    }
    float* f = reinterpret_cast<float*>(o);
    memcpy(f, u.p, 42 * 4);  // p v q w r joint_angles yaw weights are contiguous in update_data_t
    memcpy(f + 42, u.Alpha_K, 48);
    memcpy(f + 54, u.traj, (size_t)48 * horizon);
    unsigned char* g = o + (size_t)(54 + 12 * horizon) * 4;
    memcpy(g, u.gait, (size_t)2 * horizon);
    memset(g + 2 * horizon, 0, stride - ((size_t)(54 + 12 * horizon) * 4 + 2 * horizon));
  }
  return HMPC_OK;
}

// ---------------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------------
HMPC_EXTERNC const char* hmpc_last_error(void) { return g_err.c_str(); }

// ---------------------------------------------------------------------------------------------------
// multi-GPU (SURVEY.md 8e): one process per GPU, contiguous batch slices, identical kernels, no data-path collective;
// ONE ncclAllGather of the float results when a consumer needs the whole batch on every device.  NCCL is looked up at
// run time (libnccl.so.2 — the copy the process already holds when PyTorch is loaded), so the library has no link
// dependency on it and single-GPU users never touch it.
// ---------------------------------------------------------------------------------------------------
struct Id128 { char b[128]; };  // ncclUniqueId, passed by value
namespace {
struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, Id128, int) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
}  // namespace
namespace {
NcclApi g_nccl;
bool nccl_load()
{
  if (g_nccl.h) return true;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) { g_err = std::string("NCCL not found: ") + dlerror(); return false; }
  g_nccl.GetUniqueId = reinterpret_cast<int (*)(void*)>(dlsym(h, "ncclGetUniqueId"));
  g_nccl.CommInitRank = reinterpret_cast<int (*)(void**, int, Id128, int)>(dlsym(h, "ncclCommInitRank"));
  g_nccl.AllGather = reinterpret_cast<int (*)(const void*, void*, size_t, int, void*, cudaStream_t)>(dlsym(h, "ncclAllGather"));
  g_nccl.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(h, "ncclCommDestroy"));
  g_nccl.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(h, "ncclGetErrorString"));
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllGather || !g_nccl.CommDestroy) {
    g_err = "NCCL library lacks ncclGetUniqueId / ncclCommInitRank / ncclAllGather / ncclCommDestroy";
    return false;
  }
  g_nccl.h = h;
  return true;
}
bool nccl_fail(int rc, const char* what)
{
  if (rc == 0) return false;
  g_err = std::string(what) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "NCCL error");
  return true;
}
void shard_release(hmpc_ctx* c)
{
  if (c->nccl && g_nccl.CommDestroy) g_nccl.CommDestroy(c->nccl);
  c->nccl = nullptr;
  for (int i = 0; i < 2; i++) {
    if (c->shard_buf[i]) cudaFree(c->shard_buf[i]);
    if (c->gathered[i]) cudaEventDestroy(c->gathered[i]);
    c->shard_buf[i] = nullptr;
    c->gathered[i] = nullptr;
  }
  if (c->solved) cudaEventDestroy(c->solved);
  if (c->gstream) cudaStreamDestroy(c->gstream);
  c->solved = nullptr;
  c->gstream = nullptr;
}
}  // namespace

HMPC_EXTERNC int hmpc_shard_unique_id(void* id128)
{
  if (!id128) { g_err = "hmpc_shard_unique_id: null argument"; return HMPC_ERR_ARG; }
  if (!nccl_load()) return HMPC_ERR_CUDA;
  if (nccl_fail(g_nccl.GetUniqueId(id128), "ncclGetUniqueId")) return HMPC_ERR_CUDA;
  return HMPC_OK;
}

HMPC_EXTERNC int hmpc_shard_init(hmpc_ctx* c, int rank, int world, const void* id128)
{
  if (!c || !id128 || world < 1 || rank < 0 || rank >= world) { g_err = "hmpc_shard_init: bad argument"; return HMPC_ERR_ARG; }
  if (c->nccl) { g_err = "hmpc_shard_init: context already belongs to a shard group"; return HMPC_ERR_ARG; }
  if (!nccl_load()) return HMPC_ERR_CUDA;
  CK(cudaSetDevice(c->device));
  Id128 id;
  memcpy(id.b, id128, 128);
  if (nccl_fail(g_nccl.CommInitRank(&c->nccl, world, id, rank), "ncclCommInitRank")) return HMPC_ERR_CUDA;
  c->shard_rank = rank;
  c->shard_world = world;
  const size_t nw = (size_t)12 * c->horizon;
  CK(cudaStreamCreateWithFlags(&c->gstream, cudaStreamNonBlocking));
  CK(cudaEventCreateWithFlags(&c->solved, cudaEventDisableTiming));
  for (int i = 0; i < 2; i++) {
    CK(cudaMalloc(&c->shard_buf[i], (size_t)c->max_batch * nw * sizeof(float)));
    // a robot no sharded call has solved yet is gathered as zeros (the masked calls carry unlisted rows forward)
    CK(cudaMemsetAsync(c->shard_buf[i], 0, (size_t)c->max_batch * nw * sizeof(float), c->stream));
    CK(cudaEventCreateWithFlags(&c->gathered[i], cudaEventDisableTiming));
  }
  return HMPC_OK;
}

HMPC_EXTERNC int hmpc_shard_wait(hmpc_ctx* c)
{
  if (!c || !c->nccl) { g_err = "hmpc_shard_wait: call hmpc_shard_init first"; return HMPC_ERR_ARG; }
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->gstream));
  return HMPC_OK;
}

HMPC_EXTERNC void hmpc_destroy(hmpc_ctx* c)
{
  if (!c) return;
  cudaSetDevice(c->device);
  for (const hmpc_ctx::Run& r : c->runs) cudaHostUnregister(reinterpret_cast<void*>(r.lo));
  c->runs.clear();
  c->pins.clear();
  if (c->d_rec) cudaFree(c->d_rec);
  if (c->d_out) cudaFree(c->d_out);
  if (c->d_status) cudaFree(c->d_status);
  if (c->d_counts) cudaFree(c->d_counts);
  if (c->d_lists) cudaFree(c->d_lists);
  if (c->d_cls) cudaFree(c->d_cls);
  if (c->d_ref) cudaFree(c->d_ref);
  if (c->d_mq) cudaFree(c->d_mq);
  if (c->h_multi) cudaFreeHost(c->h_multi);
  if (c->d_smtraj) cudaFree(c->d_smtraj);
  if (c->h_smulti) cudaFreeHost(c->h_smulti);
  shard_release(c);
  if (c->d_ws) cudaFree(c->d_ws);
  if (c->d_shift) cudaFree(c->d_shift);
  if (c->h_shift) cudaFreeHost(c->h_shift);
  if (c->h_pred) cudaFreeHost(c->h_pred);
  if (c->h_cert) cudaFreeHost(c->h_cert);
  if (c->h_mask) cudaFreeHost(c->h_mask);
  if (c->d_states) cudaFree(c->d_states);
  if (c->h_states) cudaFreeHost(c->h_states);
  if (c->h_rec) cudaFreeHost(c->h_rec);
  if (c->h_out) cudaFreeHost(c->h_out);
  if (c->h_cls) cudaFreeHost(c->h_cls);
  delete c->pool;
  if (c->stream) cudaStreamDestroy(c->stream);
  for (int i = 0; i < 3; i++)
    if (c->xstream[i]) cudaStreamDestroy(c->xstream[i]);
  delete c;
}

HMPC_EXTERNC hmpc_ctx* hmpc_create(int max_batch, int horizon, int device)
{
  if (max_batch < 1 || horizon < 1 || horizon > HMPC_MAX_HORIZON) {
    g_err = "hmpc_create: need max_batch >= 1 and 1 <= horizon <= 16";
    return nullptr;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= device || device < 0) {
    g_err = "hmpc_create: no usable CUDA device (this library has no CPU path)";
    return nullptr;
  }
  hmpc_ctx* c = new hmpc_ctx;
  c->device = device;
  c->max_batch = max_batch;
  c->horizon = horizon;
  c->rec_stride = (int)hmpc_record_bytes(horizon);
  cudaDeviceProp prop{};
  bool bad = cuda_fail(cudaSetDevice(device), "cudaSetDevice") ||
             cuda_fail(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties");
  if (!bad && (prop.major != 9 || prop.minor != 0)) {  // sm_90a code runs on compute capability 9.0 only
    g_err = "hmpc_create: kernels are built for sm_90a only; device is sm_" + std::to_string(prop.major) +
            std::to_string(prop.minor);
    bad = true;
  }
  if (!bad) {
    c->sm_count = prop.multiProcessorCount;
    bad = cuda_fail(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking), "cudaStreamCreate") ||
          cuda_fail(cudaStreamCreateWithFlags(&c->xstream[0], cudaStreamNonBlocking), "cudaStreamCreate") ||
          cuda_fail(cudaStreamCreateWithFlags(&c->xstream[1], cudaStreamNonBlocking), "cudaStreamCreate") ||
          cuda_fail(cudaStreamCreateWithFlags(&c->xstream[2], cudaStreamNonBlocking), "cudaStreamCreate") ||
          cuda_fail(cudaMalloc(&c->d_rec, (size_t)max_batch * c->rec_stride), "cudaMalloc records") ||
          cuda_fail(cudaMalloc(&c->d_out, (size_t)max_batch * c->row_bytes()), "cudaMalloc results") ||
          cuda_fail(cudaMalloc(&c->d_counts, 4 * sizeof(int)), "cudaMalloc counts") ||
          cuda_fail(cudaMalloc(&c->d_lists, (size_t)NCHUNK * hmpc::host_lists_ints(max_batch) * sizeof(int)), "cudaMalloc lists") ||
          cuda_fail(cudaMalloc(&c->d_ws, (size_t)max_batch * hmpc::WS_STATE_INTS * sizeof(int)), "cudaMalloc working sets") ||
          cuda_fail(cudaMemset(c->d_ws, 0, (size_t)max_batch * hmpc::WS_STATE_INTS * sizeof(int)), "cudaMemset working sets") ||
          cuda_fail(cudaMalloc(&c->d_shift, (size_t)max_batch * sizeof(int)), "cudaMalloc shifts") ||
          cuda_fail(cudaMallocHost(&c->h_shift, (size_t)max_batch * sizeof(int)), "cudaMallocHost shifts") ||
          cuda_fail(cudaMallocHost(&c->h_mask, (size_t)max_batch), "cudaMallocHost mask") ||
          cuda_fail(cudaMalloc(&c->d_cls, (size_t)CLS_SLOTS * hmpc::ClassSlot::cls_slot_ints(max_batch) * sizeof(int)), "cudaMalloc class lists") ||
          cuda_fail(cudaMemset(c->d_cls, 0, (size_t)CLS_SLOTS * hmpc::ClassSlot::cls_slot_ints(max_batch) * sizeof(int)), "cudaMemset class lists") ||
          cuda_fail(cudaMalloc(&c->d_ref, (size_t)NCHUNK * (1 + (size_t)max_batch) * sizeof(int)), "cudaMalloc refinement lists") ||
          cuda_fail(cudaMalloc(&c->d_status, (size_t)max_batch * 4), "cudaMalloc status") ||
          cuda_fail(cudaMalloc(&c->d_states, (size_t)max_batch * sizeof(hmpc_state_t)), "cudaMalloc states") ||
          cuda_fail(cudaMallocHost(&c->h_states, (size_t)max_batch * sizeof(hmpc_state_t)), "cudaMallocHost states") ||
          cuda_fail(cudaMallocHost(&c->h_rec, (size_t)max_batch * c->rec_stride), "cudaMallocHost records") ||
          cuda_fail(cudaMallocHost(&c->h_out, (size_t)max_batch * c->row_bytes()), "cudaMallocHost results") ||
          cuda_fail(cudaMallocHost(&c->h_cls, (size_t)NCHUNK * hmpc::host_lists_ints(max_batch) * sizeof(int)), "cudaMallocHost lists") ||
          build_classes(c) != HMPC_OK;
  }
  if (!bad) {
    const char* br = getenv("HMPC_BLOCK_ROUNDS");
    if (br) c->cfg.block_rounds = atoi(br);
    if (const char* bm = getenv("HMPC_BLOCK_MIN")) c->cfg.block_min = atoi(bm);
    if (const char* km = getenv("HMPC_KAPPA_MAX")) c->cfg.kappa_max = atof(km);
    if (const char* kr = getenv("HMPC_KAPPA_REFINE")) c->cfg.kappa_refine = atof(kr);
    if (const char* kx = getenv("HMPC_KAPPA_MAX_REFINED")) c->cfg.kappa_max_refined = atof(kx);
    const char* ls = getenv("HMPC_LOCKSTEP");
    if (ls) c->cfg.lockstep = atoi(ls);
    const char* wm = getenv("HMPC_WARM_START");
    if (wm) c->warm_start = atoi(wm);
  }
  if (!bad && max_batch >= 256) {
    const char* e = getenv("HMPC_HOST_THREADS");
    int nt = e ? atoi(e) : 4;
    const int hw = (int)std::thread::hardware_concurrency();
    if (hw > 0 && nt > hw) nt = hw;
    if (nt > 1) c->pool = new HostPool(nt - 1);
  }
  if (bad) {
    std::string keep = g_err;
    hmpc_destroy(c);
    g_err = keep;
    return nullptr;
  }
  return c;
}

HMPC_EXTERNC int hmpc_set_problem(hmpc_ctx* c, const problem_setup* s)
{
  if (!c || !s) { g_err = "hmpc_set_problem: null argument"; return HMPC_ERR_ARG; }
  if (s->horizon != c->horizon) { g_err = "hmpc_set_problem: horizon differs from the context's"; return HMPC_ERR_ARG; }
  c->cfg.dt = s->dt;
  c->cfg.f_max = s->f_max;
  return HMPC_OK;
}

namespace {
// The device-resident chain: one launch per class, all enqueued on `st`; with io.mask (device-readable [B]) the selection
// kernel first, and with io.states the preparation of the robots class 0 runs over (hmpc_chain.h).  No classification kernel: the class-0 launch runs over every instance (or, in a masked call, over the list
// the selection kernel built from the mask) and hands the ones with more stance blocks than it holds to class 1's list.
// An eager chain uses the parity of its call count: the previous call's class-0 launch zeroed those lengths.  A graph
// replays the lengths it was recorded with and nothing zeroes them between replays, so a chain recorded into a graph
// uses the capture slot, starts with a memset node that zeroes both parities (the wave-barrier counter and the
// refinement list length included), and leaves the eager call count alone.
// With `mq`, the multi-query instantiations of the classes run the chain (hmpc_chain.h: MultiIO): class 0 over the robots,
// the later classes over lists of up to io.batch * K candidates.
int enqueue_solve(hmpc_ctx* c, const hmpc::SolveIO& io, cudaStream_t st, const hmpc::MultiIO* mq = nullptr)
{
  if (io.batch > c->max_batch) { g_err = "batch exceeds the context's capacity"; return HMPC_ERR_ARG; }
  CK(cudaSetDevice(c->device));
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  CK(cudaStreamIsCapturing(st, &cap));
  const bool capturing = cap != cudaStreamCaptureStatusNone;
  const int slot = capturing ? CAPTURE_SLOT : EAGER_SLOT;
  const hmpc::ClassSlot s{c->d_cls + (size_t)slot * hmpc::ClassSlot::cls_slot_ints(c->max_batch), c->max_batch,
                          capturing ? 0 : (int)(c->eager_calls++ & 1u)};
  if (capturing) CK(cudaMemsetAsync(s.base, 0, hmpc::ClassSlot::HEAD_INTS * sizeof(int), st));
  const hmpc::ChainLists lists = hmpc::slot_lists(s, io.mask != nullptr, c->cfg.refine);
  const bool pdl = pdl_enabled();
  if (io.mask) {
    // counts[0] of this parity was cleared by the previous call's class-0 launch: the kernel waits for it (griddepcontrol.wait)
    // before its first store, and class 0 reads the list after its own wait
    CK(launch_chain(hmpc::hmpc_select_kernel<hmpc::SELECT_THREADS>, dim3(1), dim3(hmpc::SELECT_THREADS), 0, st, pdl, io.mask,
                    io.batch, s.list0(), s.counts()));
    CK(cudaGetLastError());
  }
  if (io.states) {
    // the states chain: records of the listed robots (every robot without a mask) into io.records, read by class 0; with
    // commands, then their candidates' trajectories
    if (int rc = launch_prepare(hmpc::prepare_args(c->horizon, io, lists), st, pdl)) return rc;
    if (mq && mq->cmd)
      if (int rc = launch_prepare_traj(hmpc::prepare_traj_args(c->horizon, io, lists, *mq), st, pdl)) return rc;
  }
  const int items = mq ? io.batch * mq->K : io.batch;
  for (int i = 0; i < c->ncls; i++)
    if (int rc = launch_class(c, i, io, lists, i == 0 ? io.batch : items, st, pdl, mq)) return rc;
  // the refinement class at the end of the chain: exits at once when nobody was handed over
  if (c->cfg.refine) return launch_class(c, hmpc::REFINE_CLASS, io, lists, items, st, pdl, mq);
  return HMPC_OK;
}

// a device-resident call on device records and outputs.  warm: robot i's proposal is its set in the context's d_ws, moved
// io.shifts[i] steps (NULL: every robot one step, the closed loop's tick); HMPC_WARM_START=0 makes it a cold solve
hmpc::SolveIO device_call(const hmpc_ctx* c, const void* d_records, int B, float* d_wrench, int* d_status, float* d_tau, bool warm)
{
  hmpc::SolveIO io;
  io.records = d_records;
  io.batch = B;
  io.wrench = d_wrench;
  io.status = d_status;
  io.tau = d_tau;
  if (warm && c->warm_start) io.ws = c->d_ws, io.warm = true;
  return io;
}

// Host-buffer path, staged: the host has the contact tables in hand while it packs, so it builds the class lists itself
// (hmpc::classify_host) and launches only the non-empty classes — no classification kernel, no empty launches.
// Working-set overflow cannot escalate here (enqueue_overflow_retry), nor can the refinement class run (enqueue_refine_retry).
// A chunk is robots [b0, b0 + nb) on stream st with their device views (io), their host-built class lists (lists; d_lists:
// the device copy) and their refinement list (ref; null while refinement is off).
struct Chunk { int b0, nb; cudaStream_t st; hmpc::SolveIO io; int *lists, *d_lists, *ref; };

int enqueue_solve_hostlists(hmpc_ctx* c, const Chunk& ch, bool zero_copy)
{
  int* h_block = ch.lists;
  int* d_block = zero_copy ? h_block : ch.d_lists;  // zero-copy: pinned + mapped, the kernels read the lists over PCIe
  if (!zero_copy) {  // counts + class-0 list (+ class-1 list when it is not empty) in one copy
    const size_t ints = h_block[1] > 0 ? hmpc::host_list(h_block, c->max_batch, 1) - h_block + h_block[1] : hmpc::HOST_LIST_HEAD + h_block[0];
    CK(cudaMemcpyAsync(d_block, h_block, ints * sizeof(int), cudaMemcpyHostToDevice, ch.st));
  }
  const hmpc::ChainLists lists = hmpc::host_lists(d_block, c->max_batch, ch.ref, false);
  if (ch.ref) CK(cudaMemsetAsync(lists.ref_count, 0, sizeof(int), ch.st));
  for (int i = 0; i < 2; i++)
    if (h_block[i] > 0)
      if (int rc = launch_class(c, i, ch.io, lists, h_block[i], ch.st)) return rc;
  return HMPC_OK;
}

// Working-set overflow in a host-list launch (rare: massively degenerate optima).  Only the instances that overflowed are
// solved again, from where the device-resident chain would have taken them: class 0's by class 1, class 1's by class 2,
// with escalation from the one to the other.  The rest of the chunk keeps its results and its recorded working sets, and an
// instance that overflowed kept its proposal (the kernel does not record a set for it), so results, statuses and working
// sets are those of the device-resident path.  The chunk's class lists are reused for the retry's.
// `mask` (the chunk's, host) or NULL: the status words of robots it does not list are stale and are not looked at.
int enqueue_overflow_retry(hmpc_ctx* c, const Chunk& ch, const int* h_status, const unsigned char* mask)
{
  const int mb = c->max_batch, nb = ch.nb;
  int* h_block = ch.lists;
  std::vector<char> was_cls1(nb, 0);
  for (int j = 0; j < h_block[1]; j++) was_cls1[hmpc::host_list(h_block, mb, 1)[j]] = 1;
  int n[3] = {0, 0, 0};
  for (int i = 0; i < nb; i++) {
    if ((mask && !mask[i]) || HMPC_STATUS_CODE(h_status[i]) != hmpc::ST_WS_CAP) continue;
    const int next = was_cls1[i] ? 2 : 1;
    if (next < c->ncls) hmpc::host_list(h_block, mb, next)[n[next]++] = i;  // (class 1 as the last class: its overflow is final)
  }
  h_block[0] = 0;
  h_block[1] = n[1];
  h_block[2] = n[2];
  h_block[3] = 0;
  CK(cudaMemcpyAsync(ch.d_lists, h_block, (hmpc::host_list(h_block, mb, 2) - h_block + n[2]) * sizeof(int), cudaMemcpyHostToDevice, ch.st));
  const hmpc::ChainLists lists = hmpc::host_lists(ch.d_lists, mb, ch.ref, true);
  for (int i = 1; i < c->ncls; i++) {
    const int cnt = (i == 1) ? n[1] : n[1] + n[2];  // class 2's list grows by class 1's escalations
    if (cnt > 0)
      if (int rc = launch_class(c, i, ch.io, lists, cnt, ch.st)) return rc;
  }
  return HMPC_OK;
}

// Refinement in a host-list launch: the kernels pushed the instances beyond the conditioning limit to the chunk's refinement
// list (device memory), and the refinement class solves them as it does at the end of the device-resident chain.  Called
// when refinement is on and a status of the chunk has code 4 (a non-positive pivot is not on the list).
int enqueue_refine_retry(hmpc_ctx* c, const Chunk& ch)
{
  return launch_class(c, hmpc::REFINE_CLASS, ch.io, hmpc::host_lists(ch.d_lists, c->max_batch, ch.ref, false), ch.nb, ch.st);
}
}  // namespace

// The kernels stage a record with a 1-D bulk copy (cp.async.bulk), whose global source must be 16-byte aligned: the record
// stride is a multiple of 16 by construction, the base pointer is the caller's (a sliced tensor view may not be).
static int check_device_records(const hmpc_ctx* c, const void* d_records, int B, const char* who)
{
  if (B > c->max_batch) { g_err = std::string(who) + ": batch exceeds the context's capacity"; return HMPC_ERR_ARG; }
  if (reinterpret_cast<uintptr_t>(d_records) & 15u) { g_err = std::string(who) + ": d_records must be 16-byte aligned"; return HMPC_ERR_ARG; }
  return HMPC_OK;
}

// profiling hook: device buffer [batch][32] of clock64() stage timestamps, or NULL to switch off
HMPC_EXTERNC void hmpc_debug_set_clock_buffer(long long* d_buf) { g_dbg_clk = d_buf; }

// fault-injection hook (tests): the next n host-buffer solves return HMPC_ERR_CUDA without touching the device — what a
// run-time CUDA failure looks like to the callers (the reference boundary's status path, tests/test_zzz_reference_status_path.py)
namespace { int g_fail_next_solves = 0; }
HMPC_EXTERNC void hmpc_debug_fail_next_solves(int n) { g_fail_next_solves = n; }

HMPC_EXTERNC int hmpc_launches_per_solve(const hmpc_ctx* c) { return c ? c->ncls + (c->cfg.refine ? 1 : 0) : 0; }

HMPC_EXTERNC int hmpc_set_refinement(hmpc_ctx* c, int on)
{
  if (!c) { g_err = "hmpc_set_refinement: null context"; return HMPC_ERR_ARG; }
  c->cfg.refine = on ? 1 : 0;
  return HMPC_OK;
}

// launch configuration of class `cls` (HMPC_REFINEMENT_CLASS: the refinement class): out[0..5] = threads, dynamic smem
// bytes, working-set capacity, resident-grid cap (CTAs), max blocks of 6 variables, sweep strip width
HMPC_EXTERNC int hmpc_class_config(const hmpc_ctx* c, int cls, int* out)
{
  if (!c || !out || cls < 0 || (cls >= c->ncls && cls != HMPC_REFINEMENT_CLASS)) return HMPC_ERR_ARG;
  const ClassCfg& k = cls == HMPC_REFINEMENT_CLASS ? c->ref : c->cls[cls];
  out[0] = k.threads; out[1] = k.smem; out[2] = k.qmax; out[3] = k.grid_cap; out[4] = k.nb_cap;
  out[5] = 8;  // sweep tile edge (8x8 mma.m8n8k4.f64 accumulator tiles)
  return HMPC_OK;
}

HMPC_EXTERNC int hmpc_solve_device(hmpc_ctx* c, const void* d_records, int B, float* d_wrench, int* d_status,
                                   void* stream)
{
  if (!c || !d_records || !d_wrench || !d_status || B < 0) { g_err = "hmpc_solve_device: bad argument"; return HMPC_ERR_ARG; }
  if (B == 0) return HMPC_OK;
  if (int rc = check_device_records(c, d_records, B, "hmpc_solve_device")) return rc;
  return enqueue_solve(c, device_call(c, d_records, B, d_wrench, d_status, nullptr, false), static_cast<cudaStream_t>(stream));
}

HMPC_EXTERNC int hmpc_solve_device_ex(hmpc_ctx* c, const void* d_records, int B, float* d_wrench, int* d_status,
                                      float* d_tau, void* stream)
{
  if (!c || !d_records || !d_wrench || !d_status || B < 0) { g_err = "hmpc_solve_device_ex: bad argument"; return HMPC_ERR_ARG; }
  if (B == 0) return HMPC_OK;
  if (int rc = check_device_records(c, d_records, B, "hmpc_solve_device_ex")) return rc;
  return enqueue_solve(c, device_call(c, d_records, B, d_wrench, d_status, d_tau, false), static_cast<cudaStream_t>(stream));
}

HMPC_EXTERNC int hmpc_solve_device_warm(hmpc_ctx* c, const void* d_records, int B, float* d_wrench, int* d_status, float* d_tau,
                                        const int* d_shift, void* stream)
{
  if (!c || !d_records || !d_wrench || !d_status || B < 0) { g_err = "hmpc_solve_device_warm: bad argument"; return HMPC_ERR_ARG; }
  if (B == 0) return HMPC_OK;
  if (int rc = check_device_records(c, d_records, B, "hmpc_solve_device_warm")) return rc;
  hmpc::SolveIO io = device_call(c, d_records, B, d_wrench, d_status, d_tau, true);
  io.shifts = d_shift;
  return enqueue_solve(c, io, static_cast<cudaStream_t>(stream));
}

HMPC_EXTERNC int hmpc_solve_device_masked(hmpc_ctx* c, const void* d_records, int B, const unsigned char* d_mask, float* d_wrench,
                                          int* d_status, float* d_tau, const int* d_shift, void* stream)
{
  if (!c || !d_records || !d_mask || !d_wrench || !d_status || B < 0) {
    g_err = "hmpc_solve_device_masked: bad argument";
    return HMPC_ERR_ARG;
  }
  if (B == 0) return HMPC_OK;
  if (int rc = check_device_records(c, d_records, B, "hmpc_solve_device_masked")) return rc;
  hmpc::SolveIO io = device_call(c, d_records, B, d_wrench, d_status, d_tau, true);
  io.shifts = d_shift;
  io.mask = d_mask;
  return enqueue_solve(c, io, static_cast<cudaStream_t>(stream));
}

HMPC_EXTERNC int hmpc_assemble_device(hmpc_ctx* c, const void* d_records, int B, float* d_H, float* d_g,
                                      float* d_Fblk, float* d_lb, float* d_ub, void* stream)
{
  if (!c || !d_records || !d_H || !d_g || !d_Fblk || !d_lb || !d_ub || B < 0) {
    g_err = "hmpc_assemble_device: bad argument";
    return HMPC_ERR_ARG;
  }
  if (B == 0) return HMPC_OK;
  if (int rc = check_device_records(c, d_records, B, "hmpc_assemble_device")) return rc;
  CK(cudaSetDevice(c->device));
  // the last class over every robot (no list), dumping its QP data
  hmpc::SolveIO io = device_call(c, d_records, B, nullptr, c->d_status, nullptr, false);
  io.dump_H = d_H;
  io.dump_g = d_g;
  io.dump_F = d_Fblk;
  io.dump_lb = d_lb;
  io.dump_ub = d_ub;
  hmpc::ChainLists lists;
  lists.counts = c->d_counts;
  return launch_class(c, c->ncls - 1, io, lists, B, static_cast<cudaStream_t>(stream));
}

static_assert(sizeof(hmpc_state_t) == 352 && offsetof(hmpc_state_t, gait) == 39 * 8, "hmpc_state_t layout (hmpc_prepare_kernel)");

HMPC_EXTERNC int hmpc_prepare_device(hmpc_ctx* c, const hmpc_state_t* d_states, int B, double dtMPC, void* d_records,
                                     void* stream)
{
  if (!c || !d_states || !d_records || B < 0) { g_err = "hmpc_prepare_device: bad argument"; return HMPC_ERR_ARG; }
  if (B == 0) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  hmpc::SolveIO io;
  io.states = d_states;
  io.records = d_records;
  io.batch = B;
  io.dt_mpc = dtMPC;
  return launch_prepare(hmpc::prepare_args(c->horizon, io, hmpc::ChainLists{}), static_cast<cudaStream_t>(stream), false);
}

HMPC_EXTERNC int hmpc_solve_states_device_masked(hmpc_ctx* c, const hmpc_state_t* d_states, int B, const unsigned char* d_mask,
                                                 double dtMPC, void* d_records, float* d_wrench, int* d_status, float* d_tau,
                                                 const int* d_shift, void* stream)
{
  if (!c || !d_states || !d_mask || !d_records || !d_wrench || !d_status || B < 0) {
    g_err = "hmpc_solve_states_device_masked: bad argument";
    return HMPC_ERR_ARG;
  }
  if (B == 0) return HMPC_OK;
  if (int rc = check_device_records(c, d_records, B, "hmpc_solve_states_device_masked")) return rc;
  hmpc::SolveIO io = device_call(c, d_records, B, d_wrench, d_status, d_tau, true);
  io.shifts = d_shift;
  io.mask = d_mask;
  io.states = d_states;
  io.dt_mpc = dtMPC;
  return enqueue_solve(c, io, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------
// the MPC's plan: predicted states under the discrete model of the solved QP (hmpc_predict_kernel)
// ---------------------------------------------------------------------------------------------------
HMPC_EXTERNC int hmpc_predict_device(hmpc_ctx* c, const void* d_records, int B, const unsigned char* d_mask, const float* d_wrench,
                                     float* d_pred, void* stream)
{
  if (!c || !d_records || !d_wrench || !d_pred || B < 0 || B > c->max_batch) {
    g_err = "hmpc_predict_device: bad argument (null pointer or batch > capacity)";
    return HMPC_ERR_ARG;
  }
  if (B == 0) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  return launch_predict(c, d_records, c->rec_stride, B, d_mask, d_wrench, d_pred, static_cast<cudaStream_t>(stream));
}

// test hook: 1 when the last hmpc_predict_batch that launched ran in place, 0 when it staged, -1 before any
namespace { int g_predict_in_place = -1; }
HMPC_EXTERNC int hmpc_debug_last_predict_in_place(void) { return g_predict_in_place; }

// In place when the records, the wrenches and the plans lie in buffers registered with hmpc_pin_host_buffer: the kernel reads
// the update_data_t rows and the double wrenches where they lie and writes the plans there.  Otherwise the listed robots'
// first 19 floats go to the record staging (h_rec, record stride) and their wrenches to h_pred, which the kernel reads
// mapped, and their plans come back from h_pred.  The same kernel on the same bytes: both modes give the same plans.
HMPC_EXTERNC int hmpc_predict_batch(hmpc_ctx* c, const update_data_t* in, int B, const unsigned char* mask, const double* wrench,
                                    double* pred_out)
{
  if (!c || !in || !wrench || !pred_out || B < 0 || B > c->max_batch) {
    g_err = "hmpc_predict_batch: bad argument (null pointer or batch > capacity)";
    return HMPC_ERR_ARG;
  }
  if (B == 0) return HMPC_OK;
  if (mask && std::all_of(mask, mask + B, [](unsigned char m) { return m == 0; })) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  const size_t nw = (size_t)12 * c->horizon, rs = (size_t)c->rec_stride;
  const unsigned char* m = nullptr;
  if (mask) {
    memcpy(c->h_mask, mask, (size_t)B);  // pinned: the kernel reads it mapped
    m = c->h_mask;
  }
  auto listed = [&](int i) { return !mask || mask[i] != 0; };
  if (c->pinned(in, (size_t)B * sizeof(update_data_t)) && c->pinned(wrench, B * nw * sizeof(double)) &&
      c->pinned(pred_out, B * nw * sizeof(double))) {
    g_predict_in_place = 1;
    if (int rc = launch_predict(c, in, (int)sizeof(update_data_t), B, m, wrench, pred_out, c->stream)) return rc;
    CK(cudaStreamSynchronize(c->stream));
    return HMPC_OK;
  }
  g_predict_in_place = 0;
  if (!c->h_pred) CK(cudaMallocHost(&c->h_pred, 2 * (size_t)c->max_batch * nw * sizeof(double)));
  double* hw = c->h_pred;
  double* hp = c->h_pred + (size_t)c->max_batch * nw;
  for (int i = 0; i < B; i++)
    if (listed(i)) {
      memcpy(c->h_rec + i * rs, in[i].p, 19 * sizeof(float));  // p v q w r, contiguous in update_data_t
      memcpy(hw + i * nw, wrench + i * nw, nw * sizeof(double));
    }
  if (int rc = launch_predict(c, c->h_rec, c->rec_stride, B, m, hw, hp, c->stream)) return rc;
  CK(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < B; i++)
    if (listed(i)) memcpy(pred_out + i * nw, hp + i * nw, nw * sizeof(double));
  return HMPC_OK;
}

// ---------------------------------------------------------------------------------------------------
// the certificate: first-order optimality of a wrench for its row (hmpc_certify_kernel)
// ---------------------------------------------------------------------------------------------------
HMPC_EXTERNC int hmpc_certify_device(hmpc_ctx* c, const void* d_records, int B, const unsigned char* d_mask,
                                     const float* d_wrench, hmpc_certificate_t* d_cert, float* d_lambda, void* stream)
{
  if (!c || !d_records || !d_wrench || !d_cert || B < 0 || B > c->max_batch) {
    g_err = "hmpc_certify_device: bad argument (null pointer or batch > capacity)";
    return HMPC_ERR_ARG;
  }
  if (B == 0) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  return launch_certify(c, d_records, hmpc::packed_rows(c->horizon), B, d_mask, d_wrench, d_cert, d_lambda,
                        static_cast<cudaStream_t>(stream));
}

// test hook: 1 when the last hmpc_certify_batch that launched ran in place, 0 when it staged, -1 before any
namespace { int g_certify_in_place = -1; }
HMPC_EXTERNC int hmpc_debug_last_certify_in_place(void) { return g_certify_in_place; }

// In place when the rows, the wrenches, the certificates and the multipliers (when asked for) lie in registered buffers.
// Otherwise the listed robots' update_data_t rows and wrenches go to h_cert, which the kernel reads mapped in the same
// layout, and their certificates and multipliers come back from it.  The same kernel on the same bytes either way.
HMPC_EXTERNC int hmpc_certify_batch(hmpc_ctx* c, const update_data_t* in, int B, const unsigned char* mask, const double* wrench,
                                    hmpc_certificate_t* cert_out, double* lambda_out)
{
  if (!c || !in || !wrench || !cert_out || B < 0 || B > c->max_batch) {
    g_err = "hmpc_certify_batch: bad argument (null pointer or batch > capacity)";
    return HMPC_ERR_ARG;
  }
  if (B == 0) return HMPC_OK;
  if (mask && std::all_of(mask, mask + B, [](unsigned char m) { return m == 0; })) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  const size_t nw = (size_t)12 * c->horizon, nl = (size_t)16 * c->horizon;
  const unsigned char* m = nullptr;
  if (mask) {
    memcpy(c->h_mask, mask, (size_t)B);  // pinned: the kernel reads it mapped
    m = c->h_mask;
  }
  auto listed = [&](int i) { return !mask || mask[i] != 0; };
  if (c->pinned(in, (size_t)B * sizeof(update_data_t)) && c->pinned(wrench, B * nw * sizeof(double)) &&
      c->pinned(cert_out, B * sizeof(hmpc_certificate_t)) && (!lambda_out || c->pinned(lambda_out, B * nl * sizeof(double)))) {
    g_certify_in_place = 1;
    if (int rc = launch_certify(c, in, hmpc::update_rows(), B, m, wrench, cert_out, lambda_out, c->stream)) return rc;
    CK(cudaStreamSynchronize(c->stream));
    return HMPC_OK;
  }
  g_certify_in_place = 0;
  const size_t mb = (size_t)c->max_batch;
  if (!c->h_cert)
    CK(cudaMallocHost(&c->h_cert, mb * (sizeof(update_data_t) + (nw + nl) * sizeof(double) + sizeof(hmpc_certificate_t))));
  update_data_t* hr = reinterpret_cast<update_data_t*>(c->h_cert);
  double* hw = reinterpret_cast<double*>(hr + mb);
  double* hl = hw + mb * nw;
  hmpc_certificate_t* hc = reinterpret_cast<hmpc_certificate_t*>(hl + mb * nl);
  for (int i = 0; i < B; i++)
    if (listed(i)) {
      hr[i] = in[i];
      memcpy(hw + i * nw, wrench + i * nw, nw * sizeof(double));
    }
  if (int rc = launch_certify(c, hr, hmpc::update_rows(), B, m, hw, hc, lambda_out ? hl : nullptr, c->stream)) return rc;
  CK(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < B; i++)
    if (listed(i)) {
      cert_out[i] = hc[i];
      if (lambda_out) memcpy(lambda_out + i * nl, hl + i * nl, nl * sizeof(double));
    }
  return HMPC_OK;
}

// ---------------------------------------------------------------------------------------------------
// several reference trajectories per robot (hmpc_chain.h: MultiIO)
// ---------------------------------------------------------------------------------------------------
static int check_multi(const hmpc_ctx* c, int B, int K, const char* who)
{
  if (B < 0 || K < 1 || (long long)B * K > c->max_batch) {
    g_err = std::string(who) + ": bad argument (B < 0, K < 1 or B*K > capacity)";
    return HMPC_ERR_ARG;
  }
  return HMPC_OK;
}

static hmpc::MultiIO multi_io(const hmpc_ctx* c, const float* traj, int K)
{
  hmpc::MultiIO mq;
  mq.traj = traj;
  mq.K = K;
  for (int i = 0; i < 4; i++) mq.scratch[i] = c->d_mq + c->mq_off[i];
  return mq;
}

HMPC_EXTERNC int hmpc_solve_device_multi(hmpc_ctx* c, const void* d_records, int B, int K, const float* d_traj,
                                         const unsigned char* d_mask, float* d_wrench, int* d_status, double* d_cost,
                                         void* stream)
{
  if (!c || !d_records || !d_traj || !d_wrench || !d_status) { g_err = "hmpc_solve_device_multi: null argument"; return HMPC_ERR_ARG; }
  if (int rc = check_multi(c, B, K, "hmpc_solve_device_multi")) return rc;
  if (B == 0) return HMPC_OK;
  if (int rc = check_device_records(c, d_records, B, "hmpc_solve_device_multi")) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  hmpc::SolveIO io = device_call(c, d_records, B, d_wrench, d_status, nullptr, false);
  io.mask = d_mask;
  const hmpc::MultiIO mq = multi_io(c, d_traj, K);
  if (int rc = enqueue_solve(c, io, st, &mq)) return rc;
  if (!d_cost) return HMPC_OK;
  return launch_multi_cost(c, d_records, hmpc::packed_rows(c->horizon), B, K, d_mask, d_traj, d_wrench, d_cost, st);
}

namespace { int g_multi_in_place = -1; }
HMPC_EXTERNC int hmpc_debug_last_multi_in_place(void) { return g_multi_in_place; }

// The device-resident chain in the in-place mode (the kernels gather the update_data_t rows and store double wrenches), on the
// caller's arrays when they are pinned, else on copies of the listed robots' rows in h_multi, which the kernels read mapped.
HMPC_EXTERNC int hmpc_solve_batch_multi(hmpc_ctx* c, const update_data_t* in, int B, int K, const float* traj,
                                        const unsigned char* mask, double* wrench_out, int* status, double* cost_out)
{
  if (!c || !in || !traj || !wrench_out || !status) { g_err = "hmpc_solve_batch_multi: null argument"; return HMPC_ERR_ARG; }
  if (int rc = check_multi(c, B, K, "hmpc_solve_batch_multi")) return rc;
  if (B == 0) return HMPC_OK;
  if (mask && std::all_of(mask, mask + B, [](unsigned char m) { return m == 0; })) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  const size_t nw = (size_t)12 * c->horizon, R = (size_t)B * K, mb = (size_t)c->max_batch;
  const unsigned char* m = nullptr;
  if (mask) {
    memcpy(c->h_mask, mask, (size_t)B);  // pinned: the selection kernel and the cost kernel read it mapped
    m = c->h_mask;
  }
  auto listed = [&](int i) { return !mask || mask[i] != 0; };
  const bool in_place = c->pinned(in, (size_t)B * sizeof(update_data_t)) && c->pinned(traj, R * nw * sizeof(float)) &&
                        c->pinned(wrench_out, R * nw * sizeof(double)) && c->pinned(status, R * sizeof(int)) &&
                        (!cost_out || c->pinned(cost_out, R * sizeof(double)));
  g_multi_in_place = in_place ? 1 : 0;
  const update_data_t* rows = in;
  const float* tr = traj;
  double* w = wrench_out;
  int* st = status;
  double* cost = cost_out;
  if (!in_place) {  // [max_batch rows | max_batch x 12N traj floats | ... wrench doubles | status ints | cost doubles]
    if (!c->h_multi)
      CK(cudaMallocHost(&c->h_multi, mb * (sizeof(update_data_t) + nw * (sizeof(float) + sizeof(double)) + sizeof(int) + sizeof(double))));
    update_data_t* hr = reinterpret_cast<update_data_t*>(c->h_multi);
    float* ht = reinterpret_cast<float*>(hr + mb);
    double* hw = reinterpret_cast<double*>(ht + mb * nw);
    double* hc = hw + mb * nw;
    int* hs = reinterpret_cast<int*>(hc + mb);
    for (int i = 0; i < B; i++)
      if (listed(i)) {
        hr[i] = in[i];
        memcpy(ht + (size_t)i * K * nw, traj + (size_t)i * K * nw, K * nw * sizeof(float));
      }
    rows = hr, tr = ht, w = hw, st = hs, cost = cost_out ? hc : nullptr;
  }
  hmpc::SolveIO io;
  io.raw = rows;
  io.batch = B;
  io.wrench64 = w;
  io.status = st;
  io.mask = m;
  const hmpc::MultiIO mq = multi_io(c, tr, K);
  if (int rc = enqueue_solve(c, io, c->stream, &mq)) return rc;
  if (cost)
    if (int rc = launch_multi_cost(c, rows, hmpc::update_rows(), B, K, m, tr, w, cost, c->stream)) return rc;
  CK(cudaStreamSynchronize(c->stream));
  int rc = HMPC_OK;
  for (int i = 0; i < B; i++) {
    if (!listed(i)) continue;
    const size_t r0 = (size_t)i * K;
    if (!in_place) {
      memcpy(wrench_out + r0 * nw, w + r0 * nw, K * nw * sizeof(double));
      memcpy(status + r0, st + r0, K * sizeof(int));
      if (cost_out) memcpy(cost_out + r0, cost + r0, K * sizeof(double));
    }
    for (int k = 0; k < K; k++)
      if (HMPC_STATUS_CODE(status[r0 + k]) != 0) rc = HMPC_ERR_NOT_CONVERGED;
  }
  if (rc) g_err = "hmpc_solve_batch_multi: at least one candidate did not reach a KKT point (see status[])";
  return rc;
}

// ---------------------------------------------------------------------------------------------------
// candidate commands per robot, from its state (hmpc_chain.h: PrepareTrajArgs)
// ---------------------------------------------------------------------------------------------------
static_assert(sizeof(hmpc_command_t) == 7 * 8 && offsetof(hmpc_state_t, state_des) == 32 * 8 &&
                  offsetof(hmpc_state_t, world_position_desired) == 37 * 8 && offsetof(hmpc_command_t, world_position_desired) == 5 * 8,
              "hmpc_command_t is the state's bytes [256, 312) (hmpc_prepare_traj_kernel)");

// The chain of a multi-command states call on `io` (states, records, outputs, mask set) with K commands `cmd` and trajectory
// buffer `traj`: preparation, classes, cost, pick.  T: the wrench's element type (float: io.wrench, double: io.wrench64).
template <typename T>
static int enqueue_states_multi(hmpc_ctx* c, const hmpc::SolveIO& io, int K, const hmpc_command_t* cmd, float* traj, double* cost,
                                int* best, float* tau, cudaStream_t st)
{
  hmpc::MultiIO mq = multi_io(c, traj, K);
  mq.cmd = reinterpret_cast<const double*>(cmd);
  if (int rc = enqueue_solve(c, io, st, &mq)) return rc;
  const T* w;
  if constexpr (sizeof(T) == 4) w = io.wrench; else w = io.wrench64;
  if (int rc = launch_multi_cost(c, io.records, hmpc::packed_rows(c->horizon), io.batch, K, io.mask, traj, w, cost, st)) return rc;
  return launch_pick(c, const_cast<void*>(io.records), io.batch, K, io.mask, traj, w, io.status, cost, best, tau, st);
}

HMPC_EXTERNC int hmpc_solve_states_device_multi(hmpc_ctx* c, const hmpc_state_t* d_states, int B, int K, const hmpc_command_t* d_cmd,
                                                const unsigned char* d_mask, double dtMPC, void* d_records, float* d_traj,
                                                float* d_wrench, int* d_status, double* d_cost, int* d_best, float* d_tau,
                                                void* stream)
{
  if (!c || !d_states || !d_cmd || !d_records || !d_traj || !d_wrench || !d_status || !d_cost || !d_best) {
    g_err = "hmpc_solve_states_device_multi: null argument";
    return HMPC_ERR_ARG;
  }
  if (int rc = check_multi(c, B, K, "hmpc_solve_states_device_multi")) return rc;
  if (B == 0) return HMPC_OK;
  if (int rc = check_device_records(c, d_records, B, "hmpc_solve_states_device_multi")) return rc;
  hmpc::SolveIO io = device_call(c, d_records, B, d_wrench, d_status, nullptr, false);
  io.mask = d_mask;
  io.states = d_states;
  io.dt_mpc = dtMPC;
  return enqueue_states_multi<float>(c, io, K, d_cmd, d_traj, d_cost, d_best, d_tau, static_cast<cudaStream_t>(stream));
}

namespace { int g_states_multi_in_place = -1; }
HMPC_EXTERNC int hmpc_debug_last_states_multi_in_place(void) { return g_states_multi_in_place; }

// The chain of hmpc_solve_states_device_multi on the context's records and trajectory buffer, with double wrenches: on the
// caller's arrays when they are pinned (the kernels read the states and commands and store the results where they lie),
// else on copies of the listed robots' rows in h_smulti, which the kernels read and write mapped.  Torques go through the
// pinned result staging (h_out) as float rows and are widened here, as in the other host calls.
HMPC_EXTERNC int hmpc_solve_batch_states_multi(hmpc_ctx* c, const hmpc_state_t* in, int B, int K, const hmpc_command_t* cmd,
                                               const unsigned char* mask, double dtMPC, double* wrench_out, int* status,
                                               double* cost_out, int* best, double* tau_out)
{
  if (!c || !in || !cmd || !wrench_out || !status || !cost_out || !best) {
    g_err = "hmpc_solve_batch_states_multi: null argument";
    return HMPC_ERR_ARG;
  }
  if (int rc = check_multi(c, B, K, "hmpc_solve_batch_states_multi")) return rc;
  if (B == 0) return HMPC_OK;
  if (mask && std::all_of(mask, mask + B, [](unsigned char m) { return m == 0; })) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  const size_t nw = (size_t)12 * c->horizon, R = (size_t)B * K, mb = (size_t)c->max_batch;
  if (!c->d_smtraj) CK(cudaMalloc(&c->d_smtraj, mb * nw * sizeof(float)));
  const unsigned char* m = nullptr;
  if (mask) {
    memcpy(c->h_mask, mask, (size_t)B);  // pinned: the selection kernel, the cost and the pick kernel read it mapped
    m = c->h_mask;
  }
  auto listed = [&](int i) { return !mask || mask[i] != 0; };
  const bool in_place = c->pinned(in, (size_t)B * sizeof(hmpc_state_t)) && c->pinned(cmd, R * sizeof(hmpc_command_t)) &&
                        c->pinned(wrench_out, R * nw * sizeof(double)) && c->pinned(status, R * sizeof(int)) &&
                        c->pinned(cost_out, R * sizeof(double)) && c->pinned(best, (size_t)B * sizeof(int));
  g_states_multi_in_place = in_place ? 1 : 0;
  const hmpc_state_t* states = in;
  const hmpc_command_t* cm = cmd;
  double* w = wrench_out;
  int* st = status;
  double* cost = cost_out;
  int* bst = best;
  if (!in_place) {  // [max_batch states | max_batch commands | max_batch x 12N wrench doubles | cost doubles | status ints | best ints]
    if (!c->h_smulti)
      CK(cudaMallocHost(&c->h_smulti, mb * (sizeof(hmpc_state_t) + sizeof(hmpc_command_t) + nw * sizeof(double) + sizeof(double) +
                                            2 * sizeof(int))));
    hmpc_state_t* hs = reinterpret_cast<hmpc_state_t*>(c->h_smulti);
    hmpc_command_t* hc = reinterpret_cast<hmpc_command_t*>(hs + mb);
    double* hw = reinterpret_cast<double*>(hc + mb);
    double* hcost = hw + mb * nw;
    int* hst = reinterpret_cast<int*>(hcost + mb);
    for (int i = 0; i < B; i++)
      if (listed(i)) {
        hs[i] = in[i];
        memcpy(hc + (size_t)i * K, cmd + (size_t)i * K, K * sizeof(hmpc_command_t));
      }
    states = hs, cm = hc, w = hw, st = hst, cost = hcost, bst = hst + mb;
  }
  float* tau = tau_out ? c->rows(c->h_out, 0, c->max_batch).tau : nullptr;  // pinned, written mapped
  hmpc::SolveIO io;
  io.states = states;
  io.dt_mpc = dtMPC;
  io.records = c->d_rec;
  io.batch = B;
  io.wrench64 = w;
  io.status = st;
  io.mask = m;
  if (int rc = enqueue_states_multi<double>(c, io, K, cm, c->d_smtraj, cost, bst, tau, c->stream)) return rc;
  CK(cudaStreamSynchronize(c->stream));
  int rc = HMPC_OK;
  for (int i = 0; i < B; i++) {
    if (!listed(i)) continue;
    const size_t r0 = (size_t)i * K;
    if (!in_place) {
      memcpy(wrench_out + r0 * nw, w + r0 * nw, K * nw * sizeof(double));
      memcpy(status + r0, st + r0, K * sizeof(int));
      memcpy(cost_out + r0, cost + r0, K * sizeof(double));
      best[i] = bst[i];
    }
    if (tau_out)
      for (int j = 0; j < 10; j++) tau_out[(size_t)i * 10 + j] = (double)tau[(size_t)i * 10 + j];
    if (best[i] < 0) rc = HMPC_ERR_NOT_CONVERGED;
  }
  if (rc) g_err = "hmpc_solve_batch_states_multi: no candidate of at least one robot reached a KKT point (see best[], status[])";
  return rc;
}

HMPC_EXTERNC int hmpc_pin_host_buffer(hmpc_ctx* c, void* ptr, size_t bytes)
{
  if (!c || !ptr || bytes == 0) { g_err = "hmpc_pin_host_buffer: bad argument"; return HMPC_ERR_ARG; }
  if (c->pinned(ptr, bytes)) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  // registration is page-granular and two small caller arrays may share a page: register only the page runs of
  // [ptr, ptr+bytes) that no earlier pin covers
  const uintptr_t PG = (uintptr_t)(sysconf(_SC_PAGESIZE) > 0 ? sysconf(_SC_PAGESIZE) : 4096);  // 64 KiB on some aarch64 hosts
  const uintptr_t lo = reinterpret_cast<uintptr_t>(ptr) & ~(PG - 1);
  const uintptr_t hi = (reinterpret_cast<uintptr_t>(ptr) + bytes + PG - 1) & ~(PG - 1);
  auto covered = [&](uintptr_t pg) {
    for (const hmpc_ctx::Run& r : c->runs)
      if (pg >= r.lo && pg < r.hi) return true;
    return false;
  };
  for (uintptr_t pg = lo; pg < hi;) {
    if (covered(pg)) { pg += PG; continue; }
    uintptr_t end = pg + PG;
    while (end < hi && !covered(end)) end += PG;
    void* base = reinterpret_cast<void*>(pg);
    {
      cudaError_t re = cudaHostRegister(base, end - pg, cudaHostRegisterMapped | cudaHostRegisterPortable);
      if (re == cudaErrorHostMemoryAlreadyRegistered) cudaGetLastError();  // registered by somebody else: usable as it is
      else if (cuda_fail(re, "cudaHostRegister")) return HMPC_ERR_CUDA;
    }
    void* dptr = nullptr;
    cudaError_t e = cudaHostGetDevicePointer(&dptr, base, 0);
    if (e != cudaSuccess || dptr != base) {  // the in-place mode hands host addresses to the kernels
      cudaHostUnregister(base);
      g_err = "hmpc_pin_host_buffer: this device cannot address registered host memory through the host pointer";
      return HMPC_ERR_CUDA;
    }
    c->runs.push_back({pg, end});
    pg = end;
  }
  c->pins.push_back({static_cast<char*>(ptr), bytes});
  return HMPC_OK;
}

HMPC_EXTERNC int hmpc_unpin_host_buffer(hmpc_ctx* c, void* ptr)
{
  if (!c || !ptr) { g_err = "hmpc_unpin_host_buffer: bad argument"; return HMPC_ERR_ARG; }
  size_t idx = c->pins.size();
  for (size_t i = 0; i < c->pins.size(); i++)
    if (c->pins[i].base == static_cast<char*>(ptr)) idx = i;
  if (idx == c->pins.size()) { g_err = "hmpc_unpin_host_buffer: pointer was not pinned through this context"; return HMPC_ERR_ARG; }
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < 3; i++) CK(cudaStreamSynchronize(c->xstream[i]));
  c->pins.erase(c->pins.begin() + idx);
  // release the page runs no remaining pin touches
  for (size_t r = 0; r < c->runs.size();) {
    bool used = false;
    for (const hmpc_ctx::Pin& p : c->pins) {
      const uintptr_t a = reinterpret_cast<uintptr_t>(p.base), b = a + p.bytes;
      used |= (a < c->runs[r].hi && b > c->runs[r].lo);
    }
    if (used) { r++; continue; }
    CK(cudaHostUnregister(reinterpret_cast<void*>(c->runs[r].lo)));
    c->runs.erase(c->runs.begin() + r);
  }
  return HMPC_OK;
}

static_assert(sizeof(hmpc_rollout_t) == 80 && offsetof(hmpc_rollout_t, gait_offset) == 48, "hmpc_rollout_t layout (hmpc_advance_kernel)");

HMPC_EXTERNC int hmpc_rollout_device(hmpc_ctx* c, hmpc_state_t* d_states, hmpc_rollout_t* d_loop, int B, int ticks,
                                     double dtMPC, float* d_wrench_log, void* d_record_log, void* stream)
{
  if (!c || !d_states || !d_loop || B < 0 || B > c->max_batch || ticks < 1) {
    g_err = "hmpc_rollout_device: bad argument (null pointer, batch > capacity or ticks < 1)";
    return HMPC_ERR_ARG;
  }
  if (B == 0) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const ResultRows scratch = c->rows(c->d_out, 0, c->max_batch);  // the context's own result area is the loop's scratch
  for (int t = 0; t < ticks; t++) {
    int rc = hmpc_prepare_device(c, d_states, B, dtMPC, c->d_rec, st);
    if (rc != HMPC_OK) return rc;
    if (d_record_log)
      CK(cudaMemcpyAsync(static_cast<unsigned char*>(d_record_log) + (size_t)t * B * c->rec_stride, c->d_rec,
                         (size_t)B * c->rec_stride, cudaMemcpyDeviceToDevice, st));
    rc = enqueue_solve(c, device_call(c, c->d_rec, B, scratch.wrench, scratch.status, nullptr, true), st);
    if (rc != HMPC_OK) return rc;
    hmpc::hmpc_advance_kernel<<<(B + 63) / 64, 64, 0, st>>>(reinterpret_cast<unsigned char*>(d_states),
                                                            reinterpret_cast<unsigned char*>(d_loop), B, c->horizon, dtMPC,
                                                            scratch.wrench, scratch.status,
                                                            d_wrench_log ? d_wrench_log + (size_t)t * B * 12 : nullptr);
    CK(cudaGetLastError());
  }
  return HMPC_OK;
}

HMPC_EXTERNC int hmpc_reset_warm_start(hmpc_ctx* c, void* stream)
{
  if (!c) { g_err = "hmpc_reset_warm_start: null context"; return HMPC_ERR_ARG; }
  CK(cudaSetDevice(c->device));
  CK(cudaMemsetAsync(c->d_ws, 0, (size_t)c->max_batch * hmpc::WS_STATE_INTS * sizeof(int), static_cast<cudaStream_t>(stream)));
  return HMPC_OK;
}

static_assert(sizeof(hmpc_swing_t) == 72 && offsetof(hmpc_swing_t, first_swing) == 64, "hmpc_swing_t layout (hmpc_swing_kernel)");
static_assert(sizeof(hmpc_swing_cmd_t) == 232 && offsetof(hmpc_swing_cmd_t, swing) == 224, "hmpc_swing_cmd_t layout (hmpc_swing_kernel)");

HMPC_EXTERNC int hmpc_swing_device(hmpc_ctx* c, const hmpc_state_t* d_states, const hmpc_rollout_t* d_loop, const double* d_phase,
                                   hmpc_swing_t* d_swing, int B, double dt, double dtSwing, hmpc_swing_cmd_t* d_cmd, void* stream)
{
  if (!c || !d_states || !d_loop || !d_phase || !d_swing || !d_cmd || B < 0) { g_err = "hmpc_swing_device: bad argument"; return HMPC_ERR_ARG; }
  if (B == 0) return HMPC_OK;
  CK(cudaSetDevice(c->device));
  hmpc::hmpc_swing_kernel<<<(B + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const unsigned char*>(d_states), reinterpret_cast<const unsigned char*>(d_loop), d_phase,
      reinterpret_cast<unsigned char*>(d_swing), B, c->horizon, dt, dtSwing, reinterpret_cast<unsigned char*>(d_cmd));
  CK(cudaGetLastError());
  return HMPC_OK;
}

// ---------------------------------------------------------------------------------------------------
// host-buffer calls (hmpc_solve_batch and its variants): the caller's arrays are in host memory
// ---------------------------------------------------------------------------------------------------
namespace {
// What one host-buffer call asks for.  Unused pointers stay null.
struct HostCall {
  HostCall(const update_data_t* in, int B, double* w, double* t, int* st) : records(in), batch(B), wrench(w), tau(t), status(st) {}
  HostCall(const hmpc_state_t* in, int B, double dt, double* w, double* t, int* st)
      : states(in), dt_mpc(dt), batch(B), wrench(w), tau(t), status(st) {}
  HostCall& warm_start(const int* s, const unsigned char* m = nullptr) { warm = true, shift = s, mask = m; return *this; }
  const update_data_t* records = nullptr;  // the reference's records in, or
  const hmpc_state_t* states = nullptr;    // robot states, prepared into records on the device with the MPC step dt_mpc
  double dt_mpc = 0.0;
  int batch = 0;
  double *wrench = nullptr, *tau = nullptr;  // [batch][12N], [batch][10] joint torques
  int* status = nullptr;                     // [batch]
  bool warm = false;                         // propose each robot's working set of its last warm call, moved shift[i] steps
  const int* shift = nullptr;                // (null: one step each)
  const unsigned char* mask = nullptr;       // [batch]: only robots with mask[i] != 0 are solved and have their rows written
  float* shard_wrench = nullptr;             // the sharded calls in place: the kernels also store float wrenches here,
  const float* shard_prev = nullptr;         // (masked) the carry kernel fills the unlisted rows from this buffer,
  cudaEvent_t shard_solved = nullptr;        // and this event is recorded behind them
  bool listed(int i) const { return !mask || mask[i] != 0; }
};

// The mode of a host-buffer call (DESIGN.md §3): in place when the records (or states), the wrenches and the status words
// (if asked for) lie in buffers registered with hmpc_pin_host_buffer, else staged in chunks (solve_batch_impl).
constexpr int ZERO_COPY_MAX = 1536;  // above it, packing that overlaps the kernels wins

bool runs_in_place(const hmpc_ctx* c, const HostCall& h)
{
  const size_t B = (size_t)h.batch;
  const bool in = h.records ? c->pinned(h.records, B * sizeof(update_data_t)) : c->pinned(h.states, B * sizeof(hmpc_state_t));
  return in && c->pinned(h.wrench, B * 12 * c->horizon * sizeof(double)) && (!h.status || c->pinned(h.status, B * sizeof(int)));
}

// HMPC_TRACE: microseconds from the start of a staged call to each point, one line on stderr per call
struct Trace {
  double t[4 * NCHUNK + 2];
  int n = 0;
  void mark()
  {
    static const bool on = getenv("HMPC_TRACE") != nullptr;
    timespec ts;
    if (on && clock_gettime(CLOCK_MONOTONIC, &ts) == 0) t[n++] = ts.tv_sec * 1e6 + ts.tv_nsec * 1e-3;
  }
  void end(int B)
  {
    mark();
    if (n == 0) return;  // (HMPC_TRACE unset)
    fprintf(stderr, "[hmpc trace] B=%d us since entry:", B);
    for (int i = 1; i < n; i++) fprintf(stderr, " %.0f", t[i] - t[0]);
    fprintf(stderr, "  (per chunk: packed, enqueued; then per chunk: synced; end)\n");
  }
};

// HMPC_OK when every listed robot of rows [b0, b0 + nb) reached a KKT point (st: their status words)
int check_converged(const HostCall& h, const int* st, int b0, int nb)
{
  for (int i = 0; i < nb; i++)
    if (h.listed(b0 + i) && HMPC_STATUS_CODE(st[i]) != 0) {
      g_err = "hmpc_solve_batch: at least one instance did not reach a KKT point (see status[])";
      return HMPC_ERR_NOT_CONVERGED;
    }
  return HMPC_OK;
}

// The device-resident chain on the caller's records (states: prepared into the context's d_rec first), double results
// stored into the caller's arrays: the call is launches and one synchronize.
int solve_in_place(hmpc_ctx* c, const HostCall& h, const int* shifts)
{
  const ResultRows scratch = c->rows(c->h_out, 0, c->max_batch);
  int* st = h.status ? h.status : scratch.status;
  float* tau = h.tau ? scratch.tau : nullptr;
  if (h.mask) memcpy(c->h_mask, h.mask, (size_t)h.batch);  // pinned: the selection kernel reads it mapped
  hmpc::SolveIO io = device_call(c, h.states ? c->d_rec : nullptr, h.batch, h.shard_wrench, st, tau, h.warm);
  io.raw = h.records, io.states = h.states, io.dt_mpc = h.dt_mpc;
  io.wrench64 = h.wrench, io.shifts = shifts, io.mask = h.mask ? c->h_mask : nullptr;
  if (int rc = enqueue_solve(c, io, c->stream)) return rc;
  if (h.shard_prev)
    if (int rc = launch_carry(c->h_mask, h.batch, c->horizon, h.shard_prev, h.shard_wrench, c->stream)) return rc;
  if (h.shard_solved) CK(cudaEventRecord(h.shard_solved, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  if (h.tau)
    for (int i = 0; i < h.batch; i++)
      if (h.listed(i))
        for (int j = 0; j < 10; j++) h.tau[(size_t)i * 10 + j] = (double)tau[(size_t)i * 10 + j];
  return check_converged(h, st, 0, h.batch);
}

// fn(r0, r1) over rows [b0, b0 + nb), split among the helper threads for large chunks
template <typename F>
void over_rows(const hmpc_ctx* c, int b0, int nb, F fn)
{
  if (!c->pool || nb < 128) return fn(b0, b0 + nb);
  c->pool->parallel([&](int part, int nparts) { fn(b0 + (int)((long long)nb * part / nparts), b0 + (int)((long long)nb * (part + 1) / nparts)); });
}

// Packs the chunk's records (or stages its states and prepares them on the device), copies them over (copy pipeline),
// classifies on the host, launches the classes over the host-built lists and copies the results back (copy pipeline).
int stage_chunk(hmpc_ctx* c, const HostCall& h, bool zc, Chunk& ch, const int* shifts, Trace& tr)
{
  const int b0 = ch.b0, nb = ch.nb;
  const size_t rs = (size_t)c->rec_stride, sb = sizeof(hmpc_state_t);
  if (h.states) {  // (in a masked call the unlisted robots' records are built too, and not read)
    memcpy(c->h_states + b0 * sb, h.states + b0, nb * sb);
    tr.mark();
    if (!zc) CK(cudaMemcpyAsync(c->d_states + b0 * sb, c->h_states + b0 * sb, nb * sb, cudaMemcpyHostToDevice, ch.st));
    if (int rc = hmpc_prepare_device(c, reinterpret_cast<const hmpc_state_t*>((zc ? c->h_states : c->d_states) + b0 * sb), nb,
                                     h.dt_mpc, c->d_rec + b0 * rs, ch.st))
      return rc;
  } else {  // every robot of the chunk, or only the listed ones (the kernels read no other record)
    over_rows(c, b0, nb, [&](int r0, int r1) {
      if (!h.mask) hmpc_pack_records(h.records + r0, r1 - r0, c->horizon, c->h_rec + r0 * rs);
      else
        for (int i = r0; i < r1; i++)
          if (h.mask[i]) hmpc_pack_records(h.records + i, 1, c->horizon, c->h_rec + i * rs);
    });
    tr.mark();
    if (!zc) CK(cudaMemcpyAsync(c->d_rec + b0 * rs, c->h_rec + b0 * rs, nb * rs, cudaMemcpyHostToDevice, ch.st));
  }
  const ResultRows out = c->rows(zc ? c->h_out : c->d_out, b0, nb, h.tau != nullptr);
  ch.io = device_call(c, ((zc && !h.states) ? c->h_rec : c->d_rec) + b0 * rs, nb, out.wrench, out.status, out.tau, h.warm);
  if (ch.io.ws) ch.io.ws += (size_t)b0 * hmpc::WS_STATE_INTS;
  if (shifts && !zc) CK(cudaMemcpyAsync(c->d_shift + b0, shifts + b0, (size_t)nb * sizeof(int), cudaMemcpyHostToDevice, ch.st));
  if (shifts) ch.io.shifts = (zc ? shifts : c->d_shift) + b0;  // zero-copy: mapped, like the records and lists of this mode
  hmpc::classify_host(c->horizon, c->cfg.f_max, c->cls[0].nb_hi, h.states ? h.states[b0].gait : h.records[b0].gait,
                      h.states ? sizeof(hmpc_state_t) : sizeof(update_data_t), nb, ch.lists, c->max_batch, h.mask ? h.mask + b0 : nullptr);
  if (int rc = enqueue_solve_hostlists(c, ch, zc)) return rc;
  if (!zc) CK(cudaMemcpyAsync(c->rows(c->h_out, b0, nb).wrench, out.wrench, out.bytes, cudaMemcpyDeviceToHost, ch.st));
  tr.mark();
  return HMPC_OK;
}

// Rows [b0, b0 + nb) of the staged results `r` into the caller's arrays, the listed rows only: wrenches and torques
// widened to double, status words copied.
void widen_rows(const hmpc_ctx* c, const HostCall& h, const ResultRows& r, int b0, int nb)
{
  const size_t nw = (size_t)12 * c->horizon;
  over_rows(c, b0, nb, [&](int r0, int r1) {
    for (int row = r0; row < r1; row++) {
      if (!h.listed(row)) continue;
      const size_t i = (size_t)(row - b0);  // the row in the chunk
      double* w = h.wrench + (size_t)row * nw;
      const float* src = r.wrench + i * nw;
      for (size_t e = 0; e < nw; e++) w[e] = (double)src[e];
      if (h.tau)
        for (int j = 0; j < 10; j++) h.tau[(size_t)row * 10 + j] = (double)r.tau[i * 10 + j];
      if (h.status) h.status[row] = r.status[i];
    }
  });
}

// Waits for the chunk, solves again what its host-list launches left (working-set overflow: enqueue_overflow_retry;
// instances beyond the conditioning limit while refinement is on: enqueue_refine_retry) and widens its results.
int finish_chunk(hmpc_ctx* c, const HostCall& h, bool zc, Chunk& ch, Trace& tr)
{
  CK(cudaStreamSynchronize(ch.st));
  tr.mark();
  const ResultRows r = c->rows(c->h_out, ch.b0, ch.nb, h.tau != nullptr);
  bool overflow = false, not_spd = false;
  for (int i = 0; i < ch.nb; i++) {
    overflow |= h.listed(ch.b0 + i) && HMPC_STATUS_CODE(r.status[i]) == hmpc::ST_WS_CAP;
    not_spd |= h.listed(ch.b0 + i) && HMPC_STATUS_CODE(r.status[i]) == hmpc::ST_NOT_SPD;
  }
  const bool refine = c->cfg.refine && not_spd;  // instances handed to the refinement class (on its device-side list)
  if (overflow || refine) {
    int rc = overflow ? enqueue_overflow_retry(c, ch, r.status, h.mask ? h.mask + ch.b0 : nullptr) : HMPC_OK;
    if (rc == HMPC_OK && refine) rc = enqueue_refine_retry(c, ch);
    if (rc != HMPC_OK) return rc;
    if (!zc) CK(cudaMemcpyAsync(r.wrench, ch.io.wrench, r.bytes, cudaMemcpyDeviceToHost, ch.st));
    CK(cudaStreamSynchronize(ch.st));
  }
  widen_rows(c, h, r, ch.b0, ch.nb);
  return HMPC_OK;
}

// Every host-buffer call.  With a mask the context's staging rows of unlisted robots keep stale results, which nothing reads.
int solve_batch_impl(hmpc_ctx* c, const HostCall& h)
{
  const int B = h.batch;
  if (!c || (!h.records && !h.states) || !h.wrench || B < 0 || B > c->max_batch) {
    g_err = "hmpc_solve_batch: bad argument (null pointer or batch > capacity)";
    return HMPC_ERR_ARG;
  }
  if (B == 0) return HMPC_OK;
  if (h.mask && std::all_of(h.mask, h.mask + B, [](unsigned char m) { return m == 0; })) return HMPC_OK;
  if (g_fail_next_solves > 0) {
    g_fail_next_solves--;
    g_err = "injected failure (hmpc_debug_fail_next_solves)";
    return HMPC_ERR_CUDA;
  }
  CK(cudaSetDevice(c->device));
  const int* shifts = nullptr;  // warm start (device_call): per-robot shifts from the pinned copy of h.shift
  if (h.warm && c->warm_start && h.shift) {
    memcpy(c->h_shift, h.shift, (size_t)B * sizeof(int));
    shifts = c->h_shift;
  }
  if (runs_in_place(c, h)) return solve_in_place(c, h, shifts);
  const bool zc = B <= ZERO_COPY_MAX;                  // zero-copy staging, in one chunk
  const int nch = zc ? 1 : (c->pool ? 2 : NCHUNK);     // else the copy pipeline (no chunk is empty: B > ZERO_COPY_MAX)
  const cudaStream_t sts[NCHUNK] = {c->stream, c->xstream[0], c->xstream[1], c->xstream[2]};
  Chunk ch[NCHUNK];
  Trace tr;
  tr.mark();
  for (int k = 0; k < nch; k++) {
    const int b0 = (int)((long long)B * k / nch), nb = (int)((long long)B * (k + 1) / nch) - b0;
    const size_t li = (size_t)k * hmpc::host_lists_ints(c->max_batch);
    int* ref = c->cfg.refine ? c->d_ref + (size_t)k * (1 + (size_t)c->max_batch) : nullptr;
    ch[k] = Chunk{b0, nb, sts[k], {}, c->h_cls + li, c->d_lists + li, ref};
    if (int rc = stage_chunk(c, h, zc, ch[k], shifts, tr)) return rc;
  }
  int rc = HMPC_OK;
  for (int k = 0; k < nch; k++) {
    if (int e = finish_chunk(c, h, zc, ch[k], tr)) return e;
    if (check_converged(h, c->rows(c->h_out, ch[k].b0, ch[k].nb).status, ch[k].b0, ch[k].nb)) rc = HMPC_ERR_NOT_CONVERGED;
  }
  tr.end(B);
  return rc;
}
}  // namespace

HMPC_EXTERNC int hmpc_solve_batch(hmpc_ctx* c, const update_data_t* in, int B, double* wrench_out, int* status)
{
  return hmpc_solve_batch_ex(c, in, B, wrench_out, nullptr, status);
}

HMPC_EXTERNC int hmpc_solve_batch_ex(hmpc_ctx* c, const update_data_t* in, int B, double* wrench_out, double* tau_out,
                                     int* status)
{
  return solve_batch_impl(c, HostCall(in, B, wrench_out, tau_out, status));
}

HMPC_EXTERNC int hmpc_solve_batch_warm(hmpc_ctx* c, const update_data_t* in, int B, double* wrench_out, double* tau_out,
                                       int* status, const int* shift)
{
  if (!in) { g_err = "hmpc_solve_batch_warm: bad argument (null records)"; return HMPC_ERR_ARG; }
  return solve_batch_impl(c, HostCall(in, B, wrench_out, tau_out, status).warm_start(shift));
}

HMPC_EXTERNC int hmpc_solve_batch_masked(hmpc_ctx* c, const update_data_t* in, int B, const unsigned char* mask, double* wrench_out,
                                         double* tau_out, int* status, const int* shift)
{
  if (!in || !mask) { g_err = "hmpc_solve_batch_masked: bad argument (null records or mask)"; return HMPC_ERR_ARG; }
  return solve_batch_impl(c, HostCall(in, B, wrench_out, tau_out, status).warm_start(shift, mask));
}

HMPC_EXTERNC int hmpc_solve_batch_states(hmpc_ctx* c, const hmpc_state_t* in, int B, double dtMPC, double* wrench_out,
                                         double* tau_out, int* status)
{
  return solve_batch_impl(c, HostCall(in, B, dtMPC, wrench_out, tau_out, status));
}

HMPC_EXTERNC int hmpc_solve_batch_states_warm(hmpc_ctx* c, const hmpc_state_t* in, int B, double dtMPC, double* wrench_out,
                                              double* tau_out, int* status, const int* shift)
{
  if (!in) { g_err = "hmpc_solve_batch_states_warm: bad argument (null states)"; return HMPC_ERR_ARG; }
  return solve_batch_impl(c, HostCall(in, B, dtMPC, wrench_out, tau_out, status).warm_start(shift));
}

HMPC_EXTERNC int hmpc_solve_batch_states_masked(hmpc_ctx* c, const hmpc_state_t* in, int B, const unsigned char* mask,
                                                double dtMPC, double* wrench_out, double* tau_out, int* status, const int* shift)
{
  if (!in || !mask) { g_err = "hmpc_solve_batch_states_masked: bad argument (null states or mask)"; return HMPC_ERR_ARG; }
  return solve_batch_impl(c, HostCall(in, B, dtMPC, wrench_out, tau_out, status).warm_start(shift, mask));
}

namespace {
// The sharded calls: the host-buffer call `h` on this rank's slice, then this tick's float rows into shard_buf[par] and,
// with d_all, the gather of that buffer.  The rows of the robots `h` lists (all without a mask) are this call's results;
// the carry kernel copies the others from the previous tick's buffer, so every row is the robot's latest.
int solve_sharded(hmpc_ctx* c, HostCall h, float* d_all, const char* who)
{
  if (!c || !c->nccl) { g_err = std::string(who) + ": call hmpc_shard_init first"; return HMPC_ERR_ARG; }
  if (h.batch < 1 || h.batch > c->max_batch) { g_err = std::string(who) + ": every rank needs 1 <= B_local <= capacity"; return HMPC_ERR_ARG; }
  CK(cudaSetDevice(c->device));
  const int B = h.batch, par = (int)(c->shard_tick & 1u);
  const size_t nw = (size_t)12 * c->horizon;
  float* cur = c->shard_buf[par];
  const float* prev = c->shard_buf[par ^ 1];
  const bool none = h.mask && std::all_of(h.mask, h.mask + B, [](unsigned char m) { return m == 0; });  // nothing is solved
  // the gather that last read `cur` (two ticks ago) must be done before this tick overwrites it — a stream-side wait, the
  // host does not block
  CK(cudaStreamWaitEvent(c->stream, c->gathered[par], 0));
  if (runs_in_place(c, h) && !none)  // the kernels store the listed rows, the carry the others, both before `solved`
    h.shard_wrench = cur, h.shard_prev = h.mask ? prev : nullptr, h.shard_solved = c->solved;
  const int rc = solve_batch_impl(c, h);
  if (rc != HMPC_OK && rc != HMPC_ERR_NOT_CONVERGED) return rc;
  if (!h.shard_solved) {
    // staged (or nothing solved): the listed rows' float results from the caller's array, then the carry
    if (!none) {
      std::vector<float> tmp((size_t)B * nw);
      for (int i = 0; i < B; i++)
        if (h.listed(i))
          for (size_t e = 0; e < nw; e++) tmp[i * nw + e] = (float)h.wrench[i * nw + e];
      CK(cudaMemcpyAsync(cur, tmp.data(), tmp.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    }
    if (h.mask) {
      memcpy(c->h_mask, h.mask, (size_t)B);  // pinned: read mapped, like the selection kernel's
      if (int e = launch_carry(c->h_mask, B, c->horizon, prev, cur, c->stream)) return e;
    }
    CK(cudaEventRecord(c->solved, c->stream));
    CK(cudaStreamSynchronize(c->stream));
  }
  c->shard_tick++;
  if (d_all) {
    // the path's ONE collective: every rank's slice of float wrenches to every device, beside the next tick
    CK(cudaStreamWaitEvent(c->gstream, c->solved, 0));
    if (nccl_fail(g_nccl.AllGather(cur, d_all, (size_t)B * nw, /* ncclFloat32 */ 7, c->nccl, c->gstream), "ncclAllGather"))
      return HMPC_ERR_CUDA;
    CK(cudaEventRecord(c->gathered[par], c->gstream));
  }
  return rc;
}
}  // namespace

HMPC_EXTERNC int hmpc_solve_batch_sharded(hmpc_ctx* c, const update_data_t* in_local, int B_local, double* wrench_local,
                                          int* status_local, float* d_all)
{
  return solve_sharded(c, HostCall(in_local, B_local, wrench_local, nullptr, status_local), d_all, "hmpc_solve_batch_sharded");
}

HMPC_EXTERNC int hmpc_solve_batch_sharded_warm(hmpc_ctx* c, const update_data_t* in_local, int B_local,
                                               const unsigned char* mask_local, double* wrench_local, double* tau_local,
                                               int* status_local, const int* shift_local, float* d_all)
{
  if (!in_local) { g_err = "hmpc_solve_batch_sharded_warm: bad argument (null records)"; return HMPC_ERR_ARG; }
  return solve_sharded(c, HostCall(in_local, B_local, wrench_local, tau_local, status_local).warm_start(shift_local, mask_local),
                       d_all, "hmpc_solve_batch_sharded_warm");
}

HMPC_EXTERNC int hmpc_solve_batch_states_sharded_warm(hmpc_ctx* c, const hmpc_state_t* in_local, int B_local,
                                                      const unsigned char* mask_local, double dtMPC, double* wrench_local,
                                                      double* tau_local, int* status_local, const int* shift_local, float* d_all)
{
  if (!in_local) { g_err = "hmpc_solve_batch_states_sharded_warm: bad argument (null states)"; return HMPC_ERR_ARG; }
  return solve_sharded(c, HostCall(in_local, B_local, dtMPC, wrench_local, tau_local, status_local).warm_start(shift_local, mask_local),
                       d_all, "hmpc_solve_batch_states_sharded_warm");
}

// ---------------------------------------------------------------------------------------------------
// Part 1: the reference's boundary on a one-robot context (process-global, single caller thread —
// the same contract as the reference's globals, convexMPC_interface.cpp:13-20)
// ---------------------------------------------------------------------------------------------------
namespace {
hmpc_ctx* g_ctx = nullptr;
// the reference's `update` record, the solution buffer and the status word live in ONE page-aligned block that is
// registered with the context, so the one-robot tick runs in place (no packing / staging copies)
struct RefBlock {
  update_data_t update;                       // zero-initialised, like the reference's static `update`
  double soln[12 * HMPC_MAX_HORIZON];
  int status;
};
RefBlock* g_blk = nullptr;
update_data_t g_update_early;  // update_solver_settings may be called before setup_problem
update_data_t& ref_update() { return g_blk ? g_blk->update : g_update_early; }
int g_soln_len = 0;
int g_has_solved = 0;
int g_ref_rc = HMPC_OK;       // result of the last update_problem_data (hmpc_reference_last_rc)
bool g_ref_failing = false;   // inside an episode of failing ticks (the message is printed once per episode)
bool g_ref_warm = false;      // hmpc_reference_set_warm_start: update_problem_data proposes the previous tick's working set
bool g_ref_refine = false;    // hmpc_reference_set_refinement: the one-robot context solves beyond the conditioning limit

[[noreturn]] void die(const char* where)
{
  fprintf(stderr, "[hector_mpc_b200] %s: %s\n", where, hmpc_last_error());
  abort();
}
}  // namespace

HMPC_EXTERNC void setup_problem(double dt, int horizon, double mu, double f_max)
{
  if (horizon > 19) {  // SolverMPC.cpp:140-143 throws here; a C boundary must not leak exceptions
    g_err = "horizon is too long!";
    die("setup_problem");
  }
  if (!g_ctx || g_ctx->horizon != horizon) {
    if (g_ctx) hmpc_destroy(g_ctx);
    g_ctx = hmpc_create(1, horizon, 0);  // refuses horizons above HMPC_MAX_HORIZON
    if (!g_ctx) die("setup_problem");
    hmpc_set_refinement(g_ctx, g_ref_refine ? 1 : 0);
    if (!g_blk) {
      void* mem = nullptr;
      const size_t bytes = (sizeof(RefBlock) + 4095) / 4096 * 4096;
      if (posix_memalign(&mem, 4096, bytes) != 0) { g_err = "out of memory"; die("setup_problem"); }
      memset(mem, 0, bytes);
      g_blk = static_cast<RefBlock*>(mem);
      g_blk->update = g_update_early;
    }
    memset(g_blk->soln, 0, sizeof(g_blk->soln));
    g_soln_len = 12 * horizon;
    // in-place ticks; if registration is not possible the staged path is used (same results)
    if (hmpc_pin_host_buffer(g_ctx, g_blk, (sizeof(RefBlock) + 4095) / 4096 * 4096) != HMPC_OK)
      fprintf(stderr, "[hector_mpc_b200] setup_problem: %s (using staged copies)\n", hmpc_last_error());
  }
  problem_setup s;
  s.dt = (float)dt;
  s.mu = (float)mu;
  s.f_max = (float)f_max;
  s.horizon = horizon;
  // the reference's caller sets the same problem up before every tick; a different QP (dt, f_max) forgets the warm start's
  // working set (a new context — another horizon — starts without one)
  if (s.dt != g_ctx->cfg.dt || s.f_max != g_ctx->cfg.f_max)
    if (hmpc_reset_warm_start(g_ctx, g_ctx->stream) != HMPC_OK) die("setup_problem");
  hmpc_set_problem(g_ctx, &s);
}

HMPC_EXTERNC void hmpc_reference_set_warm_start(int on) { g_ref_warm = on != 0; }

HMPC_EXTERNC void hmpc_reference_set_refinement(int on)
{
  g_ref_refine = on != 0;
  if (g_ctx) hmpc_set_refinement(g_ctx, g_ref_refine ? 1 : 0);
}

HMPC_EXTERNC void update_problem_data(double* p, double* v, double* q, double* w, double* r, double* joint_angles,
                                      double yaw, double* weights, double* state_trajectory, double* Alpha_K,
                                      int* gait)
{
  if (!g_ctx) { g_err = "update_problem_data called before setup_problem"; die("update_problem_data"); }
  const int N = g_ctx->horizon;
  // double -> float narrowing, convexMPC_interface.cpp:87-99
  for (int i = 0; i < 3; i++) { ref_update().p[i] = (float)p[i]; ref_update().v[i] = (float)v[i]; ref_update().w[i] = (float)w[i]; }
  for (int i = 0; i < 4; i++) ref_update().q[i] = (float)q[i];
  for (int i = 0; i < 6; i++) ref_update().r[i] = (float)r[i];
  for (int i = 0; i < 10; i++) ref_update().joint_angles[i] = (float)joint_angles[i];
  ref_update().yaw = (float)yaw;
  for (int i = 0; i < 12; i++) { ref_update().weights[i] = (float)weights[i]; ref_update().Alpha_K[i] = (float)Alpha_K[i]; }
  for (int i = 0; i < 12 * N; i++) ref_update().traj[i] = (float)state_trajectory[i];
  for (int i = 0; i < 2 * N; i++) ref_update().gait[i] = (unsigned char)gait[i];
  int rc = g_ref_warm ? hmpc_solve_batch_warm(g_ctx, &g_blk->update, 1, g_blk->soln, nullptr, &g_blk->status, nullptr)
                      : hmpc_solve_batch(g_ctx, &g_blk->update, 1, g_blk->soln, &g_blk->status);
  g_ref_rc = rc;
  if (rc == HMPC_ERR_NOT_CONVERGED) printf("failed to solve!\n");  // SolverMPC.cpp:714-715 (status word: hmpc_reference_last_status())
  else if (rc != HMPC_OK) {
    // a run-time failure: the controller keeps running on the last wrench and can ask why (hmpc_reference_last_rc)
    const char* ab = getenv("HMPC_REFERENCE_ABORT");
    if (ab && atoi(ab) != 0) die("update_problem_data");
    if (!g_ref_failing)
      fprintf(stderr, "[hector_mpc_b200] update_problem_data: %s — keeping the previous solution (hmpc_reference_last_rc() = %d)\n",
              hmpc_last_error(), rc);
    g_ref_failing = true;
    return;
  }
  g_ref_failing = false;
  g_has_solved = 1;
}

HMPC_EXTERNC double get_solution(int index)
{
  if (!g_has_solved) return 0.f;  // convexMPC_interface.cpp:107
  if (index < 0 || index >= g_soln_len) return 0.0;
  return g_blk->soln[index];
}

HMPC_EXTERNC void update_solver_settings(int max_iter, double rho, double sigma, double solver_alpha, double terminate,
                                         double use_jcqp)
{
  (void)use_jcqp;  // convexMPC_interface.cpp:112-118: stored, not used by the solve
  ref_update().max_iterations = max_iter;
  ref_update().rho = rho;
  ref_update().sigma = sigma;
  ref_update().solver_alpha = solver_alpha;
  ref_update().terminate = terminate;
}

// status word of the last update_problem_data (additive; not part of the reference boundary)
HMPC_EXTERNC int hmpc_reference_last_status(void) { return g_blk ? g_blk->status : 0; }
// result code of the last update_problem_data (additive): see include/hector_mpc_b200.h
HMPC_EXTERNC int hmpc_reference_last_rc(void) { return g_ref_rc; }
