// tests/host_emul/kernel_source_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only), see fake_cuda/cuda_runtime.h.
//
// Includes the product's device header through the fake CUDA prelude and runs, on the host,
//   * the one-thread-per-robot kernels  hmpc_prepare_kernel (row f-1), hmpc_advance_kernel (f-3), hmpc_swing_kernel (f-4)
//     — one call per robot with threadIdx/blockIdx set the way a launch would set them;
//   * the stage-1 device functions of the solve kernel (role_leg / role_state / role_inertia: SRBD linearisation, foot
//     rotations, constraint rows) and the joint-torque epilogue function (leg_torque, f-2).
//   * the selection kernel and the solve kernel itself (all stages), one OS thread per CUDA thread of one CTA at a time,
//     in the launch sequences of hmpc_capi.cu (emul_solve).  The kernel variants, the class shapes, the class-list memory
//     and every launch's arguments come from the library's own hmpc_chain.h.
// so that the CPU suite (tests/test_kernel_source_on_host.py, test_warm_start_calls.py, test_masked_solve.py,
// test_refinement.py) can hold the kernels' SOURCE to the oracle / to the reference's compiled controller without a GPU.
// race_driver.cpp makes the same source a command-line program for ThreadSanitizer.
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

// HMPC_DEVICE_HEADER: hector_simulation_b200/csrc/hmpc_device.cuh after the test's build step (test_kernel_source_on_host.py,
// `_host_buildable`) has made the handful of substitutions a host compiler needs, each asserted to hit exactly once:
//   - the four PTX helper bodies (mbar_init / mbar_expect_tx / mbar_wait / bulk_g2s) -> calls to hmpc_emul_* (cuda_runtime.h)
//   - the `rcp.approx.ftz.f64` seed of fast_rcp -> `1.0 / x` (the Newton steps that follow are kept)
//   - the dynamic shared-memory declaration -> a pointer to the emulated CTA's buffer
//   - the body of dmma884 (mma.sync.m8n8k4.f64) -> hmpc_emul_dmma884, a warp-collective exchange + fused multiply-adds
//   - every other `asm volatile(...)` (fences, griddepcontrol: no arithmetic) -> nothing
// Everything else is the product's source, byte for byte.
#include HMPC_DEVICE_HEADER
#include "../../hector_simulation_b200/csrc/hmpc_chain.h"

thread_local hmpc_emul_dim3 threadIdx, blockIdx, blockDim, gridDim;
thread_local hmpc_emul::Cta* hmpc_emul_cta = nullptr;

namespace hmpc_emul {
unsigned char* cta_smem()
{
  alignas(16) static unsigned char buf[256 * 1024];
  return buf;
}
}  // namespace hmpc_emul

namespace {
// run `fn()` on NT OS threads as the NT CUDA threads of the single CTA of a 1-CTA grid
template <class F>
void run_cta(int NT, F fn)
{
  hmpc_emul::Cta* cta = new hmpc_emul::Cta;
  cta->bar.count = NT;
  for (int w = 0; w < 32; w++) cta->warps[w].bar.count = 32;
  std::vector<std::thread> th;
  th.reserve(NT);
  for (int t = 0; t < NT; t++)
    th.emplace_back([=] {
      threadIdx = {(unsigned)t, 0, 0};
      blockIdx = {0, 0, 0};
      blockDim = {(unsigned)NT, 1, 1};
      gridDim = {1, 1, 1};
      hmpc_emul_cta = cta;
      fn();
      hmpc_emul_cta = nullptr;
    });
  for (auto& x : th) x.join();
  delete cta;
}

// hmpc_capi.cu's launch of class `cls`: its arguments (hmpc::launch_args), and one emulated CTA that walks every instance
// of the class
void run_class(const hmpc::SolverSettings& S, int N, int ncls, int cls, const hmpc::ClassCfg& k, const hmpc::SolveIO& io,
               const hmpc::ChainLists& lists)
{
  const hmpc::KernelArgs ka = hmpc::launch_args(S, N, ncls, cls, k, io, lists);
  switch (k.variant) {
#define HMPC_RUN(ID, NT, MB, NF, CL) \
  case ID: run_cta(NT, [=] { hmpc::hmpc_solve_kernel<NT, MB, NF, CL>(ka); }); return;
    HMPC_VARIANTS(HMPC_RUN)
#undef HMPC_RUN
  }
  hmpc_emul::die("no such kernel variant");
}
void run_select(const unsigned char* mask, int B, int* list, int* count)
{
  run_cta(hmpc::SELECT_THREADS, [=] { hmpc::hmpc_select_kernel<hmpc::SELECT_THREADS>(mask, B, list, count); });
}
// hmpc_create's settings, read per call: the same environment overrides, plus the two tolerances (the tolerance-sweep test)
hmpc::SolverSettings settings(int refine)
{
  hmpc::SolverSettings S;
  if (const char* e = getenv("HMPC_TOL_KKT")) S.tol_kkt = atof(e);
  if (const char* e = getenv("HMPC_TOL_DEP")) S.tol_dep = atof(e);
  if (const char* e = getenv("HMPC_KAPPA_MAX")) S.kappa_max = atof(e);
  if (const char* e = getenv("HMPC_BLOCK_MIN")) S.block_min = atoi(e);
  if (const char* e = getenv("HMPC_BLOCK_ROUNDS")) S.block_rounds = atoi(e);
  S.refine = refine;
  return S;
}
const unsigned kBlock = 128;
inline void set_thread(int i)
{
  blockDim = {kBlock, 1, 1};
  blockIdx = {(unsigned)i / kBlock, 0, 0};
  threadIdx = {(unsigned)i % kBlock, 0, 0};
  gridDim = {1u << 20, 1, 1};
}
}  // namespace

extern "C" {

int emul_ws_ints() { return hmpc::WS_STATE_INTS; }
int emul_select_threads() { return hmpc::SELECT_THREADS; }

int emul_record_stride(int N) { return hmpc::record_stride(N); }

void emul_prepare(const unsigned char* states, int batch, int N, double dtMPC, unsigned char* records)
{
  for (int i = 0; i < batch; i++) {
    set_thread(i);
    hmpc::hmpc_prepare_kernel(states, batch, N, dtMPC, records, hmpc::record_stride(N));
  }
}

void emul_advance(unsigned char* states, unsigned char* loop, int batch, int N, double dtMPC, const float* wrench,
                  const int* status)
{
  for (int i = 0; i < batch; i++) {
    set_thread(i);
    hmpc::hmpc_advance_kernel(states, loop, batch, N, dtMPC, wrench, status, nullptr);
  }
}

void emul_swing(const unsigned char* states, const unsigned char* loop, const double* phase, unsigned char* swing, int batch,
                int n_iterations, double dt, double dtSwing, unsigned char* cmd)
{
  for (int i = 0; i < batch; i++) {
    set_thread(i);
    hmpc::hmpc_swing_kernel(states, loop, phase, swing, batch, n_iterations, dt, dtSwing, cmd);
  }
}

/* stage 1 of the solve kernel on one packed record's floats `rf` (layout: hmpc_device.cuh, "record floats"):
 * Fblk [192] (both legs' constraint rows), x0 [13], Acd [169], Bcd [156] — pre-zeroed as the kernel does. */
void emul_stage1(const float* rf, float dt, float* Fblk, float* x0, float* Acd, float* Bcd)
{
  memset(Fblk, 0, 192 * sizeof(float));
  memset(Acd, 0, 169 * sizeof(float));
  memset(Bcd, 0, 156 * sizeof(float));
  static float x0f[16];
  alignas(16) static unsigned char scr[512];
  memset(x0f, 0, sizeof(x0f));
  // the roles are warp-cooperative (libm calls spread over lanes): one emulated warp runs them the way stage 1 does
  run_cta(32, [=] {
    const int lane = (int)threadIdx.x;
    hmpc::role_leg(rf, lane, Fblk, scr);
    hmpc::role_state(rf, dt, x0f, Acd, lane, scr + 256);
    if (lane == 31) hmpc::role_inertia(rf, dt, Bcd);
  });
  memcpy(x0, x0f, 13 * sizeof(float));
}

/* the selection kernel of a masked call on one emulated CTA: list[0 .. *count) = the robots i < B with mask[i] != 0 */
void emul_select(const unsigned char* mask, int B, int* list, int* count) { run_select(mask, B, list, count); }

/* the class shapes of horizon N (hmpc::plan_classes): out[4][6] = variant, threads, shared-memory bytes, working-set
 * capacity, blocks of 6 variables, cached columns of classes 0-2 and the refinement class; returns the number of classes */
int emul_plan(int N, int* out)
{
  hmpc::ClassCfg cls[3], ref;
  const int ncls = hmpc::plan_classes(N, cls, ref);
  for (int i = 0; i < 4; i++) {
    const hmpc::ClassCfg& k = i < 3 ? cls[i] : ref;
    const int row[6] = {k.variant, k.threads, k.smem, k.qmax, k.nb_cap, k.tcap};
    memcpy(out + 6 * i, row, sizeof row);
  }
  return ncls;
}

/* One solve call of hmpc_capi.cu on B <= 1024 robots, each class on one emulated CTA.
 *   hostlists == 0: enqueue_solve's device-resident chain over packed `records` or, in place, the caller's update_data_t
 *                   records `raw` (the in-place mode): [the selection kernel over `mask`] -> class 0 over every robot (or the
 *                   listed ones), classifying on the way -> class 1 -> class 2 through the escalation lists -> [refinement].
 *   hostlists != 0: enqueue_solve_hostlists's launches over packed `records` (the zero-copy and copy-pipeline modes): class
 *                   lists built on the host from the contact tables, no escalation; with refinement on, then
 *                   enqueue_refine_retry's launch over the instances handed over.
 * refine: hmpc_set_refinement.  ws [B][WS_STATE_INTS] working sets, written back (proposed when warm != 0, moved `shift`
 * steps, or shifts[i] when shifts is not NULL), or NULL.  Outputs: wrench [B][12N] floats and/or wrench64 doubles, status [B],
 * tau [B][10] or NULL, launched[4] = instances class 0 kept, class 1, class 2 and the refinement class took (NULL to skip).
 * Optional assembly dump (all NULL, or all given): H [B][n*n], g [B][n], Fblk [B][192], lb/ub [B][16N].
 * Returns 2 when class 0 did not clear the next call's length words. */
int emul_solve(const unsigned char* records, const unsigned char* raw, int B, int N, int hostlists, int refine,
               const unsigned char* mask, int* ws, int warm, int shift, const int* shifts, float* wrench, double* wrench64,
               int* status, float* tau, int* launched, float* dH, float* dg, float* dF, float* dlb, float* dub)
{
  if (B < 1 || B > 1024 || (!records && !raw) || (hostlists && !records)) return 1;
  const hmpc::SolverSettings S = settings(refine);
  hmpc::ClassCfg cls[3], ref;
  const int ncls = hmpc::plan_classes(N, cls, ref);
  if (ncls == 0) return 1;
  hmpc::SolveIO io;
  io.records = records;
  io.raw = raw;
  io.batch = B;
  io.wrench = wrench;
  io.wrench64 = wrench64;
  io.status = status;
  io.tau = tau;
  io.ws = ws;
  io.warm = warm != 0;
  io.shift = shift;
  io.shifts = shifts;
  io.mask = mask;
  io.dump_H = dH, io.dump_g = dg, io.dump_F = dF, io.dump_lb = dlb, io.dump_ub = dub;
  int la[4] = {0, 0, 0, 0};
  std::vector<int> mem;
  hmpc::ChainLists lists;
  if (!hostlists) {
    mem.assign(hmpc::ClassSlot::cls_slot_ints(B), 0);
    const hmpc::ClassSlot slot{mem.data(), B, 0};
    int* next = slot.counts_next();
    for (int w = 0; w < 5; w++) next[w] = 0x55;  // the class-0 launch must clear them
    lists = hmpc::slot_lists(slot, mask != nullptr, S.refine);
    if (mask) run_select(mask, B, slot.list0(), slot.counts());
    for (int i = 0; i < ncls; i++) {
      const int n = (i == 0 && !mask) ? B : lists.counts[i];
      if (n == 0) continue;
      run_class(S, N, ncls, i, cls[i], io, lists);
      la[i] = i == 0 ? n - lists.counts[1] : n;  // class 0 hands instances to class 1 as it classifies or overflows
      if (i == 0 && (next[0] | next[1] | next[2] | next[3] | next[4])) return 2;
    }
  } else {
    mem.assign(hmpc::host_lists_ints(B) + 1 + B, 0);
    int* block = mem.data();
    int* ref_list = block + hmpc::host_lists_ints(B);  // [length | entries], as hmpc_ctx::d_ref
    hmpc::classify_host(N, S.f_max, cls[0].nb_hi, records + (54 + 12 * N) * 4, hmpc::record_stride(N), B, block, B, mask);
    lists = hmpc::host_lists(block, B, S.refine ? ref_list : nullptr, false);
    for (int i = 0; i < 2; i++)
      if ((la[i] = block[i]) > 0) run_class(S, N, ncls, i, cls[i], io, lists);
  }
  if (S.refine && (la[3] = *lists.ref_count) > 0) run_class(S, N, ncls, hmpc::REFINE_CLASS, ref, io, lists);
  if (launched) memcpy(launched, la, sizeof la);
  return 0;
}

/* the torque epilogue's per-joint function: tau_j = column j of J_force_moment(q5, leg) . f6 */
double emul_leg_torque(const double* q5, int leg, int j, const double* f6) { return hmpc::leg_torque(q5, leg, j, f6); }

}  // extern "C"
