// hmpc_chain.h — the solve-kernel chain, described once for the library (hmpc_capi.cu) and for the host emulation of the
// kernel source (tests/host_emul/kernel_source_on_host.cpp): the kernel variants, the shapes of the size classes, the
// class-list memory and the arguments of every launch.  Host C++ only, no CUDA runtime calls; include hmpc_device.cuh first.
//
// One solve is a fixed sequence of launches: [selection kernel (masked calls)] -> [preparation (states in)] -> class 0
// (classifies on the way) -> class 1 -> class 2 (reached by escalation) -> [refinement class (hmpc_set_refinement)].
// A call with robot states (hmpc_state_t) in runs the preparation kernel over the selection kernel's class-0 list (or over
// every robot) into the record buffer that class 0 then reads; preparation waits for the selection kernel, class 0 for
// preparation.
#pragma once
#include <cstddef>

namespace hmpc {

// The instantiations of hmpc_solve_kernel: X(variant, threads, min CTAs/SM, fixed horizon (0 = runtime), kernel class)
//   0/1: horizon 10 fixed at compile time (class 0: 4 warps, 6 CTAs/SM — shared memory would allow 7, but at 7 the
//        register budget of 72 spills more and the 1024-robot batch was slower on the H100; class 1: 8 warps)
//   10 + 5*cls + b: runtime horizon, b-th entry of {64, 128, 192, 256, 384} threads (class 2 runs class 1's kernel)
//   20 + b: the refinement class, the same thread counts (one CTA per SM: it is rare and its shared memory is large)
//   MQ_VARIANT + v (HMPC_MQ_VARIANTS): the multi-query instantiation of variant v (hmpc_solve_device_multi), the same shape
constexpr int MQ_VARIANT = 100;
#define HMPC_VARIANTS(X) \
  X(0, 128, 6, 10, 0)    \
  X(1, 256, 2, 10, 1)    \
  X(20, 64, 1, 0, 3)     \
  X(21, 128, 1, 0, 3)    \
  X(22, 192, 1, 0, 3)    \
  X(23, 256, 1, 0, 3)    \
  X(24, 384, 1, 0, 3)    \
  X(10, 64, 8, 0, 0)     \
  X(11, 128, 6, 0, 0)    \
  X(12, 192, 3, 0, 0)    \
  X(13, 256, 2, 0, 0)    \
  X(14, 384, 1, 0, 0)    \
  X(15, 64, 8, 0, 1)     \
  X(16, 128, 6, 0, 1)    \
  X(17, 192, 3, 0, 1)    \
  X(18, 256, 2, 0, 1)    \
  X(19, 384, 1, 0, 1)
#define HMPC_MQ_VARIANTS(X) \
  X(100, 128, 6, 10, 0) \
  X(101, 256, 2, 10, 1) \
  X(120, 64, 1, 0, 3)   \
  X(121, 128, 1, 0, 3)  \
  X(122, 192, 1, 0, 3)  \
  X(123, 256, 1, 0, 3)  \
  X(124, 384, 1, 0, 3)  \
  X(110, 64, 8, 0, 0)   \
  X(111, 128, 6, 0, 0)  \
  X(112, 192, 3, 0, 0)  \
  X(113, 256, 2, 0, 0)  \
  X(114, 384, 1, 0, 0)  \
  X(115, 64, 8, 0, 1)   \
  X(116, 128, 6, 0, 1)  \
  X(117, 192, 3, 0, 1)  \
  X(118, 256, 2, 0, 1)  \
  X(119, 384, 1, 0, 1)

constexpr int REFINE_CLASS = 3;           // kernel class of the refinement class
constexpr int SMEM_MAX = 226 * 1024;      // dynamic shared memory a class may take (the H100's opt-in maximum is 227 KB)

// Launch shape of one class.  grid_cap (resident CTAs) needs the device: plan_classes leaves it 0.
struct ClassCfg {
  int nb_hi, nb_cap, qmax, threads, smem, grid_cap, variant, tcap;
  Layout L;
};

// The variant of kernel class `kcls` at horizon N: the one fixed at N when `fixed` allows it, else the runtime-horizon one
// with the fewest threads that still give `warps` warps; multi-query instantiations when `mq`.  -1 when there is none.
inline int pick_variant(int N, int kcls, int warps, bool fixed, int* threads, bool mq = false)
{
  int v = -1;
#define HMPC_PICK(ID, NT, MB, NF, CL) \
  if (CL == kcls && NF == 0 && NT >= 32 * warps && (v < 0 || NT < *threads)) v = ID, *threads = NT;
  HMPC_VARIANTS(HMPC_PICK)
#undef HMPC_PICK
#define HMPC_PICK(ID, NT, MB, NF, CL) \
  if (CL == kcls && NF == N && fixed && v >= 0) v = ID, *threads = NT;
  HMPC_VARIANTS(HMPC_PICK)
#undef HMPC_PICK
  return (v >= 0 && mq) ? MQ_VARIANT + v : v;
}

// Shapes of classes 0-2 (cls) and of the refinement class (ref) at horizon N.  Returns the number of size classes, 2 when
// class 1 already holds every row class 2 could, or 0 when the horizon is too long for the built variants.
//   class 0: at most N blocks of 6 variables (e.g. any single-support schedule); class 1: up to 2N.  Working-set overflow in
//            class 0 escalates to class 1.
//   class 2: class 1's size with as many working-set slots as one SM's shared memory holds (1 CTA/SM) and no H^-1 a_j
//            cache (its primal steps go through a full product): reached only by escalation from class 1 (massively
//            degenerate optima, e.g. all contact forces at zero).
//   refinement: class 2's shape plus the float32 H tiles and g its refinement rounds read (refine_layout).  It holds
//            double support (2N blocks) while that leaves at least class 1's working-set capacity, i.e. up to horizon 14;
//            beyond that single support (N blocks), and an instance with more stance blocks keeps its code 4.
// mq: the multi-query instantiations of the same shapes (hmpc_solve_device_multi).
inline int plan_classes(int N, ClassCfg cls[3], ClassCfg& ref, bool mq = false)
{
  const int rs = record_stride(N);
  for (int i = 0; i < 2; i++) {
    ClassCfg& k = cls[i];
    k = ClassCfg{};
    k.nb_cap = k.nb_hi = class_nb_cap(N, i);
    k.variant = pick_variant(N, i, class_warps(N, i), true, &k.threads, mq);
    if (k.variant < 0) return 0;
    k.qmax = class_qmax(N, i);
    k.tcap = class_tcap(N, i);
    k.L = make_layout(N, k.nb_cap, k.qmax, rs, k.threads / 32, k.tcap);
    k.smem = k.L.total;
  }
  ClassCfg& k = cls[2];
  k = cls[1];
  k.variant = pick_variant(N, 1, class_warps(N, 1), false, &k.threads, mq);  // (a fixed variant folds class 1's layout)
  k.qmax = 6 * k.nb_cap;
  k.tcap = 0;
  k.L = make_layout(N, k.nb_cap, k.qmax, rs, k.threads / 32, 0);
  while (k.L.total > SMEM_MAX && k.qmax > cls[1].qmax) {
    k.qmax -= 4;
    k.L = make_layout(N, k.nb_cap, k.qmax, rs, k.threads / 32, 0);
  }
  k.smem = k.L.total;
  const int ncls = k.qmax > cls[1].qmax ? 3 : 2;
  for (int nb = 2 * N;; nb = N) {
    ref = ClassCfg{};
    ref.nb_cap = ref.nb_hi = nb;
    ref.variant = pick_variant(N, REFINE_CLASS, class_warps(N, nb == N ? 0 : 1), false, &ref.threads, mq);
    if (ref.variant < 0) return 0;
    ref.qmax = 6 * nb;
    ref.L = refine_layout(N, nb, ref.qmax, rs, ref.threads / 32);
    while (ref.L.total > SMEM_MAX && ref.qmax > 4) {
      ref.qmax -= 4;
      ref.L = refine_layout(N, nb, ref.qmax, rs, ref.threads / 32);
    }
    ref.smem = ref.L.total;
    if (nb == N || (ref.L.total <= SMEM_MAX && ref.qmax >= class_qmax(N, 1))) break;
  }
  return ncls;
}

// One slot of the device-resident chain's class-list memory (hmpc_ctx::d_cls), for max_batch robots:
//   [parity 0: 8 words | parity 1: 8 words | class-1 list | class-2 list | refinement list | class-0 list of a masked call]
// The words of a parity: the list lengths of classes 0-2, class 0's wave-barrier counter, the refinement list length and
// 3 unused.  A call uses one parity; its class-0 launch clears the other's first 5 words (KernelArgs::counts_next) for
// the next call.
struct ClassSlot {
  enum : int { W_WAVE = 3, W_REF = 4, PARITY_INTS = 8, HEAD_INTS = 2 * PARITY_INTS };
  static_assert(W_REF < 5, "the class-0 launch clears 5 words of the next parity");
  int* base;
  int max_batch;
  int par;
  static size_t cls_slot_ints(int max_batch) { return HEAD_INTS + 4 * (size_t)max_batch; }
  int* counts() const { return base + PARITY_INTS * par; }
  int* counts_next() const { return base + PARITY_INTS * (par ^ 1); }
  unsigned* wave() const { return reinterpret_cast<unsigned*>(counts() + W_WAVE); }
  int* ref_count() const { return counts() + W_REF; }
  int* list(int i) const { return base + HEAD_INTS + (size_t)(i - 1) * max_batch; }  // class i = 1, 2
  int* ref_list() const { return list(3); }
  int* list0() const { return list(4); }
};

// A chunk's host-built class lists (the host-buffer modes): [4 length words | class-0 list | class-1 list | class-2 list].
constexpr int HOST_LIST_HEAD = 4;
inline size_t host_lists_ints(int max_batch) { return HOST_LIST_HEAD + 3 * (size_t)max_batch; }
inline int* host_list(int* block, int max_batch, int i) { return block + HOST_LIST_HEAD + (size_t)i * max_batch; }

// The host-buffer modes classify while they pack (the rule class 0 applies on the device): robot i of the chunk, if `mask`
// (or NULL) lists it, goes to class 0 when at most nb_hi of its 2N contact-table entries give a non-zero force bound,
// else to class 1.  gait0: robot 0's contact table, gait_stride bytes apart.
inline void classify_host(int N, float f_max, int nb_hi, const unsigned char* gait0, size_t gait_stride, int nb, int* block,
                          int max_batch, const unsigned char* mask = nullptr)
{
  for (int w = 0; w < HOST_LIST_HEAD; w++) block[w] = 0;
  for (int i = 0; i < nb; i++) {
    if (mask && !mask[i]) continue;
    int k = 0;
    for (int e = 0; e < 2 * N; e++) {
      const float ub = f_max * (float)gait0[(size_t)i * gait_stride + e];
      k += !(ub < 0.0001f && ub > -0.0001f);
    }
    const int cl = (k <= nb_hi) ? 0 : 1;
    host_list(block, max_batch, cl)[block[cl]++] = i;
  }
}

// The context's solver settings (hmpc_create fills them, environment overrides included).
struct SolverSettings {
  float dt = 0.04f, f_max = 500.f;  // hmpc_set_problem
  int max_iter = 500;               // same cap as the reference's nWSR (SolverMPC.cpp:584)
  double tol_kkt = 1e-9;            // a row counts as violated below -tol_kkt * max(1, |x0|_inf)
  double tol_dep = 1e-11;           // an entering row is dependent below tol_dep * a'H^-1a
  double kappa_max = 1.5e5;         // conditioning limit of the fp64 sweep inversion (HMPC_KAPPA_MAX; the kernel's stage 5)
  double kappa_refine = 1.5e4;      // hand-over threshold of classes 0-2 while refinement is on (HMPC_KAPPA_REFINE; DESIGN.md §2)
  double kappa_max_refined = 1e9;   // conditioning limit of the refinement class (HMPC_KAPPA_MAX_REFINED)
  int refine = 0;                   // hmpc_set_refinement: instances beyond the limit go to the refinement class, not code 4
  int block_rounds = 4;             // block start of the active-set stage (HMPC_BLOCK_ROUNDS=0: plain dual iteration, A/B runs)
  int block_min = 2;                // later rounds need at least this many entering rows (HMPC_BLOCK_MIN, A/B knob)
  int lockstep = 1;                 // waves of class 0 start together (HMPC_LOCKSTEP=0: free-running, for A/B runs)
};

// What one solve call hands its launches.  Unused pointers stay null.
struct SolveIO {
  const void* records = nullptr;             // packed records (with `states`: the buffer the preparation writes)
  const void* raw = nullptr;                 // or the caller's update_data_t records, read in place (3016-byte stride)
  const void* states = nullptr;              // or hmpc_state_t [batch] (352-byte stride): the chain prepares `records`
  double dt_mpc = 0.0;                       // the preparation's MPC step
  int batch = 0;
  float* wrench = nullptr;                   // [batch][12N] float results
  double* wrench64 = nullptr;                // [batch][12N] double results
  int* status = nullptr;                     // [batch]
  float* tau = nullptr;                      // [batch][10] joint torques
  int* ws = nullptr;                         // [batch][WS_STATE_INTS] working sets, written back; proposed when `warm`
  bool warm = false;
  int shift = 1;                             // MPC steps the horizon moved since the sets were recorded (< 0: no history)
  const int* shifts = nullptr;               // [batch] the same per robot, or null
  const unsigned char* mask = nullptr;       // masked call: class 0 runs over the list the selection kernel builds from it
  float *dump_H = nullptr, *dump_g = nullptr, *dump_F = nullptr, *dump_lb = nullptr, *dump_ub = nullptr;  // assembly dump
};

// Where a launch finds its list and hands instances over.
struct ChainLists {
  int* counts = nullptr;     // list lengths: counts[cls] is the launch's
  int* list[3] = {};         // lists of classes 0-2; null: the class runs over every robot
  int* ref_count = nullptr;  // the refinement list's length and entries (null: refinement off)
  int* ref_list = nullptr;
  // the device-resident chain (else null): class 0 classifies on the way, clears the next call's lengths (5 words) and
  // holds its waves together at the wave barrier
  int* counts_next = nullptr;
  unsigned* wave = nullptr;
  bool escalate = false;     // working-set overflow goes to the next class's list (else the caller retries)
};

// The device-resident chain in `slot`
inline ChainLists slot_lists(const ClassSlot& s, bool masked, bool refine)
{
  ChainLists l;
  l.counts = s.counts();
  l.list[0] = masked ? s.list0() : nullptr;
  l.list[1] = s.list(1);
  l.list[2] = s.list(2);
  if (refine) l.ref_count = s.ref_count(), l.ref_list = s.ref_list();
  l.escalate = true;
  l.counts_next = s.counts_next();
  l.wave = s.wave();
  return l;
}

// host-built lists in `block` (host_lists_ints), refinement list [length | entries] in `ref` or null
inline ChainLists host_lists(int* block, int max_batch, int* ref, bool escalate)
{
  ChainLists l;
  l.counts = block;
  for (int i = 0; i < 3; i++) l.list[i] = host_list(block, max_batch, i);
  if (ref) l.ref_count = ref, l.ref_list = ref + 1;
  l.escalate = escalate;
  return l;
}

// The preparation launch of a states chain: every robot, or class 0's list when the selection kernel built one.  One
// thread per list entry at most: launch prepare_grid(io.batch) CTAs of PREPARE_THREADS.
constexpr int PREPARE_THREADS = 64;
inline int prepare_grid(int batch) { return (batch + PREPARE_THREADS - 1) / PREPARE_THREADS; }
// hmpc_prepare_kernel's parameters, in its order
struct PrepareArgs {
  const unsigned char* states;
  int batch, N;
  double dtMPC;
  unsigned char* records;
  int rec_stride;
  const int* list;
  const int* count;
};
inline PrepareArgs prepare_args(int N, const SolveIO& io, const ChainLists& lists)
{
  PrepareArgs pa{};
  pa.states = static_cast<const unsigned char*>(io.states);
  pa.batch = io.batch;
  pa.N = N;
  pa.dtMPC = io.dt_mpc;
  pa.records = static_cast<unsigned char*>(const_cast<void*>(io.records));  // (written here, read by the classes)
  pa.rec_stride = record_stride(N);
  pa.list = lists.list[0];
  pa.count = lists.list[0] ? lists.counts : nullptr;  // class 0's length word is counts[0]
  return pa;
}

// The carry launch of a sharded masked call (hmpc_carry_kernel), behind the chain: one thread per 16-byte vector of the
// batch's float wrench rows, carry_grid(batch, N) CTAs of CARRY_THREADS.
inline int carry_row_vecs(int N) { return 3 * N; }  // a row is 12N floats = 48N bytes
inline int carry_grid(int batch, int N)
{
  return (int)(((long long)batch * carry_row_vecs(N) + CARRY_THREADS - 1) / CARRY_THREADS);
}

// The prediction launch (hmpc_predict_kernel): one warp per robot, predict_grid(batch) CTAs of PREDICT_THREADS.  It is not
// part of the chain: it runs behind the solve that wrote the wrenches, in plain stream order.
inline int predict_grid(int batch)
{
  constexpr int warps = PREDICT_THREADS / 32;
  return (batch + warps - 1) / warps;
}

// The certificate launch (hmpc_certify_kernel): one warp per robot, certify_grid(batch) CTAs of CERT_THREADS, behind the
// wrenches it judges in plain stream order.  Its rows come in two layouts: the packed records of the device calls and the
// update_data_t rows of the host calls.  The first 42 floats (state and weights) lie at the same offsets in both; Alpha_K,
// traj and the gait bytes do not.
inline int certify_grid(int batch)
{
  constexpr int warps = CERT_THREADS / 32;
  return (batch + warps - 1) / warps;
}
inline RowLayout packed_rows(int N) { return RowLayout{record_stride(N), 42 * 4, 54 * 4, (54 + 12 * N) * 4}; }
inline RowLayout update_rows() { return RowLayout{3016, 1896, 168, 1944}; }  // convexMPC_interface.h's update_data_t

// The arguments of the launch of class `cls` (0-2, or REFINE_CLASS: the refinement class over lists.ref_list), shaped `k`.
inline KernelArgs launch_args(const SolverSettings& S, int N, int ncls, int cls, const ClassCfg& k, const SolveIO& io,
                              const ChainLists& lists)
{
  const bool refinement = cls == REFINE_CLASS;
  const bool first = cls == 0 && lists.counts_next;  // class 0 of the device-resident chain
  KernelArgs ka{};
  ka.records = static_cast<const unsigned char*>(io.records);
  ka.raw_records = static_cast<const unsigned char*>(io.raw);
  ka.rec_stride = record_stride(N);
  ka.batch = io.batch;
  ka.horizon = N;
  ka.dt = S.dt;
  ka.f_max = S.f_max;
  ka.list = refinement ? lists.ref_list : lists.list[cls];
  ka.counts = refinement ? lists.ref_count : lists.counts;  // the refinement list's length is its counts[0]
  ka.cls = refinement ? 0 : cls;
  ka.esc_list = (!refinement && lists.escalate && cls + 1 < ncls) ? lists.list[cls + 1] : nullptr;
  ka.split_nb = first ? k.nb_hi : -1;
  if (!refinement) ka.ref_list = lists.ref_list, ka.ref_count = lists.ref_count;
  ka.counts_next = first ? lists.counts_next : nullptr;
  // (class 1 runs free: its instances differ more in length, and waiting for the slowest of every wave cost more than
  // lockstep gained)
  ka.wave_sync = (first && S.lockstep) ? lists.wave : nullptr;
  ka.nb_cap = k.nb_cap;
  ka.qmax = k.qmax;
  ka.max_iter = S.max_iter;
  ka.tol_kkt = S.tol_kkt;
  ka.tol_dep = S.tol_dep;
  ka.tcap = k.tcap;
  // the refinement class solves from the unconstrained minimiser and records an empty set
  ka.block_rounds = refinement ? 0 : S.block_rounds;
  ka.block_min = refinement ? 0 : S.block_min;
  ka.kappa_max = refinement ? S.kappa_max_refined : (S.refine ? S.kappa_refine : S.kappa_max);
  ka.warm_start = (!refinement && io.ws && io.warm) ? 1 : 0;
  ka.ws_shift = refinement ? 0 : io.shift;
  ka.ws_shifts = refinement ? nullptr : io.shifts;
  ka.ws_state = io.ws;
  ka.wrench = io.wrench;
  ka.wrench64 = io.wrench64;
  ka.status = io.status;
  ka.dbg_H = io.dump_H;
  ka.dbg_g = io.dump_g;
  ka.dbg_F = io.dump_F;
  ka.dbg_lb = io.dump_lb;
  ka.dbg_ub = io.dump_ub;
  ka.tau = io.tau;
  ka.L = k.L;
  return ka;
}

// A multi-query call (hmpc_solve_device_multi): the chain of hmpc_solve_device over the io.batch robots with the multi-query
// classes (plan_classes(..., mq = true)), K candidate trajectories per robot (traj [batch][K][12N]) and results in rows
// i*K + k of io.wrench / io.wrench64 / io.status.  Calls are cold: no working set is proposed or recorded, and no torques.
// scratch[c]: class c's scratch (REFINE_CLASS: scratch[3]), mq_scratch_floats(N) floats per CTA of its launch.
// cmd: a multi-command states call (hmpc_solve_states_device_multi, below): [batch][K] commands, 7 doubles each; the chain's
// preparation writes traj from them.
struct MultiIO {
  const float* traj = nullptr;
  int K = 1;
  float* scratch[4] = {};
  const double* cmd = nullptr;
};
inline KernelArgs multi_launch_args(const SolverSettings& S, int N, int ncls, int cls, const ClassCfg& k, const SolveIO& io,
                                    const ChainLists& lists, const MultiIO& mq)
{
  KernelArgs ka = launch_args(S, N, ncls, cls, k, io, lists);
  ka.warm_start = 0;
  ka.ws_state = nullptr;
  ka.ws_shifts = nullptr;
  ka.tau = nullptr;
  ka.mq_traj = mq.traj;
  ka.mq_k = mq.K;
  ka.mq_scratch = mq.scratch[cls == REFINE_CLASS ? 3 : cls];
  return ka;
}
// CTAs a class's multi-query scratch serves: its launches have at most grid_cap CTAs, and a class's list holds at most
// max_batch entries
inline size_t mq_scratch_ctas(const ClassCfg& k, int max_batch) { return (size_t)(k.grid_cap < max_batch ? k.grid_cap : max_batch); }

// The multi-query call's cost launch (hmpc_multi_cost_kernel): one warp per result row, multi_cost_grid(batch * K) CTAs of
// PREDICT_THREADS, behind the chain in plain stream order.
inline int multi_cost_grid(long long nrows)
{
  constexpr int warps = PREDICT_THREADS / 32;
  return (int)((nrows + warps - 1) / warps);
}

// A multi-command states call (hmpc_solve_states_device_multi, hmpc_solve_batch_states_multi), one chain on one stream:
//   [the selection kernel over the mask]
//   -> the preparation (hmpc_prepare_kernel, prepare_args) of the listed robots' records into io.records, as in the states
//      chain; its traj is the state's own command's, which the pick kernel replaces
//   -> the trajectories (hmpc_prepare_traj_kernel) of their K commands mq.cmd into mq.traj [batch][K][12N],
//      prepare_grid(io.batch * K) CTAs of PREPARE_THREADS, one thread per (robot, candidate) over class 0's list (every
//      robot without a mask)
//   -> the multi-query classes over those records and trajectories (multi_launch_args)
//   -> the cost kernel (hmpc_multi_cost_kernel, multi_cost_grid(io.batch * K))
//   -> the pick kernel (hmpc_pick_kernel, pick_grid(io.batch)): best, torques, and the chosen trajectory into the record.
// The two preparation kernels are links of the PDL chain (each waits for its predecessor and the previous call before it
// reads or stores; class 0 waits for the second); the cost and pick kernels follow in plain stream order.
struct PrepareTrajArgs {
  const unsigned char* states;
  int batch, K;
  const double* cmd;
  int N;
  double dtMPC;
  float* traj;
  const int* list;
  const int* count;
};
inline PrepareTrajArgs prepare_traj_args(int N, const SolveIO& io, const ChainLists& lists, const MultiIO& mq)
{
  const PrepareArgs pa = prepare_args(N, io, lists);
  return PrepareTrajArgs{pa.states, pa.batch, mq.K, mq.cmd, N, pa.dtMPC, const_cast<float*>(mq.traj),  // (written here, read
                         pa.list, pa.count};                                                              // by the classes)
}
// the pick launch: one warp per robot
inline int pick_grid(int batch)
{
  constexpr int warps = PREDICT_THREADS / 32;
  return (batch + warps - 1) / warps;
}

}  // namespace hmpc
