// hmpc_chain.h — the solve-kernel chain, described once for the library (hmpc_capi.cu) and for the host emulation of the
// kernel source (tests/host_emul/kernel_source_on_host.cpp): the kernel variants, the shapes of the size classes, the
// class-list memory and the arguments of every launch.  Host C++ only, no CUDA runtime calls; include hmpc_device.cuh first.
//
// One solve is a fixed sequence of launches: [selection kernel (masked calls)] -> class 0 (classifies on the way) ->
// class 1 -> class 2 (reached by escalation) -> [refinement class (hmpc_set_refinement)].
#pragma once
#include <cstddef>

namespace hmpc {

// The instantiations of hmpc_solve_kernel: X(variant, threads, min CTAs/SM, fixed horizon (0 = runtime), kernel class)
//   0/1: horizon 10 fixed at compile time (class 0: 4 warps, 6 CTAs/SM — shared memory would allow 7, but at 7 the
//        register budget of 72 spills more and the 1024-robot batch was slower on the H100; class 1: 8 warps)
//   10 + 5*cls + b: runtime horizon, b-th entry of {64, 128, 192, 256, 384} threads (class 2 runs class 1's kernel)
//   20 + b: the refinement class, the same thread counts (one CTA per SM: it is rare and its shared memory is large)
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

constexpr int REFINE_CLASS = 3;           // kernel class of the refinement class
constexpr int SMEM_MAX = 226 * 1024;      // dynamic shared memory a class may take (the H100's opt-in maximum is 227 KB)

// Launch shape of one class.  grid_cap (resident CTAs) needs the device: plan_classes leaves it 0.
struct ClassCfg {
  int nb_hi, nb_cap, qmax, threads, smem, grid_cap, variant, tcap;
  Layout L;
};

// The variant of kernel class `kcls` at horizon N: the one fixed at N when `fixed` allows it, else the runtime-horizon one
// with the fewest threads that still give `warps` warps.  -1 when there is none.
inline int pick_variant(int N, int kcls, int warps, bool fixed, int* threads)
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
  return v;
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
inline int plan_classes(int N, ClassCfg cls[3], ClassCfg& ref)
{
  const int rs = record_stride(N);
  for (int i = 0; i < 2; i++) {
    ClassCfg& k = cls[i];
    k = ClassCfg{};
    k.nb_cap = k.nb_hi = class_nb_cap(N, i);
    k.variant = pick_variant(N, i, class_warps(N, i), true, &k.threads);
    if (k.variant < 0) return 0;
    k.qmax = class_qmax(N, i);
    k.tcap = class_tcap(N, i);
    k.L = make_layout(N, k.nb_cap, k.qmax, rs, k.threads / 32, k.tcap);
    k.smem = k.L.total;
  }
  ClassCfg& k = cls[2];
  k = cls[1];
  k.variant = pick_variant(N, 1, class_warps(N, 1), false, &k.threads);  // (a fixed variant folds class 1's layout)
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
    ref.variant = pick_variant(N, REFINE_CLASS, class_warps(N, nb == N ? 0 : 1), false, &ref.threads);
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
  const void* records = nullptr;             // packed records
  const void* raw = nullptr;                 // or the caller's update_data_t records, read in place (3016-byte stride)
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

}  // namespace hmpc
