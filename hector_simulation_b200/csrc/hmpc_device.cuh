// hmpc_device.cuh — sm_90a (H100) device code of the batched force-and-moment MPC solver.
//
// One CTA solves one robot's per-tick QP end to end (DESIGN.md §3):
//   stage 0  cp.async.bulk (TMA 1-D) of the packed record into shared memory
//   stage 1  SRBD linearisation + foot rotations + constraint rows      (SolverMPC.cpp:374-433, 463-548)
//   stage 2  forward-Euler discretisation, powers, Toeplitz blocks       (SolverMPC.cpp:133-193)
//   stage 3  Hessian / gradient of the condensed QP, swing-leg removal   (SolverMPC.cpp:450-461, 557-570, 589-697)
//   stage 4  blocked symmetric sweep inversion of H on the fp64 tensor pipe: 8x8 tiles in mma.sync.m8n8k4.f64
//            accumulator fragments, one barrier per 8-pivot block step
//   stage 5  dual active-set iterations on the explicit inverse           (replaces qpOASES, SolverMPC.cpp:702-712)
//   stage 6  scatter of the optimal wrenches, eliminated entries = 0     (SolverMPC.cpp:720-732)
//
// Stages 1-3 reproduce the reference's float32 arithmetic operation by operation (separately rounded
// multiply and add, same summation order) so that the QP data equals the oracle's bit for bit; they use
// the *_rn intrinsics, which the compiler never contracts into FMAs.  Stages 4-5 work in float64 on the
// float32-rounded data, like the reference hands float data to a double solver (SolverMPC.cpp:573-577).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace hmpc {

#define FM(a, b) __fmul_rn((a), (b))
#define FA(a, b) __fadd_rn((a), (b))
#define FS(a, b) __fsub_rn((a), (b))
#define FD(a, b) __fdiv_rn((a), (b))
#define DM(a, b) __dmul_rn((a), (b))
#define DA(a, b) __dadd_rn((a), (b))
#define DS(a, b) __dsub_rn((a), (b))

// termination codes (low byte of the status word, include/hector_mpc_b200.h)
enum : int { ST_OK = 0, ST_ITER_CAP = 1, ST_WS_CAP = 2, ST_INFEASIBLE = 3, ST_NOT_SPD = 4 };

// ------------------------------------------------------------------------------------------------
// shared-memory carve-up (byte offsets), computed once on the host and passed by value
// ------------------------------------------------------------------------------------------------
struct Layout {
  int H, gq, x0, nrm, fz, blk, keep, misc, uni;
  // solver view of the union
  int T, Sv, lam, dv, rr, wsl, zb;
  // sweep view of the union
  int Pb, Ws;
  // assembly view of the union
  int rec, x0f, Acd, Bcd, P, M, dd, fbl, comb;
  // refinement class only (refine_layout): float32 lower H tiles and gradient, kept for the refinement rounds
  int Hc, gc;
  int total;
};

__host__ __device__ constexpr int align16(int x) { return (x + 15) & ~15; }

// H and H^-1 live in shared memory as the lower 8x8 tiles of the symmetric matrix (diagonal tiles complete): tile
// (I,J), J <= I, at (I(I+1)/2 + J) * 64 elements, row-major inside.  During assembly the elements are the reference's
// float32 values; the sweep leaves float64 there.
__host__ __device__ constexpr int toff(int I, int J) { return (I * (I + 1) / 2 + J) * 64; }

__host__ __device__ constexpr Layout make_layout(int N, int nb_cap, int qmax, int rec_stride, int nwarps, int tcap)
{
  Layout L{};
  const int n = 6 * nb_cap;
  const int nt8 = (n + 7) / 8, ntile = nt8 * (nt8 + 1) / 2;
  int o = 0;
  L.H = o;    o += ntile * 64 * 8;
  L.gq = o;   o += nt8 * 8 * 8;       // gradient, zero-padded to whole tiles
  L.x0 = o;   o += n * 8;             // unconstrained minimiser
  L.nrm = o;  o += 2 * 10 * 6 * 8;    // the 20 distinct constraint normals
  L.fz = o;   o += align16(nb_cap * 8);  // per block: f_max * gait (right-hand side of the Fz upper bound)
  L.blk = o;  o += align16((nb_cap + 2 * N) * 4);  // block -> (step,leg) and (step,leg) -> block
  L.keep = o; o += 64;     // joint angles + quaternion survive the union's reuse (torque epilogue)
  L.misc = o; o += 512;
  L.uni = o;
  int s = L.uni;  // solver view; one slot more than the capacity: the entering row needs one while a blocking row leaves
  const int ns = qmax + 1;
  L.T = s;    s += (tcap + 1) * n * 8;              // H^-1 a_j of the first tcap working-set slots + one column for an entering row beyond them
  L.Sv = s;   s += ns * (ns + 1) / 2 * 8;           // (A_W H^-1 A_W')^-1, packed lower rows
  L.lam = s;  s += ns * 8;
  L.dv = s;   s += 2 * (ns + 2) * 8;                // step-direction scratch / double-buffered pivot column of the block start
  L.rr = s;   s += ns * 8;
  L.wsl = s;  s += align16(ns * 4);
  L.zb = L.gq;  // the gradient is spent once x0 is known (the steps that also keep A_W'r there order the two uses by a barrier)
  // sweep view: the tiles live in registers during the sweep, so its buffers take H's place when they fit there
  const int sweep_bytes = 2 * nt8 * 64 * 8 + nwarps * 2 * 64 * 8;
  int w = (sweep_bytes <= ntile * 64 * 8) ? L.H : L.uni;
  L.Pb = w;   w += 2 * nt8 * 64 * 8;                // pivot panel, double-buffered
  L.Ws = w;   w += nwarps * 2 * 64 * 8;             // per warp: -W of its two tile rows, fragment order
  if (sweep_bytes <= ntile * 64 * 8) w = L.uni;
  int a = L.uni;  // assembly view
  L.rec = a;  a += align16(rec_stride);
  L.x0f = a;  a += 16 * 4;
  L.Acd = a;  a += align16(169 * 4);
  L.Bcd = a;  a += align16(156 * 4);
  L.P = a;    a += 2 * align16(169 * 4);
  L.M = a;    a += align16(N * 72 * 4);
  L.dd = a;   a += align16(12 * N * 4);
  L.fbl = a;  a += 192 * 4;
  L.comb = a; a += align16(4 * N * 4);
  int m = s > a ? s : a;
  m = m > w ? m : w;
  L.total = align16(m);
  return L;
}

// The refinement class (CLS 3): make_layout without column cache, plus two regions that stage 4 would otherwise overwrite —
// a copy of the float32 lower H tiles (the sweep inverts them in place) and of the gradient (gq becomes zb).
__host__ __device__ constexpr Layout refine_layout(int N, int nb_cap, int qmax, int rec_stride, int nwarps)
{
  Layout L = make_layout(N, nb_cap, qmax, rec_stride, nwarps, 0);
  const int n = 6 * nb_cap, nt8 = (n + 7) / 8;
  L.Hc = L.total;
  L.gc = L.Hc + align16(nt8 * (nt8 + 1) / 2 * 64 * 4);
  L.total = align16(L.gc + n * 8);
  return L;
}

// packed record stride (include/hector_mpc_b200.h: hmpc_record_bytes)
__host__ __device__ constexpr int record_stride(int N) { return align16((54 + 12 * N) * 4 + 2 * N); }

// size classes: class 0 holds at most N blocks of 6 variables, class 1 up to 2N.  Working-set capacity: 2N + 4 rows for
// class 0 (a walking gait ends with about one active row per stance step; 24 at N = 10), 31 for class 1; an instance that needs more
// escalates to the next class (class 2 = class 1's size with as many slots as shared memory holds).
__host__ __device__ constexpr int class_nb_cap(int N, int cls) { return N * (1 + cls); }
// The H^-1 a_j cache costs n doubles per working-set slot.  Class 0 caches the first N + 4 slots (a walking gait ends with
// about one active row per stance step) and holds up to 2N + 4 rows: the rare instance that needs more than the cache takes
// its primal steps through a full H^-1 product for the uncached slots instead of escalating to the next class.  The
// long-horizon double-support class (extension configs) and class 2 do without the cache and spend the room on capacity.
__host__ __device__ constexpr int class_tcap(int N, int cls)
{
  const int n = 6 * class_nb_cap(N, cls);
  const int t = cls == 0 ? N + 4 : (N <= 10 ? 31 : 0);
  return t < n ? t : n;
}
__host__ __device__ constexpr int class_qmax(int N, int cls)
{
  const int n = 6 * class_nb_cap(N, cls);
  const int q = cls == 0 ? 2 * N + 4 : (N <= 10 ? 31 : 96);  // (the block start handles up to 31 rows: one mask word)
  return q < n ? q : n;
}
// warps a class needs: one per pair of tile rows of the sweep, one thread per constraint row (3 blocks of 10 per warp)
__host__ __device__ constexpr int class_warps(int N, int cls)
{
  const int nb = class_nb_cap(N, cls), n = 6 * nb, nt8 = (n + 7) / 8;
  const int w_sweep = (nt8 + 1) / 2, w_rows = (nb + 2) / 3;  // three blocks of ten rows per warp
  return w_sweep > w_rows ? w_sweep : w_rows;
}
__host__ __device__ constexpr Layout class_layout(int N, int cls, int nwarps)
{
  return make_layout(N, class_nb_cap(N, cls), class_qmax(N, cls), record_stride(N), nwarps, class_tcap(N, cls));
}

struct KernelArgs {
  const unsigned char* records;  // packed device records
  const unsigned char* raw_records;  // or: the caller's own update_data_t array (3016-byte stride, pinned + mapped host
                                     // memory), read in place over PCIe — nullptr in the packed modes
  int rec_stride;                // bytes, multiple of 16
  int batch;
  int horizon;                   // N
  float dt;
  float f_max;
  const int* list;               // instances of this launch's class (nullptr: identity over [0,batch))
  int* counts;                   // [ncls] list lengths (device); counts[cls] is this launch's
  int cls;                       // class index of this launch
  int* esc_list;                 // next class's list (working-set overflow escalation, size-class hand-over) or nullptr
  int split_nb;                  // >= 0: classify in this launch — an instance with more stance blocks goes to esc_list
  int* ref_list;                 // refinement class's list: instances whose scaled condition number exceeds kappa_max (no
                                 // non-positive pivot) are pushed here instead of ending with code 4; or nullptr (refinement off)
  int* ref_count;                // its length word
  int* counts_next;              // the next call's list lengths (5 words), zeroed by this launch (device-resident chain), or nullptr
  unsigned* wave_sync;           // arrival counter of the wave barrier of multi-wave launches (zero at launch), or nullptr
  int nb_cap;                    // capacity (blocks of 6 variables) the shared-memory carve is sized for
  int qmax;                      // working-set capacity
  int max_iter;
  double tol_kkt;                // a row counts as violated below -tol_kkt * max(1, |x0|_inf)   (default 1e-9)
  double tol_dep;                // an entering row is dependent on the working set when its curvature falls below tol_dep * a'H^-1a (1e-11)
  int tcap;                      // working-set slots with a cached H^-1 a_j column (runtime-layout launches; fixed: class_tcap)
  int block_rounds;              // rounds of the block start of the active-set stage (0: plain dual iteration from x0)
  int block_min;                 // rounds after the first run only with at least this many entering rows
  double kappa_max;              // conditioning limit of the sweep inversion: max_i H_ii (H^-1)_ii beyond it -> ST_NOT_SPD
  int warm_start;                // 1: propose the working set in `ws_state` (previous tick) to the block start
  int ws_shift;                  // MPC steps the horizon moved since that tick (the closed loop: 1); < 0: no history
  const int* ws_shifts;          // [batch] the same per robot (overrides ws_shift), or nullptr
  int* ws_state;                 // [batch][WS_STATE_INTS] persistent working sets, read (warm_start) and written back; or nullptr
  float* wrench;                 // [batch][12N] float results, or nullptr
  double* wrench64;              // [batch][12N] double results, or nullptr
  int* status;                   // [batch]
  // assembly dump (parity hook); all null in production launches
  float* dbg_H;                  // [batch][12N*12N]
  float* dbg_g;                  // [batch][12N]
  float* dbg_F;                  // [batch][192]
  float* dbg_lb;                 // [batch][16N]
  float* dbg_ub;                 // [batch][16N]
  float* tau;                    // [batch][10] joint torques of the first-step wrench (row f-2), or nullptr
  long long* dbg_clk;            // [batch][32] stage timestamps (clock64) of thread 0, profiling hook; null in production
  Layout L;
  // multi-query launches (hmpc_solve_kernel<..., MQ = true>): K reference trajectories per robot, results in row i*K + k
  const float* mq_traj;          // [batch][K][12N] the candidates' trajectories (the record's own traj is not used)
  int mq_k;                      // K
  float* mq_scratch;             // [gridDim.x][mq_scratch_floats(N)]: what stage 2 of a CTA's robot leaves for its later candidates
};

// Multi-query scratch of one CTA, floats: x0 (16) | Acd (172) | Bcd (156) | the state weights (12) | M (72N).  Stage 5 reuses
// the union these live in, so the later candidates of a robot read them back from here.
__host__ __device__ constexpr int mq_scratch_floats(int N) { return 16 + 172 + 156 + 12 + 72 * N; }

// ------------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// programmatic dependent launch (sm_90+): a kernel launched with the stream-serialization attribute may start while
// its predecessor drains; it must not touch anything the predecessor (or, transitively, earlier kernels) produces or
// still reads before pdl_wait() returns.  Both are no-ops for ordinary launches.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase)
{
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
// TMA 1-D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ int leg_of(int c12) { return (c12 / 3) & 1; }            // column of a 12-wide step -> leg
__device__ __forceinline__ int loc_of(int c12) { return (c12 % 3) + (c12 >= 6 ? 3 : 0); }  // -> slot in [F(3) M(3)]
__device__ __forceinline__ int col12_of(int leg, int loc) { return (loc < 3) ? 3 * leg + loc : 6 + 3 * leg + (loc - 3); }

// store element (i,j), i >= j, of the symmetric float32 Hessian into the tile layout (both triangles of a diagonal tile)
__device__ __forceinline__ void hput(float* Hf, int i, int j, float v)
{
  const int I = i >> 3, J = j >> 3;
  Hf[toff(I, J) + ((i & 7) << 3) + (j & 7)] = v;
  if (I == J) Hf[toff(I, I) + ((j & 7) << 3) + (i & 7)] = v;
}

// sum_c Hinv(i, j0 + c) * v[c], c < 6, j0 a multiple of 6: the six columns touch at most two tiles
__device__ __forceinline__ double hinv_dot6(const double* Hi, int i, int j0, const double* v)
{
  const int I = i >> 3, ir = i & 7;
  const int J0 = j0 >> 3, c0 = j0 & 7, J1 = J0 + 1;
  const int sA = (I >= J0) ? 1 : 8, sB = (I >= J1) ? 1 : 8;
  const double* pA = Hi + ((I >= J0) ? toff(I, J0) + ir * 8 + c0 : toff(J0, I) + c0 * 8 + ir);
  const double* pB = Hi + ((I >= J1) ? toff(I, J1) + ir * 8 : toff(J1, I) + ir) - (8 - c0) * sB;
  double acc = 0.0;
#pragma unroll
  for (int c = 0; c < 6; c++) acc = fma((c0 + c < 8) ? pA[c * sA] : pB[c * sB], v[c], acc);
  return acc;
}

// row i of the symmetric tile-stored matrix times a vector padded to whole tiles
__device__ __forceinline__ double hinv_rowdot(const double* Hi, int i, int nt8, const double* v)
{
  const int I = i >> 3, ir = i & 7;
  double acc0 = 0.0, acc1 = 0.0;
  for (int J = 0; J < nt8; J++) {
    const double* p = Hi + ((J <= I) ? toff(I, J) + ir * 8 : toff(J, I) + ir);
    const int st = (J <= I) ? 1 : 8;
    const double* vv = v + 8 * J;
#pragma unroll
    for (int c = 0; c < 8; c += 2) {
      acc0 = fma(p[c * st], vv[c], acc0);
      acc1 = fma(p[(c + 1) * st], vv[c + 1], acc1);
    }
  }
  return acc0 + acc1;
}

__device__ __forceinline__ double dot6(const double* a, const double* b)
{
  double acc = a[0] * b[0];
#pragma unroll
  for (int c = 1; c < 6; c++) acc = fma(a[c], b[c], acc);
  return acc;
}

// fp64 tensor-core MMA (SASS: DMMA.884): C[8x8] += A[8x4] * B[4x8].  Lane l = 4g + t holds A[g][t], B[t][g] and
// C[g][2t], C[g][2t+1].
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b)
{
  asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// Pivot-panel tiles are kept in "fragment order": element (r,c) at (c>>2)*32 + r*4 + (c&3), so that the A/B operand
// fragment of k-half h is the contiguous run [h*32 + lane] and the accumulator pair of lane 4g+t is one 16-byte word.
__device__ __forceinline__ int frag_pair(int lane) { return ((lane & 2) << 4) + ((lane >> 2) << 2) + ((lane & 1) << 1); }
__device__ __forceinline__ int frag_elem(int r, int c) { return ((c >> 2) << 5) + (r << 2) + (c & 3); }

// Eigen 3x3 inverse restated (oracle: inverse3)
__device__ __forceinline__ float cof3(const float* m, int i, int j)
{
  int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return FS(FM(m[i1 * 3 + j1], m[i2 * 3 + j2]), FM(m[i1 * 3 + j2], m[i2 * 3 + j1]));
}
__device__ inline void inverse3(const float* m, float* inv)
{
  float c00 = cof3(m, 0, 0), c10 = cof3(m, 1, 0), c20 = cof3(m, 2, 0);
  float det = FA(FA(FM(c00, m[0]), FM(c10, m[3])), FM(c20, m[6]));
  float id = FD(1.0f, det);
  inv[0] = FM(c00, id);
  inv[1] = FM(c10, id);
  inv[2] = FM(c20, id);
  inv[3] = FM(cof3(m, 0, 1), id);
  inv[4] = FM(cof3(m, 1, 1), id);
  inv[5] = FM(cof3(m, 2, 1), id);
  inv[6] = FM(cof3(m, 0, 2), id);
  inv[7] = FM(cof3(m, 1, 2), id);
  inv[8] = FM(cof3(m, 2, 2), id);
}
// row-major 3x3 product, sequential k (oracle: matmul)
__device__ inline void mul3(const float* A, const float* B, float* C)
{
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      float acc = FM(A[i * 3], B[j]);
      acc = FA(acc, FM(A[i * 3 + 1], B[3 + j]));
      acc = FA(acc, FM(A[i * 3 + 2], B[6 + j]));
      C[i * 3 + j] = acc;
    }
}
// RobotState::set — Quaternionf::toRotationMatrix (RobotState.cpp:17-30)
__device__ inline void quat_to_R(const float* qq, float* R)
{
  float w = qq[0], x = qq[1], y = qq[2], z = qq[3];
  float tx = FM(2.f, x), ty = FM(2.f, y), tz = FM(2.f, z);
  float twx = FM(tx, w), twy = FM(ty, w), twz = FM(tz, w);
  float txx = FM(tx, x), txy = FM(ty, x), txz = FM(tz, x);
  float tyy = FM(ty, y), tyz = FM(tz, y), tzz = FM(tz, z);
  R[0] = FS(1.f, FA(tyy, tzz));
  R[1] = FS(txy, twz);
  R[2] = FA(txz, twy);
  R[3] = FA(txy, twz);
  R[4] = FS(1.f, FA(txx, tzz));
  R[5] = FS(tyz, twx);
  R[6] = FS(txz, twy);
  R[7] = FA(tyz, twx);
  R[8] = FS(1.f, FA(txx, tyy));
}

// Double-precision libm calls, one out-of-line copy each: inlined, every call site carries the whole routine (slow paths
// included) — about 2000 instructions of straight-line code that the instruction cache fetches once per robot.
__device__ __noinline__ void sincos_f64(double x, double* s, double* c) { sincos(x, s, c); }
__device__ __noinline__ double fmod_f64(double x, double y) { return fmod(x, y); }
__device__ __noinline__ double atan2_f64(double y, double x) { return atan2(y, x); }
__device__ __noinline__ double asin_f64(double x) { return asin(x); }

// foot rotation from the sines / cosines of five offset-corrected joint angles and of q2+q3+q4
// (SolverMPC.cpp:428-433; oracle: foot_rotation); sc = {s0, c0, s1, c1, ..., s4, c4, s234, c234}
__device__ inline void foot_rotation(const double* sc, float* Rf)
{
  const double s0 = sc[0], c0 = sc[1], s1 = sc[2], c1 = sc[3], s2 = sc[4], c2 = sc[5], s3 = sc[6], c3 = sc[7], s4 = sc[8],
               c4 = sc[9], s234 = sc[10], c234 = sc[11];
  double a = DA(DM(c0, s2), DM(DM(c2, s0), s1));
  double b = DS(DM(c0, c2), DM(DM(s0, s1), s2));
  double c = DA(DM(c2, s0), DM(DM(c0, s1), s2));
  double d = DS(DM(s0, s2), DM(DM(c0, c2), s1));
  double c3a_s3b = DA(DM(c3, a), DM(s3, b));
  double s3a_c3b = DS(DM(s3, a), DM(c3, b));
  double c3c_s3d = DS(DM(c3, c), DM(s3, d));
  double s3c_c3d = DA(DM(s3, c), DM(c3, d));
  Rf[0] = (float)DS(DM(-s4, c3a_s3b), DM(c4, s3a_c3b));
  Rf[1] = (float)DM(-c1, s0);
  Rf[2] = (float)DS(DM(c4, c3a_s3b), DM(s4, s3a_c3b));
  Rf[3] = (float)DS(DM(c4, c3c_s3d), DM(s4, s3c_c3d));
  Rf[4] = (float)DM(c0, c1);
  Rf[5] = (float)DA(DM(c4, s3c_c3d), DM(s4, c3c_s3d));
  Rf[6] = (float)DM(-s234, c1);
  Rf[7] = (float)s1;
  Rf[8] = (float)DM(c234, c1);
}

// ------------------------------------------------------------------------------------------------
// stage 1, split into three independent roles that run on different warps (each recomputes the cheap R)
// record floats: p[0..2] v[3..5] q[6..9] w[10..12] r[13..18] joint[19..28] yaw[29] weights[30..41]
//                alpha[42..53] traj[54..54+12N)  then gait bytes.   Acd/Bcd/Fblk are pre-zeroed.
// The libm calls of a role run on different lanes (one joint angle per lane, ...), the arithmetic that combines them
// on one lane as before — operation for operation the oracle's.
// ------------------------------------------------------------------------------------------------
// role "leg" (whole warp; lanes 0..9 = joints, then lanes 0..1 = legs): joint offsets + fmod (SolverMPC.cpp:374-393),
// foot rotation, the leg's 8 constraint rows (:488-548).  scr: 10 floats + pad, then 2 x 12 doubles.
__device__ inline void role_leg(const float* rf, int lane, float* Fblk, unsigned char* scr)
{
  const double PI = 3.14159265359;
  float* qf = reinterpret_cast<float*>(scr);          // [10] offset-corrected, reduced joint angles
  double* sc = reinterpret_cast<double*>(scr + 48);   // [2][12] sines / cosines per leg
  if (lane < 10) {
    const int i = lane % 5;
    float q = rf[19 + lane];
    if (i == 2) q = (float)DA((double)q, DM(0.3, PI));
    if (i == 3) q = (float)DS((double)q, DM(0.6, PI));
    if (i == 4) q = (float)DA((double)q, DM(0.3, PI));
    q = (float)fmod_f64((double)q, DM(2.0, PI));
    qf[lane] = q;
    sincos_f64((double)q, sc + 12 * (lane / 5) + 2 * i, sc + 12 * (lane / 5) + 2 * i + 1);
  }
  __syncwarp();
  if (lane >= 2) return;
  const int leg = lane;
  const float* q = qf + 5 * leg;
  const float q234 = FA(FA(q[2], q[3]), q[4]);
  sincos_f64((double)q234, sc + 12 * leg + 10, sc + 12 * leg + 11);
  float R[9], Rf[9];
  quat_to_R(rf + 6, R);
  foot_rotation(sc + 12 * leg, Rf);
  const float mu = 2.0f, lt = 0.09f, lh = 0.06f;
  const int r0 = 8 * leg, cF = 3 * leg, cM = 6 + 3 * leg;
  Fblk[(r0 + 0) * 12 + cF + 0] = -mu; Fblk[(r0 + 0) * 12 + cF + 2] = 1.f;
  Fblk[(r0 + 1) * 12 + cF + 0] = mu;  Fblk[(r0 + 1) * 12 + cF + 2] = 1.f;
  Fblk[(r0 + 2) * 12 + cF + 1] = -mu; Fblk[(r0 + 2) * 12 + cF + 2] = 1.f;
  Fblk[(r0 + 3) * 12 + cF + 1] = mu;  Fblk[(r0 + 3) * 12 + cF + 2] = 1.f;
  float v1t[3] = {FM(-lt, Rf[2]), FM(-lt, Rf[5]), FM(-lt, Rf[8])};
  float v1h[3] = {FM(-lh, Rf[2]), FM(-lh, Rf[5]), FM(-lh, Rf[8])};
  for (int j = 0; j < 3; j++) {
    float xw = FA(FA(FM(Rf[0], R[j * 3]), FM(Rf[3], R[j * 3 + 1])), FM(Rf[6], R[j * 3 + 2]));
    float yw = FA(FA(FM(Rf[1], R[j * 3]), FM(Rf[4], R[j * 3 + 1])), FM(Rf[7], R[j * 3 + 2]));
    float zt = FA(FA(FM(v1t[0], R[j * 3]), FM(v1t[1], R[j * 3 + 1])), FM(v1t[2], R[j * 3 + 2]));
    float zh = FA(FA(FM(v1h[0], R[j * 3]), FM(v1h[1], R[j * 3 + 1])), FM(v1h[2], R[j * 3 + 2]));
    Fblk[(r0 + 4) * 12 + cM + j] = xw;
    Fblk[(r0 + 5) * 12 + cF + j] = zt;
    Fblk[(r0 + 5) * 12 + cM + j] = yw;
    Fblk[(r0 + 6) * 12 + cF + j] = zh;
    Fblk[(r0 + 6) * 12 + cM + j] = (leg == 0) ? -yw : yw;  // quirk Q5
  }
  Fblk[(r0 + 7) * 12 + cF + 2] = 2.f;
}
// role "state" (whole warp; lanes 0..2 = the three Euler angles, lanes 0..1 = their sines / cosines, lane 0 the rest):
// rpy (SolverMPC.cpp:333-342), Rb (:65-89), x0 (:420), the non-trivial entries of Acd (:145,315-317).
// scr: 3 floats + pad, then 4 doubles.
__device__ inline void role_state(const float* rf, float dt, float* x0f, float* Acd, int lane, unsigned char* scr)
{
  float* rpy = reinterpret_cast<float*>(scr);
  double* sc = reinterpret_cast<double*>(scr + 16);  // sp, cp, sy, cy
  if (lane < 3) {
    const float qw = rf[6], qx = rf[7], qy = rf[8], qz = rf[9];
    if (lane == 0) {
      rpy[0] = (float)atan2_f64((double)FM(2.f, FA(FM(qw, qx), FM(qy, qz))), DS(1.0, (double)FM(2.f, FA(FM(qx, qx), FM(qy, qy)))));
    } else if (lane == 1) {
      double as_d = DM(2.0, (double)FS(FM(qw, qy), FM(qx, qz)));
      if (!(as_d < .99999)) as_d = .99999;
      const float as = (float)as_d;
      rpy[1] = (float)asin_f64((double)as);
    } else {
      rpy[2] = (float)atan2_f64((double)FM(2.f, FA(FM(qw, qz), FM(qx, qy))), DS(1.0, (double)FM(2.f, FA(FM(qy, qy), FM(qz, qz)))));
    }
  }
  __syncwarp();
  if (lane < 2) sincos_f64((double)rpy[1 + lane], sc + 2 * lane, sc + 2 * lane + 1);
  __syncwarp();
  if (lane != 0) return;
  float Rb[9];
  {
    const double sp = sc[0], cp = sc[1], sy = sc[2], cy = sc[3];
    float Rbm[9] = {(float)DM(cy, cp), (float)(-sy), 0.f, (float)DM(sy, cp), (float)cy, 0.f, (float)(-sp), 0.f, 1.f};
    inverse3(Rbm, Rb);
  }
  for (int i = 0; i < 3; i++) {
    x0f[i] = rpy[i];
    x0f[3 + i] = rf[i];
    x0f[6 + i] = rf[10 + i];
    x0f[9 + i] = rf[3 + i];
  }
  x0f[12] = 9.81f;
  for (int i = 0; i < 13; i++) Acd[i * 13 + i] = 1.f;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) Acd[i * 13 + 6 + j] = FA(0.f, FM(dt, Rb[i * 3 + j]));
  for (int i = 0; i < 3; i++) Acd[(3 + i) * 13 + 9 + i] = FA(0.f, FM(dt, 1.f));
  Acd[11 * 13 + 12] = FA(0.f, FM(dt, -1.f));
}
// role "inertia": I_world, its inverse (SolverMPC.cpp:421, 320) and Bcd = dt*B (:146, 323-330), m = 9.0 (:423)
__device__ inline void role_inertia(const float* rf, float dt, float* Bcd)
{
  float R[9], Iinv[9];
  quat_to_R(rf + 6, R);
  {
    const float Ib[3] = {0.5413f, 0.5200f, 0.0691f};
    float RI[9], Rt[9], Iw[9];
    for (int i = 0; i < 3; i++)
      for (int k = 0; k < 3; k++) {
        RI[i * 3 + k] = FM(R[i * 3 + k], Ib[k]);
        Rt[i * 3 + k] = R[k * 3 + i];
      }
    mul3(RI, Rt, Iw);
    inverse3(Iw, Iinv);
  }
  for (int b = 0; b < 2; b++) {
    float rx = rf[13 + 0 + b], ry = rf[13 + 2 + b], rz = rf[13 + 4 + b];
    float cm[9] = {0.f, -rz, ry, rz, 0.f, -rx, -ry, rx, 0.f};
    float blk[9];
    mul3(Iinv, cm, blk);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) Bcd[(6 + i) * 12 + b * 3 + j] = FM(dt, blk[i * 3 + j]);
  }
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      float v = FM(dt, Iinv[i * 3 + j]);
      Bcd[(6 + i) * 12 + 6 + j] = v;
      Bcd[(6 + i) * 12 + 9 + j] = v;
    }
  float v = FM(dt, FD(1.f, 9.0f));
  for (int i = 0; i < 3; i++) {
    Bcd[(9 + i) * 12 + i] = v;
    Bcd[(9 + i) * 12 + 3 + i] = v;
  }
}

// Column j of the leg's 6x5 force-and-moment Jacobian (LegController.cpp:130-166, restated with the link lever
// sums S_k, C_k seen from joints 2..4), dotted with the 6-vector f: one joint torque (LegController.cpp:61).
__device__ inline double leg_torque(const double* q5, int leg, int j, const double* f)
{
  const double side = (leg == 0) ? 1.0 : -1.0;
  double s0, c0, s1, c1;
  sincos_f64(q5[0], &s0, &c0);
  sincos_f64(q5[1], &s1, &c1);
  double s234, c234, s23, c23, s2, c2;
  sincos_f64(q5[2] + q5[3] + q5[4], &s234, &c234);
  sincos_f64(q5[2] + q5[3], &s23, &c23);
  sincos_f64(q5[2], &s2, &c2);
  const double h = 0.018 * side + 0.0025, e = 0.015 * side;
  double J[6];
  if (j == 0) {
    const double S = 0.04 * s234 + 0.22 * s23 + 0.22 * s2, C = 0.04 * c234 + 0.22 * c23 + 0.22 * c2;
    const double a = e + c1 * h - s1 * C;
    J[0] = s0 * (S + 0.0135) + c0 * a;
    J[1] = s0 * a - c0 * (S + 0.0135);
    J[2] = 0.0; J[3] = 0.0; J[4] = 0.0; J[5] = 1.0;
  } else if (j == 1) {
    const double C = 0.04 * c234 + 0.22 * c23 + 0.22 * c2;
    const double b = s1 * h + c1 * C;
    J[0] = -s0 * b;
    J[1] = c0 * b;
    J[2] = s1 * C - c1 * h;
    J[3] = c0; J[4] = s0; J[5] = 0.0;
  } else {
    const double S = 0.04 * s234 + (j <= 3 ? 0.22 * s23 : 0.0) + (j == 2 ? 0.22 * s2 : 0.0);
    const double C = 0.04 * c234 + (j <= 3 ? 0.22 * c23 : 0.0) + (j == 2 ? 0.22 * c2 : 0.0);
    J[0] = s0 * s1 * S - c0 * C;
    J[1] = -s0 * C - c0 * s1 * S;
    J[2] = c1 * S;
    J[3] = -c1 * s0; J[4] = c0 * c1; J[5] = s1;
  }
  double t = 0.0;
#pragma unroll
  for (int r = 0; r < 6; r++) t = fma(J[r], f[r], t);
  return t;
}

// Row f-2: the feed-forward torque of joint j of leg `leg`, tau = J_force_moment^T * f_ff with f_ff = -rBody [F; M] of the leg's
// first-step wrench w [6] (ConvexMPCLocomotion.cpp:419-440, LegController.cpp:57-63); a swing leg (w null) gets no
// feed-forward force.  q10: a record's 10 joint-angle floats, quat: its 4 quaternion floats.  W: the wrench's element type
// (rounded to float first).  The pick kernel (hmpc_pick_kernel) runs it; it states the solve kernel's torque epilogue (stage
// 6) operation for operation, which keeps its own inline copy so that its instruction schedule stays as it is.
template <typename W>
__device__ __forceinline__ float joint_torque(const float* q10, const float* quat, int leg, int j, const W* w)
{
  const double PI = 3.14159265359;
  double q5[5];
#pragma unroll
  for (int i = 0; i < 5; i++) q5[i] = (double)q10[5 * leg + i];
  q5[2] -= 0.3 * PI;  // undo the caller's second offset: LegController's own angles
  q5[3] += 0.6 * PI;
  q5[4] -= 0.3 * PI;
  const double qw = quat[0], qx = quat[1], qy = quat[2], qz = quat[3];
  const double R[9] = {1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qw * qz), 2 * (qx * qz + qw * qy),
                       2 * (qx * qy + qw * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qw * qx),
                       2 * (qx * qz - qw * qy), 2 * (qy * qz + qw * qx), 1 - 2 * (qx * qx + qy * qy)};
  double fw[6] = {0, 0, 0, 0, 0, 0};
  if (w) {
#pragma unroll
    for (int r = 0; r < 3; r++) {  // rBody = R^T
      fw[r] = -(R[0 * 3 + r] * (double)(float)w[0] + R[1 * 3 + r] * (double)(float)w[1] + R[2 * 3 + r] * (double)(float)w[2]);
      fw[3 + r] = -(R[0 * 3 + r] * (double)(float)w[3] + R[1 * 3 + r] * (double)(float)w[4] + R[2 * 3 + r] * (double)(float)w[5]);
    }
  }
  return (float)leg_torque(q5, leg, j, fw);
}

// fast fp64 reciprocal: MUFU.RCP64H seed (relative error 9.9e-7 on the H100, tests/tools/ubench.cu) + two Newton steps:
// identical to the IEEE quotient on 5e7 probe values, a third step changes nothing; the IEEE division sequence is ~6x
// the instructions and the reciprocals sit on the critical chains of the tile inversions and the Schur sweeps
__device__ __forceinline__ double fast_rcp(double x)
{
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  double e = fma(-x, r, 1.0);
  r = fma(e, r, r);
  e = fma(-x, r, 1.0);
  r = fma(e, r, r);
  return r;
}

// order-preserving map float -> uint (for REDUX.MIN)
__device__ __forceinline__ unsigned fkey(float f)
{
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Inverse of a symmetric positive definite 8x8 tile held in accumulator-fragment layout (lane 4g+t: a[g][2t], a[g][2t+1]),
// by eight in-register sweeps; the reciprocal of pivot p+1 is predicted while pivot p is applied, so the dependent chain
// per pivot is one reciprocal plus two multiply-adds.  Returns true if a pivot was not positive.
__device__ __forceinline__ bool tile_inverse_spd(double& a0, double& a1, int lane)
{
  const int g = lane >> 2, t4 = lane & 3;
  bool bad = false;
  double inv = fast_rcp(__shfl_sync(0xffffffffu, a0, 0));
#pragma unroll
  for (int p = 0; p < 8; p++) {
    const double selp = (p & 1) ? a1 : a0;  // the element whose column has p's parity
    const double colp = __shfl_sync(0xffffffffu, selp, 4 * g + (p >> 1));  // a[g][p]
    const double r0 = __shfl_sync(0xffffffffu, a0, 4 * p + t4);            // a[p][2t], a[p][2t+1]
    const double r1 = __shfl_sync(0xffffffffu, a1, 4 * p + t4);
    const double d = __shfl_sync(0xffffffffu, selp, 4 * p + (p >> 1));     // a[p][p]
    bad |= !(d > 0.0);
    double invn = 0.0;
    if (p < 7) {  // next pivot after this sweep: a[p+1][p+1] - a[p+1][p]^2 / a[p][p]
      const double e = __shfl_sync(0xffffffffu, selp, 4 * (p + 1) + (p >> 1));
      const double dn0 = __shfl_sync(0xffffffffu, ((p + 1) & 1) ? a1 : a0, 4 * (p + 1) + ((p + 1) >> 1));
      invn = fast_rcp(fma(-e * inv, e, dn0));
    }
    const double f = colp * inv;
    double n0 = fma(-f, r0, a0), n1 = fma(-f, r1, a1);
    if (g == p) { n0 = r0 * inv; n1 = r1 * inv; }
    if (t4 == (p >> 1)) {
      const double pc = (g == p) ? -inv : f;
      if (p & 1) n1 = pc; else n0 = pc;
    }
    a0 = n0;
    a1 = n1;
    inv = invn;
  }
  a0 = -a0;
  a1 = -a1;
  return bad;
}

// working-set entry: block index in the high bits, normal index (leg*10+type) in the low byte
__device__ __forceinline__ int ws_pack(int blk, int nidx) { return (blk << 8) | nidx; }
__device__ __forceinline__ int tri(int s) { return s * (s + 1) / 2; }

// ------------------------------------------------------------------------------------------------
// row f-1: the caller's data preparation, one thread per robot (ConvexMPCLocomotion.cpp:283-406 followed by the
// double -> float narrowing of update_problem_data, convexMPC_interface.cpp:87-99).  Double arithmetic with
// explicitly rounded operations in the reference's order, so the packed record equals the host-prepared one.
// `states` points at hmpc_state_t records (352 bytes): 39 doubles then the gait bytes.
// ------------------------------------------------------------------------------------------------
// Row i of `records` is robot i's record.  `list` and its length word `count` (the masked chain: the selection kernel's
// class-0 list), or null: every robot in [0, batch).  With a list, thread t prepares robot list[t] for t < *count and no
// other record is written.
__global__ void hmpc_prepare_kernel(const unsigned char* states, int batch, int N, double dtMPC, unsigned char* records,
                                    int rec_stride, const int* list = nullptr, const int* count = nullptr)
{
  pdl_trigger();  // class 0 may become resident; it waits for this kernel before it reads the records
  // In the chain, the list comes from the selection kernel, and the previous call's kernels may still read the record
  // buffer: nothing is read or stored before they have completed.  A no-op for an ordinary launch.
  pdl_wait();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (list ? *count : batch)) return;
  const int i = list ? list[t] : t;
  const double* s = reinterpret_cast<const double*>(states + (size_t)i * 352);
  const unsigned char* gait = states + (size_t)i * 352 + 39 * 8;
  const double* pos = s;            // [3]
  const double* vw = s + 3;         // [3]
  const double* qt = s + 6;         // [4]
  const double* ow = s + 10;        // [3]
  const double* rpy = s + 13;       // [3]
  const double* lq = s + 16;        // [10]
  const double* lp = s + 26;        // [2][3]
  const double* sd = s + 32;        // roll, pitch, vx, vy, yaw rate
  const double* wpd = s + 37;       // [2]
  float* f = reinterpret_cast<float*>(records + (size_t)i * rec_stride);
  // body -> world rotation (= rBody^T), ori::quaternionToRotationMatrix before its transpose
  const double e0 = qt[0], e1 = qt[1], e2 = qt[2], e3 = qt[3];
  const double R[9] = {DS(1.0, DM(2.0, DA(DM(e2, e2), DM(e3, e3)))), DM(2.0, DS(DM(e1, e2), DM(e0, e3))), DM(2.0, DA(DM(e1, e3), DM(e0, e2))),
                       DM(2.0, DA(DM(e1, e2), DM(e0, e3))), DS(1.0, DM(2.0, DA(DM(e1, e1), DM(e3, e3)))), DM(2.0, DS(DM(e2, e3), DM(e0, e1))),
                       DM(2.0, DS(DM(e1, e3), DM(e0, e2))), DM(2.0, DA(DM(e2, e3), DM(e0, e1))), DS(1.0, DM(2.0, DA(DM(e1, e1), DM(e2, e2))))};
  for (int k = 0; k < 3; k++) { f[k] = (float)pos[k]; f[3 + k] = (float)vw[k]; f[10 + k] = (float)ow[k]; }
  for (int k = 0; k < 4; k++) f[6 + k] = (float)qt[k];
  // foot positions: pFoot = position + rBody^T (hip + leg.p); r[k] = pFoot[k%2][k/2] - position[k/2]   (:58-62, :315-319)
  double pf[2][3];
  for (int leg = 0; leg < 2; leg++) {
    const double hp[3] = {DA(-0.005, lp[3 * leg]), DA(leg == 0 ? -0.057 : 0.057, lp[3 * leg + 1]), DA(-0.126, lp[3 * leg + 2])};
    for (int a = 0; a < 3; a++)
      pf[leg][a] = DA(pos[a], DA(DA(DM(R[a * 3], hp[0]), DM(R[a * 3 + 1], hp[1])), DM(R[a * 3 + 2], hp[2])));
  }
  for (int k = 0; k < 6; k++) f[13 + k] = (float)DS(pf[k % 2][k / 2], pos[k / 2]);
  // joint angles: second offset + fmod (:289-313)
  const double PI = 3.14159265359, PI2 = DM(2.0, PI);
  for (int leg = 0; leg < 2; leg++) {
    double q5[5];
    for (int k = 0; k < 5; k++) q5[k] = lq[5 * leg + k];
    q5[2] = DA(q5[2], DM(0.3, PI));
    q5[3] = DS(q5[3], DM(0.6, PI));
    q5[4] = DA(q5[4], DM(0.3, PI));
    for (int k = 0; k < 5; k++) f[19 + 5 * leg + k] = (float)fmod(q5[k], PI2);
  }
  const double yaw = rpy[2];
  f[29] = (float)yaw;
  const float Qw[12] = {100, 100, 250, 200, 200, 300, 1, 1, 1, 1, 1, 1};                           // :321
  const float Al[12] = {1e-4f, 1e-4f, 5e-4f, 1e-4f, 1e-4f, 5e-4f, 1e-2f, 1e-2f, 1e-2f, 1e-2f, 1e-2f, 1e-2f};  // :322
  for (int k = 0; k < 12; k++) { f[30 + k] = Qw[k]; f[42 + k] = Al[k]; }
  // reference trajectory (:331-399)
  const double vdr[3] = {sd[2], sd[3], 0.0};
  double vdw[3];
  for (int a = 0; a < 3; a++) vdw[a] = DA(DA(DM(R[a * 3], vdr[0]), DM(R[a * 3 + 1], vdr[1])), DM(R[a * 3 + 2], vdr[2]));
  const double mpe = .05;
  double xS = wpd[0], yS = wpd[1];
  if (DS(xS, pos[0]) > mpe) xS = DA(pos[0], mpe);
  if (DS(pos[0], xS) > mpe) xS = DS(pos[0], mpe);
  if (DS(yS, pos[1]) > mpe) yS = DA(pos[1], mpe);
  if (DS(pos[1], yS) > mpe) yS = DS(pos[1], mpe);
  const double ti[12] = {sd[0], sd[1], 0.0, xS, yS, 0.55, 0, 0, sd[4], vdw[0], vdw[1], 0};
  for (int st = 0; st < N; st++) {
    double tr[12];
    for (int j = 0; j < 12; j++) tr[j] = ti[j];
    if (st == 0) {
      tr[0] = rpy[0]; tr[1] = rpy[1]; tr[2] = rpy[2];
      tr[3] = pos[0]; tr[4] = pos[1]; tr[5] = pos[2];
    } else {
      const double idt = DM((double)st, dtMPC);
      tr[3] = DA(vdw[0] == 0 ? ti[3] : pos[0], DM(idt, vdw[0]));
      tr[4] = DA(vdw[1] == 0 ? ti[4] : pos[1], DM(idt, vdw[1]));
      tr[2] = (sd[4] == 0) ? ti[2] : DA(yaw, DM(idt, sd[4]));
    }
    for (int j = 0; j < 12; j++) f[54 + 12 * st + j] = (float)tr[j];
  }
  unsigned char* g = records + (size_t)i * rec_stride + (54 + 12 * N) * 4;
  for (int e = 0; e < 2 * N; e++) g[e] = gait[e];
  for (int e = (54 + 12 * N) * 4 + 2 * N; e < rec_stride; e++) records[(size_t)i * rec_stride + e] = 0;
}

// The reference trajectory (:331-399) of one command into out [12N]: R the body -> world rotation, pos and rpy the state's,
// sd (roll, pitch, body vx, vy, yaw rate) and wpd [2] the command (hmpc_state_t::state_des, world_position_desired).  The
// operations of hmpc_prepare_kernel's trajectory block, one for one and explicitly rounded, so a candidate's trajectory is
// the traj that kernel writes for a state with that command, bit for bit.  (hmpc_prepare_kernel keeps its own inline copy:
// calling this function from it changed that kernel's register assignment and instruction schedule.)
__device__ __forceinline__ void prepare_traj(const double* R, const double* pos, const double* rpy, const double* sd,
                                             const double* wpd, int N, double dtMPC, float* out)
{
  const double yaw = rpy[2];
  const double vdr[3] = {sd[2], sd[3], 0.0};
  double vdw[3];
  for (int a = 0; a < 3; a++) vdw[a] = DA(DA(DM(R[a * 3], vdr[0]), DM(R[a * 3 + 1], vdr[1])), DM(R[a * 3 + 2], vdr[2]));
  const double mpe = .05;
  double xS = wpd[0], yS = wpd[1];
  if (DS(xS, pos[0]) > mpe) xS = DA(pos[0], mpe);
  if (DS(pos[0], xS) > mpe) xS = DS(pos[0], mpe);
  if (DS(yS, pos[1]) > mpe) yS = DA(pos[1], mpe);
  if (DS(pos[1], yS) > mpe) yS = DS(pos[1], mpe);
  const double ti[12] = {sd[0], sd[1], 0.0, xS, yS, 0.55, 0, 0, sd[4], vdw[0], vdw[1], 0};
  for (int st = 0; st < N; st++) {
    double tr[12];
    for (int j = 0; j < 12; j++) tr[j] = ti[j];
    if (st == 0) {
      tr[0] = rpy[0]; tr[1] = rpy[1]; tr[2] = rpy[2];
      tr[3] = pos[0]; tr[4] = pos[1]; tr[5] = pos[2];
    } else {
      const double idt = DM((double)st, dtMPC);
      tr[3] = DA(vdw[0] == 0 ? ti[3] : pos[0], DM(idt, vdw[0]));
      tr[4] = DA(vdw[1] == 0 ? ti[4] : pos[1], DM(idt, vdw[1]));
      tr[2] = (sd[4] == 0) ? ti[2] : DA(yaw, DM(idt, sd[4]));
    }
    for (int j = 0; j < 12; j++) out[12 * st + j] = (float)tr[j];
  }
}

// The trajectories of a multi-command states call (hmpc_solve_states_device_multi): for each robot the chain's
// hmpc_prepare_kernel prepares, the reference trajectories of its K commands cmd[i][k] (hmpc_command_t: 7 doubles, laid out
// like the state's bytes [256, 312)) into traj[i][k] [12N].  One thread per (robot, candidate); `list` / `count` as in
// hmpc_prepare_kernel, with K threads per list entry.  Launch shape: hmpc_chain.h, prepare_grid(batch * K).
__global__ void hmpc_prepare_traj_kernel(const unsigned char* states, int batch, int K, const double* cmd, int N, double dtMPC,
                                         float* traj, const int* list, const int* count)
{
  pdl_trigger();  // class 0 may become resident; it waits for this kernel before it reads the trajectories
  pdl_wait();     // (the list, and the previous call's readers of traj, as in hmpc_prepare_kernel)
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (list ? *count : batch) * K) return;
  const int e = t / K, k = t % K;
  const int i = list ? list[e] : e;
  const double* s = reinterpret_cast<const double*>(states + (size_t)i * 352);
  const double e0 = s[6], e1 = s[7], e2 = s[8], e3 = s[9];  // the quaternion: hmpc_prepare_kernel's body -> world rotation
  const double R[9] = {DS(1.0, DM(2.0, DA(DM(e2, e2), DM(e3, e3)))), DM(2.0, DS(DM(e1, e2), DM(e0, e3))), DM(2.0, DA(DM(e1, e3), DM(e0, e2))),
                       DM(2.0, DA(DM(e1, e2), DM(e0, e3))), DS(1.0, DM(2.0, DA(DM(e1, e1), DM(e3, e3)))), DM(2.0, DS(DM(e2, e3), DM(e0, e1))),
                       DM(2.0, DS(DM(e1, e3), DM(e0, e2))), DM(2.0, DA(DM(e2, e3), DM(e0, e1))), DS(1.0, DM(2.0, DA(DM(e1, e1), DM(e2, e2))))};
  const size_t q = (size_t)i * K + k;
  prepare_traj(R, s, s + 13, cmd + q * 7, cmd + q * 7 + 5, N, dtMPC, traj + q * 12 * N);
}

// ------------------------------------------------------------------------------------------------
// row f-3: advance every robot by one MPC tick after a solve (one thread per robot, plain fp64).
//   states  hmpc_state_t [batch] (352 B)      loop  hmpc_rollout_t [batch] (80 B)
//   wrench  float [batch][12N] (solution)      status int [batch]
// Plant: the single rigid body of SolverMPC.cpp:312-331 integrated with forward Euler (SolverMPC.cpp:145-146), feet
// pinned in the world.  Gait: GaitGenerator.cpp:85-103.  Touch-down placement: ConvexMPCLocomotion.cpp:119-160.
// ------------------------------------------------------------------------------------------------
__device__ inline int gait_contact(int it, int N, int offset, int duration)
{
  int progress = it % N - offset;
  if (progress < 0) progress += N;
  return progress < duration ? 1 : 0;
}
__device__ inline void quat_to_R_f64(const double* qt, double* R)
{
  const double e0 = qt[0], e1 = qt[1], e2 = qt[2], e3 = qt[3];
  R[0] = DS(1.0, DM(2.0, DA(DM(e2, e2), DM(e3, e3)))); R[1] = DM(2.0, DS(DM(e1, e2), DM(e0, e3))); R[2] = DM(2.0, DA(DM(e1, e3), DM(e0, e2)));
  R[3] = DM(2.0, DA(DM(e1, e2), DM(e0, e3))); R[4] = DS(1.0, DM(2.0, DA(DM(e1, e1), DM(e3, e3)))); R[5] = DM(2.0, DS(DM(e2, e3), DM(e0, e1)));
  R[6] = DM(2.0, DS(DM(e1, e3), DM(e0, e2))); R[7] = DM(2.0, DA(DM(e2, e3), DM(e0, e1))); R[8] = DS(1.0, DM(2.0, DA(DM(e1, e1), DM(e2, e2))));
}
__global__ void hmpc_advance_kernel(unsigned char* states, unsigned char* loop, int batch, int N, double dtMPC,
                                    const float* wrench, const int* status, float* wrench_log)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch) return;
  double* s = reinterpret_cast<double*>(states + (size_t)i * 352);
  unsigned char* gait = states + (size_t)i * 352 + 39 * 8;
  double* feet = reinterpret_cast<double*>(loop + (size_t)i * 80);
  int* li = reinterpret_cast<int*>(loop + (size_t)i * 80 + 48);  // offset[2] duration[2] iteration failures iters ticks
  double* pos = s; double* vw = s + 3; double* qt = s + 6; double* ow = s + 10; double* rpy = s + 13;
  double* lp = s + 26; const double* sd = s + 32; double* wpd = s + 37;
  double u[12];
  for (int k = 0; k < 12; k++) u[k] = (double)wrench[(size_t)i * 12 * N + k];
  if (wrench_log) for (int k = 0; k < 12; k++) wrench_log[(size_t)i * 12 + k] = wrench[(size_t)i * 12 * N + k];
  const int stw = status[i];
  li[5] += ((stw & 0xFF) != 0);
  li[6] += (stw >> 8) & 0xFFF;
  li[7] += 1;
  double R[9];
  quat_to_R_f64(qt, R);
  // commanded velocity in the world and the position set-point (ConvexMPCLocomotion.cpp:46-56, 338-346)
  double vdw[3];
  for (int a = 0; a < 3; a++) vdw[a] = R[a * 3] * sd[2] + R[a * 3 + 1] * sd[3];
  for (int a = 0; a < 2; a++) {
    double w = wpd[a];
    if (w - pos[a] > 0.05) w = pos[a] + 0.05;
    if (pos[a] - w > 0.05) w = pos[a] - 0.05;
    wpd[a] = w + dtMPC * vdw[a];
  }
  // rigid body: torque about the CoM and net force of the two foot wrenches [F0 F1 M0 M1]
  double tq[3] = {u[6] + u[9], u[7] + u[10], u[8] + u[11]};
  for (int leg = 0; leg < 2; leg++) {
    const double rx = feet[3 * leg] - pos[0], ry = feet[3 * leg + 1] - pos[1], rz = feet[3 * leg + 2] - pos[2];
    const double fx = u[3 * leg], fy = u[3 * leg + 1], fz = u[3 * leg + 2];
    tq[0] += ry * fz - rz * fy;
    tq[1] += rz * fx - rx * fz;
    tq[2] += rx * fy - ry * fx;
  }
  // world inertia R I R^T and its inverse applied to the torque:  I_w^-1 tq = R I^-1 R^T tq
  const double Iinv[3] = {1.0 / 0.5413, 1.0 / 0.5200, 1.0 / 0.0691};  // RobotState.cpp:45
  double tb[3], dw[3];
  for (int a = 0; a < 3; a++) tb[a] = (R[a] * tq[0] + R[3 + a] * tq[1] + R[6 + a] * tq[2]) * Iinv[a];
  for (int a = 0; a < 3; a++) dw[a] = R[a * 3] * tb[0] + R[a * 3 + 1] * tb[1] + R[a * 3 + 2] * tb[2];
  // Euler-angle rates: rpy' = E^-1 omega, E = [[cy cp, -sy, 0], [sy cp, cy, 0], [-sp, 0, 1]]
  double sy, cy, sp, cp;
  sincos(rpy[2], &sy, &cy);
  sincos(rpy[1], &sp, &cp);
  const double a0 = (cy * ow[0] + sy * ow[1]) / cp;     // roll rate
  const double a1 = -sy * ow[0] + cy * ow[1];           // pitch rate
  const double a2 = ow[2] + sp * a0;                    // yaw rate
  const double mass = 9.0;                              // SolverMPC.cpp:423
  const double nrpy[3] = {rpy[0] + dtMPC * a0, rpy[1] + dtMPC * a1, rpy[2] + dtMPC * a2};
  const double np_[3] = {pos[0] + dtMPC * vw[0], pos[1] + dtMPC * vw[1], pos[2] + dtMPC * vw[2]};
  const double nw[3] = {ow[0] + dtMPC * dw[0], ow[1] + dtMPC * dw[1], ow[2] + dtMPC * dw[2]};
  const double nv[3] = {vw[0] + dtMPC * ((u[0] + u[3]) / mass), vw[1] + dtMPC * ((u[1] + u[4]) / mass),
                        vw[2] + dtMPC * ((u[2] + u[5]) / mass - 9.81)};
  for (int a = 0; a < 3; a++) { rpy[a] = nrpy[a]; pos[a] = np_[a]; ow[a] = nw[a]; vw[a] = nv[a]; }
  // orientation quaternion of the new Euler angles (ori::rpyToQuat: yaw * pitch * roll)
  double sr, cr, spp, cpp, syy, cyy;
  sincos(nrpy[0] * 0.5, &sr, &cr);
  sincos(nrpy[1] * 0.5, &spp, &cpp);
  sincos(nrpy[2] * 0.5, &syy, &cyy);
  qt[0] = cyy * cpp * cr + syy * spp * sr;
  qt[1] = cyy * cpp * sr - syy * spp * cr;
  qt[2] = cyy * spp * cr + syy * cpp * sr;
  qt[3] = syy * cpp * cr - cyy * spp * sr;
  quat_to_R_f64(qt, R);
  // next tick's contact table; a leg that goes swing -> stance is placed
  const int it = li[4] + 1;
  li[4] = it;
  for (int leg = 0; leg < 2; leg++) {
    const int was = gait[leg];
    const int now = gait_contact(it, N, li[leg], li[2 + leg]);
    if (!was && now) {
      const double hip[3] = {-0.005, leg == 0 ? -0.057 : 0.057, -0.126};
      const double stance_t = 0.5 * (double)li[2 + leg] * dtMPC;
      for (int a = 0; a < 2; a++) {
        double rel = nv[a] * stance_t + 0.02 * (nv[a] - vdw[a]);
        rel = fmin(fmax(rel, -0.4), 0.4);
        feet[3 * leg + a] = np_[a] + R[a * 3] * hip[0] + R[a * 3 + 1] * hip[1] + R[a * 3 + 2] * hip[2] + rel;
      }
      feet[3 * leg + 2] = 0.0;
    }
  }
  for (int st = 0; st < N; st++)
    for (int leg = 0; leg < 2; leg++) gait[2 * st + leg] = (unsigned char)gait_contact(it + st, N, li[leg], li[2 + leg]);
  // leg-frame foot positions the next preparation will read: p = rBody (pFoot - position) - hip
  for (int leg = 0; leg < 2; leg++) {
    const double hip[3] = {-0.005, leg == 0 ? -0.057 : 0.057, -0.126};
    const double d0 = feet[3 * leg] - np_[0], d1 = feet[3 * leg + 1] - np_[1], d2 = feet[3 * leg + 2] - np_[2];
    for (int a = 0; a < 3; a++) lp[3 * leg + a] = R[a] * d0 + R[3 + a] * d1 + R[6 + a] * d2 - hip[a];
  }
}

// ------------------------------------------------------------------------------------------------
// row f-4: the swing-leg controller, one thread per robot (swingLegController::updateSwingLeg,
// src/common/SwingLegController.cpp:46-219; Gait::getSwingSubPhase, GaitGenerator.cpp:54-80; Bezier swing trajectory,
// FootSwingTrajectory.cpp:17-36 + Interpolation.h:53-74).  fp64 with explicitly rounded operations in the reference's
// order (no FMA contraction), so the only differences to the CPU restatement are the last bits of asin/acos.
//   states hmpc_state_t (352 B)   loop hmpc_rollout_t (80 B)   swing hmpc_swing_t (72 B)   cmd hmpc_swing_cmd_t (232 B)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double bezier_f64(double y0, double yf, double x)
{
  const double b = DA(DM(DM(x, x), x), DM(3.0, DM(DM(x, x), DS(1.0, x))));
  return DA(y0, DM(b, DS(yf, y0)));
}
__device__ __forceinline__ double clamp_f64(double v, double lo, double hi) { return fmax(lo, fmin(v, hi)); }
__device__ __forceinline__ double dot3_rn(double a0, double b0, double a1, double b1, double a2, double b2)
{
  return DA(DA(DM(a0, b0), DM(a1, b1)), DM(a2, b2));
}
__global__ void hmpc_swing_kernel(const unsigned char* states, const unsigned char* loop, const double* phase,
                                  unsigned char* swing, int batch, int n_iterations, double dt, double dtSwing,
                                  unsigned char* cmd)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch) return;
  const double* s = reinterpret_cast<const double*>(states + (size_t)i * 352);
  const double* pos = s; const double* vw = s + 3; const double* qt = s + 6;
  const double* lq = s + 16; const double* lp = s + 26; const double* sd = s + 32;
  const int* li = reinterpret_cast<const int*>(loop + (size_t)i * 80 + 48);  // offset[2] duration[2] ...
  double* sw_p0 = reinterpret_cast<double*>(swing + (size_t)i * 72);
  double* sw_time = sw_p0 + 6;
  int* sw_first = reinterpret_cast<int*>(swing + (size_t)i * 72 + 64);
  double* out = reinterpret_cast<double*>(cmd + (size_t)i * 232);  // pf[6] p_des[6] v_des[6] q_des[10] | swing[2]
  int* out_swing = reinterpret_cast<int*>(cmd + (size_t)i * 232 + 224);
  for (int k = 0; k < 28; k++) out[k] = 0.0;
  out_swing[0] = out_swing[1] = 0;
  double R[9];  // body -> world; rBody = R^T
  quat_to_R_f64(qt, R);
  const double hipy[2] = {-0.057, 0.057};
  // updateFootPosition (:61-70)
  double pfw[2][3];
  for (int leg = 0; leg < 2; leg++) {
    const double hp0 = DA(-0.005, lp[3 * leg]), hp1 = DA(hipy[leg], lp[3 * leg + 1]), hp2 = DA(-0.126, lp[3 * leg + 2]);
    for (int a = 0; a < 3; a++) pfw[leg][a] = DA(pos[a], dot3_rn(R[a * 3], hp0, R[a * 3 + 1], hp1, R[a * 3 + 2], hp2));
    pfw[leg][2] = 0.0;
  }
  // Gait::getSwingSubPhase (GaitGenerator.cpp:54-80)
  double sst[2];
  for (int leg = 0; leg < 2; leg++) {
    const double offp = __ddiv_rn((double)li[leg], (double)n_iterations);
    const double durp = __ddiv_rn((double)li[2 + leg], (double)n_iterations);
    double so = DA(offp, durp);
    if (so > 1) so = DS(so, 1.);
    const double sdur = DS(1., durp);
    double pr = DS(phase[i], so);
    if (pr < 0) pr = DA(pr, 1.);
    if (pr > sdur) pr = 0.;
    else pr = __ddiv_rn(pr, sdur);
    sst[leg] = pr;
  }
  const int g_stance = li[2], g_swing = n_iterations - li[2];
  // updateSwingTimes (:82-93)
  for (int leg = 0; leg < 2; leg++) {
    if (sw_first[leg]) {
      sw_time[leg] = DM(dtSwing, (double)g_swing);
    } else {
      sw_time[leg] = DS(sw_time[leg], dt);
      if (sw_time[leg] <= 0) sw_first[leg] = 1;
    }
  }
  // computeFootPlacement (:98-128)
  double vdw[3];
  for (int a = 0; a < 3; a++) vdw[a] = dot3_rn(R[a * 3], sd[2], R[a * 3 + 1], sd[3], R[a * 3 + 2], 0.0);
  double Pf[2][3];
  for (int leg = 0; leg < 2; leg++) {
    for (int a = 0; a < 3; a++)
      Pf[leg][a] = DA(DA(pos[a], dot3_rn(R[a * 3], -0.005, R[a * 3 + 1], hipy[leg], R[a * 3 + 2], -0.126)), DM(vw[a], sw_time[leg]));
    for (int a = 0; a < 2; a++) {
      const double rel = DA(DM(DM(DM(DM(1.75, vw[a]), 0.5), (double)g_stance), dtSwing), DM(0.1, DS(vw[a], vdw[a])));
      const float relf = fminf(fmaxf((float)rel, -(float)0.3), (float)0.3);  // float clamp as written (:117-118)
      Pf[leg][a] = DA(Pf[leg][a], (double)relf);
    }
    Pf[leg][2] = 0.0;
    for (int a = 0; a < 3; a++) out[3 * leg + a] = Pf[leg][a];
  }
  // computeFootDesiredPosition (:134-155) + computeIK (:160-193)
  const double PI = 3.14159265358979323846;  // M_PI
  for (int leg = 0; leg < 2; leg++) {
    if (!(sst[leg] > 0)) continue;
    out_swing[leg] = 1;
    if (sw_first[leg]) {
      sw_first[leg] = 0;
      for (int a = 0; a < 3; a++) sw_p0[3 * leg + a] = pfw[leg][a];
    }
    const double ph = sst[leg], height = 0.15;
    const double* p0 = sw_p0 + 3 * leg;
    double pd[3];
    for (int a = 0; a < 2; a++) pd[a] = bezier_f64(p0[a], Pf[leg][a], ph);
    pd[2] = (ph < 0.5) ? bezier_f64(p0[2], DA(p0[2], height), DM(ph, 2.0)) : bezier_f64(DA(p0[2], height), Pf[leg][2], DS(DM(ph, 2.0), 1.0));
    const double side_w = (leg == 1) ? 1.0 : -1.0;
    const double hoff[3] = {-0.015, DM(side_w, -0.055), 0.0};
    const double d0 = DS(pd[0], pos[0]), d1 = DS(pd[1], pos[1]), d2 = DS(pd[2], pos[2]);
    double pb[3];
    for (int a = 0; a < 3; a++) {  // rBody = R^T: row a of rBody = column a of R
      pb[a] = DA(dot3_rn(R[a], d0, R[3 + a], d1, R[6 + a], d2), hoff[a]);
      out[6 + 3 * leg + a] = pb[a];
      out[12 + 3 * leg + a] = dot3_rn(R[a], DS(0.0, vw[0]), R[3 + a], DS(0.0, vw[1]), R[6 + a], DS(0.0, vw[2]));
    }
    const double side = (leg == 0) ? -1.0 : 1.0;
    const double f0 = DS(pb[0], DS(0.0465, 0.06)), f1 = DS(pb[1], 0.0), f2 = DS(pb[2], DA(-0.126, DM(-0.0705, 2.0)));
    const double d3 = sqrt(DA(DA(DM(f0, f0), DM(f1, f1)), DM(f2, f2)));
    const double dyz = sqrt(DA(DM(f1, f1), DM(f2, f2)));
    const double dh = 0.0205;
    const double dv_ = sqrt(fmax(0.00001, DS(DM(dyz, dyz), DM(dh, dh))));
    const double dxz = sqrt(DS(DM(d3, d3), DM(dh, dh)));
    const double a1 = clamp_f64(__ddiv_rn(dxz, DM(2.0, 0.22)), -1.0, 1.0);
    const double a2 = clamp_f64(__ddiv_rn(dv_, dxz), -1.0, 1.0);
    double divisor = fabs(f0);
    divisor = (divisor == 0.0) ? 1e-6 : divisor;
    double* q = out + 18 + 5 * leg;
    q[0] = 0.0;
    q[1] = DA(asin(clamp_f64(__ddiv_rn(f1, dyz), -1.0, 1.0)), asin(clamp_f64(__ddiv_rn(DM(dh, side), dyz), -1.0, 1.0)));
    q[2] = DS(acos(a1), __ddiv_rn(DM(acos(a2), f0), divisor));
    q[3] = DS(DM(2.0, asin(clamp_f64(__ddiv_rn(__ddiv_rn(dxz, 2.0), 0.22), -1.0, 1.0))), PI);
    q[4] = DS(-lq[5 * leg + 3], lq[5 * leg + 2]);
    q[2] = DS(q[2], DM(0.3, PI));
    q[3] = DA(q[3], DM(0.6, PI));
    q[4] = DS(q[4], DM(0.3, PI));
  }
}

// ------------------------------------------------------------------------------------------------
// the kernel.  NT threads = NT/32 warps: warp w owns tile rows w and NT8-1-w of the sweep, thread e owns
// constraint row e in the active-set iterations and thread NT-1-i owns variable i.
// NF > 0 fixes the horizon at compile time (layout offsets and loop bounds fold), NF == 0 reads it from
// the arguments; CLS = size class (capacity N or 2N blocks of 6 variables), or 3: the refinement class (runtime layout from
// refine_layout; it refines the final KKT solution against the stored Hessian, see the end of stage 5).
// ------------------------------------------------------------------------------------------------
// Profiling hooks (hmpc_debug_set_clock_buffer): HMPC_STAMP(i) = clock of thread 0 at point i (tests/tools/gpu_check.py).
// Built with -DHMPC_WARP_STAMPS=<k> instead, lane 0 of EVERY warp stamps the phases of block step k of stage 4
// (tests/tools/warp_stamps.py: which warp reaches the step's barrier last, and what it did before).
#ifdef HMPC_WARP_STAMPS
#define HMPC_STAMP(i) do { } while (0)
#define HMPC_WSTAMP(e) do { if (ka.dbg_clk && lane == 0 && wid < 4 && k == HMPC_WARP_STAMPS) ka.dbg_clk[(size_t)inst * 32 + wid * 8 + (e)] = clock64(); } while (0)
#else
#define HMPC_STAMP(i) do { if (ka.dbg_clk && tid == 0) ka.dbg_clk[(size_t)inst * 32 + (i)] = clock64(); } while (0)
#define HMPC_WSTAMP(e) do { } while (0)
#endif
constexpr int WS_STATE_INTS = 40;  // persistent working set of one robot: [0] = count, then (step*2+leg) << 8 | normal index

// A multi-query list entry: the robot, and its candidates [mq_first, mq_end).  Robots only (class 0), or candidates i*K + k and
// whole robots -1 - i (the later classes: `items`).
__device__ __forceinline__ int mq_robot(int ent, int K, bool items) { return !items ? ent : (ent < 0 ? -1 - ent : ent / K); }
__device__ __forceinline__ int mq_first(int ent, int K, bool items) { return (items && ent >= 0) ? ent % K : 0; }
__device__ __forceinline__ int mq_end(int ent, int K, bool items) { return (items && ent >= 0) ? ent % K + 1 : K; }

// MQ (multi-query, hmpc_solve_device_multi): a CTA takes a robot through stages 0-4 once and then runs the rest of the solve
// (the trajectory's d rows of stage 2, the gradient, stages 5-6) once per candidate trajectory k, into result row i*K + k.
// The list of class 0 (or its identity) holds robots; the lists of classes 1-2 and of the refinement class hold candidates
// i*K + k (escalated alone) or -1 - i (a robot class 0 classified out, with all K candidates).
template <int NT, int MINB, int NF, int CLS, bool MQ = false>
__global__ void __launch_bounds__(NT, MINB) hmpc_solve_kernel(const KernelArgs ka)
{
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x;
  const int lane = tid & 31, wid = tid >> 5;
  constexpr int NW = NT / 32;
  constexpr bool FIX = NF > 0;
  const int N = FIX ? NF : ka.horizon;
  const int nb_cap = FIX ? class_nb_cap(NF, CLS) : ka.nb_cap;
  const int qmax = FIX ? class_qmax(NF > 0 ? NF : 1, CLS) : ka.qmax;
  const int rec_stride = FIX ? record_stride(NF) : ka.rec_stride;
  const int tcap = FIX ? class_tcap(NF > 0 ? NF : 1, CLS) : ka.tcap;
  Layout L;
  if constexpr (FIX) {
    constexpr Layout LC = class_layout(NF, CLS, NW);
    L = LC;
  } else {
    L = ka.L;
  }
  const bool dump = (ka.dbg_H != nullptr);

  float* Hf = reinterpret_cast<float*>(smem + L.H);     // assembly: float32 Hessian tiles
  double* Hd = reinterpret_cast<double*>(smem + L.H);   // after the sweep: float64 inverse tiles
  double* gq = reinterpret_cast<double*>(smem + L.gq);
  double* x0 = reinterpret_cast<double*>(smem + L.x0);
  double* nrm = reinterpret_cast<double*>(smem + L.nrm);  // [leg*10+type][6]
  double* fz = reinterpret_cast<double*>(smem + L.fz);    // [block] f_max * gait
  int* blk_sl = reinterpret_cast<int*>(smem + L.blk);     // block -> step*2+leg
  int* sl_blk = blk_sl + nb_cap;                          // step*2+leg -> block or -1
  unsigned* redk = reinterpret_cast<unsigned*>(smem + L.misc);   // [32] warp partial keys
  int* redi = reinterpret_cast<int*>(smem + L.misc + 128);       // [32] warp partial indices
  double* redv = reinterpret_cast<double*>(smem + L.misc + 256); // [16] warp partial values
  // [0]=NB [1]=stance0 [2]=stance1 [3]=code [4]=decision [5]=dropped row [6]=ncomb [7]=free slot [8]=slots in use (step) [9]=slots in use (now)
  int* flags = reinterpret_cast<int*>(smem + L.misc + 384);
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + L.misc + 448);
  double* dsc = reinterpret_cast<double*>(smem + L.misc + 456);    // [0] step length, [1] refreshed slack of the entering row
  unsigned* amask = reinterpret_cast<unsigned*>(smem + L.misc + 480);  // [8] slots in use (bit set)

  double* T = reinterpret_cast<double*>(smem + L.T);
  double* Sv = reinterpret_cast<double*>(smem + L.Sv);
  double* lam = reinterpret_cast<double*>(smem + L.lam);
  double* dvs = reinterpret_cast<double*>(smem + L.dv);
  double* rr = reinterpret_cast<double*>(smem + L.rr);
  int* wsl = reinterpret_cast<int*>(smem + L.wsl);
  double* zb = reinterpret_cast<double*>(smem + L.zb);

  unsigned char* rec = smem + L.rec;
  const float* rf = reinterpret_cast<const float*>(rec);
  float* x0f = reinterpret_cast<float*>(smem + L.x0f);
  float* Acd = reinterpret_cast<float*>(smem + L.Acd);
  float* Bcd = reinterpret_cast<float*>(smem + L.Bcd);
  float* Mb = reinterpret_cast<float*>(smem + L.M);    // [N][6][12]: rows 0..5 of P_d*Bcd (6..11 equal Bcd's), columns grouped by leg
  float* dd = reinterpret_cast<float*>(smem + L.dd);   // [N][12]
  float* Fblk = reinterpret_cast<float*>(smem + L.fbl);
  int* comb = reinterpret_cast<int*>(smem + L.comb);   // stage-3 work list

  pdl_trigger();  // the next class's kernel may become resident while this one works
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  uint32_t phase = 0;
  pdl_wait();     // counts / lists / records come from the kernels before this one
  // the list lengths of the NEXT call (the other parity) are cleared here: every kernel of the previous call, which
  // used them, completed before pdl_wait() returned, and this call only touches its own (word 4: the refinement class's)
  if (ka.counts_next && blockIdx.x == 0 && tid < 5) ka.counts_next[tid] = 0;
  const int count = ka.list ? ka.counts[ka.cls] : ka.batch;

  // Batches of more than two waves: the resident CTAs start every wave together (a bounded global barrier between
  // waves).  All CTAs of an SM then execute the same stage at the same time and share the instruction cache lines of this
  // ~190 KB kernel; drifting apart, warps in different stages thrash it.  With two waves the second one is partial and
  // waiting for the slowest robot of the first costs more than it saves (DESIGN.md §3).  The wait is bounded: a CTA that
  // is not joined within 400 k cycles (something else holds SMs) stops waiting for good — lockstep is an optimisation, not
  // a dependency.
  const int trips = (count + (int)gridDim.x - 1) / (int)gridDim.x;
  bool lockstep = ka.wave_sync != nullptr && trips > 2;
  for (int trip = 0; trip < trips; trip++) {
    const int idx = blockIdx.x + trip * gridDim.x;
    if (lockstep && trip > 0) {
      if (tid == 0) {
        __threadfence();
        atomicAdd(ka.wave_sync, 1u);
        const unsigned target = (unsigned)trip * gridDim.x;
        const long long t0 = clock64();
        bool ok = true;
        while (atomicAdd(ka.wave_sync, 0u) < target) {
          if (clock64() - t0 > 400000ll) { ok = false; break; }
        }
        flags[15] = ok ? 1 : 0;
      }
      __syncthreads();
      if (!flags[15]) lockstep = false;
      __syncthreads();
    }
    if (idx >= count) continue;  // the last wave may not fill the grid
    // the robot (its record) and its candidates [k0, k1); one solve for every other launch
    const int inst = MQ ? mq_robot(ka.list ? ka.list[idx] : idx, ka.mq_k, CLS == 3 || ka.cls > 0)
                        : (ka.list ? ka.list[idx] : idx);
    const int k0 = MQ ? mq_first(ka.list ? ka.list[idx] : idx, ka.mq_k, CLS == 3 || ka.cls > 0) : 0;
    const int k1 = MQ ? mq_end(ka.list ? ka.list[idx] : idx, ka.mq_k, CLS == 3 || ka.cls > 0) : 1;
    HMPC_STAMP(0);
    // ---------------- stage 0: record -> shared memory (TMA bulk copy) ----------------
    const bool raw = ka.raw_records != nullptr;
    if (raw) {
      // in-place mode: gather the live pieces of the reference record (convexMPC_interface.h:19-37; 8-byte aligned,
      // so no bulk copy) into the packed layout with 8-byte loads: p..weights | Alpha_K | traj | gait
      const unsigned char* src = ka.raw_records + (size_t)inst * 3016;
      const int nt = 6 * N, ng = (2 * N + 7) / 8;
      for (int e = tid; e < 27 + nt + ng; e += NT) {
        int so, dw;  // source byte offset, destination 8-byte word
        if (e < 21) { so = 8 * e; dw = e; }
        else if (e < 27) { so = 1896 + 8 * (e - 21); dw = e; }
        else if (e < 27 + nt) { so = 168 + 8 * (e - 27); dw = e; }
        else { so = 1944 + 8 * (e - 27 - nt); dw = e; }
        reinterpret_cast<uint2*>(rec)[dw] = *reinterpret_cast<const uint2*>(src + so);
      }
    } else if (tid == 0) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // earlier generic-proxy use of the union
      mbar_expect_tx(bar, (uint32_t)rec_stride);
      bulk_g2s(rec, ka.records + (size_t)inst * rec_stride, (uint32_t)rec_stride, bar);
    }
    if (raw) {
      __syncthreads();
    } else {
      mbar_wait(bar, phase);
      phase ^= 1;
    }

    // ---------------- contact table -> reduced block list (SolverMPC.cpp:589-637) ----------------
    const unsigned char* gait = rec + (54 + 12 * N) * 4;
    if (wid == 0) {
      bool stance = false;
      if (lane < 2 * N) {
        const float ub = FM(ka.f_max, (float)gait[lane]);
        stance = !(ub < 0.0001f && ub > -0.0001f) || dump;  // swing <=> near_zero(lb) && near_zero(ub); lb == 0
      }
      const unsigned mask = __ballot_sync(0xffffffffu, stance);
      const int k = __popc(mask & ((1u << lane) - 1u));
      if (lane < 2 * N) {
        sl_blk[lane] = (stance && k < nb_cap) ? k : -1;
        if (stance && k < nb_cap) {
          blk_sl[k] = lane;
          fz[k] = (double)FM(ka.f_max, (float)gait[lane]);
        }
      }
      unsigned st0 = 0, st1 = 0;
      for (int s = 0; s < N; s++) {
        st0 |= ((mask >> (2 * s)) & 1u) << s;
        st1 |= ((mask >> (2 * s + 1)) & 1u) << s;
      }
      // stage-3 work list: (li, lj, delta) combinations that own at least one wanted H block, sorted by chain
      // length (longest first) so that the 32 items a warp runs in lockstep have similar trip counts
      int ncomb = 0;
      {
        int pk[2], km[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int c = 32 * h + lane;
          const int li = (c / N) >> 1, lj = (c / N) & 1, delta = c % N;
          unsigned need = 0;
          if (c < 4 * N) need = (li ? st1 : st0) & ((lj ? st1 : st0) >> delta);
          km[h] = need ? N - 1 - delta - (__ffs(need) - 1) : -1;
          pk[h] = li | (lj << 1) | (delta << 2) | (km[h] << 8);
        }
        const unsigned lt = (1u << lane) - 1u;
        for (int v = N - 1; v >= 0; v--) {
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const unsigned has = __ballot_sync(0xffffffffu, km[h] == v);
            if (km[h] == v) comb[ncomb + __popc(has & lt)] = pk[h];
            ncomb += __popc(has);
          }
        }
      }
      if (lane == 0) {
        flags[0] = __popc(mask);
        flags[1] = (int)st0;
        flags[2] = (int)st1;
        flags[3] = ST_OK;
        flags[6] = ncomb;
      }
    }
    // ---------------- stage 1: prologue, three roles on the other warps (beside the block list on warp 0) ----------------
    if (tid < 14) reinterpret_cast<float*>(smem + L.keep)[tid] = (tid < 10) ? rf[19 + tid] : rf[6 + tid - 10];
    {
      constexpr int WL = (NW > 3) ? 3 : 0, W1 = (NW > 1) ? 1 : 0, W2 = (NW > 2) ? 2 : 0;
      unsigned char* scr = smem + L.P;  // 432 bytes of role scratch
      // every role zeroes the sparse fp32 operand it fills (no barrier separates the roles from earlier code)
      if (wid == WL) {
        for (int e = lane; e < 192; e += 32) Fblk[e] = 0.f;
        __syncwarp();
        role_leg(rf, lane, Fblk, scr);
      }
      if (wid == W1) {
        for (int e = lane; e < 169; e += 32) Acd[e] = 0.f;
        __syncwarp();
        role_state(rf, ka.dt, x0f, Acd, lane, scr + 256);
      }
      if (wid == W2) {
        for (int e = lane; e < 156; e += 32) Bcd[e] = 0.f;
        __syncwarp();
        if (lane == 31) role_inertia(rf, ka.dt, Bcd);
      }
    }
    __syncthreads();
    const int NB = flags[0];
    if constexpr (CLS == 3) {
      if (NB > nb_cap) {  // more stance blocks than the refinement class holds: the handing class's code 4 stands
        __syncthreads();
        continue;
      }
    }
    if (ka.split_nb >= 0 && NB > ka.split_nb) {
      // size classification folded into the launch: more stance blocks than this class holds -> next class's list
      if (tid == 0) {
        const int slot = atomicAdd(&ka.counts[ka.cls + 1], 1);
        ka.esc_list[slot] = MQ ? -1 - inst : inst;  // (multi-query: the robot with all its candidates)
      }
      __syncthreads();
      continue;
    }
    const int n = 6 * NB, m = 10 * NB;
    const int NT8 = (n + 7) >> 3;
    const unsigned stmask[2] = {(unsigned)flags[1], (unsigned)flags[2]};

    for (int e = n + tid; e < 8 * NT8; e += NT) gq[e] = 0.0;  // tile padding of the gradient
    __syncthreads();

    // constraint normals (fp64 copies of the fp32 rows), "c'x >= d" form:
    // t0-3 friction (lower), t4/t5 Mx lower/upper, t6/t7 line contact (upper), t8/t9 Fz lower/upper
    for (int e = tid; e < 2 * 10 * 6; e += NT) {
      const int leg = e / 60, t = (e / 6) % 10, c = e % 6;
      const int col = col12_of(leg, c);
      const int row = (t < 5) ? t : (t == 5 ? 4 : (t < 8 ? t - 1 : 7));
      const bool neg = (t == 5 || t == 6 || t == 7 || t == 9);
      const float v = Fblk[(8 * leg + row) * 12 + col];
      nrm[e] = (double)(neg ? -v : v);
    }

    // Multi-query: everything below runs once per candidate kq (the jump back at the end); stages 2-4 skip what does not
    // depend on the trajectory after the first (the powers and Toeplitz blocks, H, the sweep), and H^-1 survives in place.
    float* const mqs = MQ ? ka.mq_scratch + (size_t)blockIdx.x * mq_scratch_floats(N) : nullptr;
    bool illc_h = false;  // the conditioning check of stage 5 (it reads the diagonal of H, which the first candidate spends)
    int kq = k0;
  next_candidate:
    const bool first = kq == k0;
    const int row = MQ ? inst * ka.mq_k + kq : inst;  // result row
    const float* trj = MQ ? ka.mq_traj + (size_t)row * 12 * N : nullptr;  // the candidate's reference trajectory
    if (MQ && !first) {
      // the stage-2 operands and the weights, back from the scratch into the union (the previous candidate's stage 5 used it)
      float* wts = reinterpret_cast<float*>(rec) + 30;
      for (int e = tid; e < mq_scratch_floats(N); e += NT) {
        const float v = mqs[e];
        if (e < 16) x0f[e] = v;
        else if (e < 16 + 172) { if (e < 16 + 169) Acd[e - 16] = v; }
        else if (e < 344) Bcd[e - 188] = v;
        else if (e < 356) wts[e - 344] = v;
        else Mb[e - 356] = v;
      }
      __syncthreads();
    }

    HMPC_STAMP(1);
    // ---------------- stage 2: powers of Acd, Toeplitz blocks, d = A_qp x0 - X_d ----------------
    // Acd = I + dt*A has the SRBD pattern (SolverMPC.cpp:312-318): Rb block (rows 0-2, cols 6-8), dt on
    // (3+c, 9+c) and -dt on (11,12).  Its powers P_k therefore differ from the identity in 14 entries only,
    //   P_k[0:3][6:9]  (k-fold rounded accumulation of dt*Rb),  P_k[3+c][9+c],  P_k[5][12],  P_k[11][12],
    // and the reference's dense sequential products reduce to the few terms below — every dropped term is an
    // exact zero product, so the values are those of the dense sums (SolverMPC.cpp:148-177).
    // Each item runs its own copy of the (one-FADD-per-step) recurrences, so the stage needs no exchange:
    //   items 0..35  : column c of rows r and 3+r of every M_k (r = item/12)   -> Mb[k][r][.], Mb[k][3+r][.]
    //   items 36..47 : row r of every d_s = P_{s+1} x0 - traj_s
    // Rows 6..11 of M_k equal Bcd's rows for every k and are read from Bcd directly by stage 3.
    for (int it = tid; it < 48; it += NT) {
      if (it < 36) {
        if (MQ && !first) continue;
        const int r = it / 12, c = it % 12;
        const float a0 = Acd[r * 13 + 6], a1 = Acd[r * 13 + 7], a2 = Acd[r * 13 + 8], ad = Acd[(3 + r) * 13 + 9 + r];
        const float b6 = Bcd[6 * 12 + c], b7 = Bcd[7 * 12 + c], b8 = Bcd[8 * 12 + c], b9 = Bcd[(9 + r) * 12 + c];
        float p0 = 0.f, p1 = 0.f, p2 = 0.f, pd = 0.f;  // P_k[r][6..8], P_k[3+r][9+r]
        float* dst = Mb + r * 12 + leg_of(c) * 6 + loc_of(c);
        for (int k = 0; k < N; k++) {
          dst[k * 72] = FA(FA(FM(p0, b6), FM(p1, b7)), FM(p2, b8));
          dst[k * 72 + 36] = FM(pd, b9);
          p0 = FA(a0, p0);
          p1 = FA(a1, p1);
          p2 = FA(a2, p2);
          pd = FA(ad, pd);
        }
      } else {
        const int r = it - 36;
        const float xr_ = x0f[r];
        if (r < 3) {
          const float a0 = Acd[r * 13 + 6], a1 = Acd[r * 13 + 7], a2 = Acd[r * 13 + 8];
          float p0 = 0.f, p1 = 0.f, p2 = 0.f;
          for (int s = 0; s < N; s++) {
            p0 = FA(a0, p0);
            p1 = FA(a1, p1);
            p2 = FA(a2, p2);
            const float acc = FA(FA(FA(xr_, FM(p0, x0f[6])), FM(p1, x0f[7])), FM(p2, x0f[8]));
            dd[12 * s + r] = FS(acc, (MQ ? trj[12 * s + r] : rf[54 + 12 * s + r]));
          }
        } else if (r < 6) {
          const float ad = Acd[r * 13 + r + 6], ag = Acd[11 * 13 + 12];
          float pd = 0.f, p5 = 0.f;  // P_k[r][r+6], P_k[5][12]
          for (int s = 0; s < N; s++) {
            p5 = FA(FM(pd, ag), p5);  // uses P_k[5][11] before it advances (only meaningful for r == 5)
            pd = FA(ad, pd);
            float acc = FA(xr_, FM(pd, x0f[r + 6]));
            if (r == 5) acc = FA(acc, FM(p5, x0f[12]));
            dd[12 * s + r] = FS(acc, (MQ ? trj[12 * s + r] : rf[54 + 12 * s + r]));
          }
        } else {
          const float ag = Acd[11 * 13 + 12];
          float p11 = 0.f;
          for (int s = 0; s < N; s++) {
            p11 = FA(ag, p11);
            const float acc = (r == 11) ? FA(xr_, FM(p11, x0f[12])) : xr_;
            dd[12 * s + r] = FS(acc, (MQ ? trj[12 * s + r] : rf[54 + 12 * s + r]));
          }
        }
      }
    }
    __syncthreads();
    if (MQ && first && k1 - k0 > 1) {
      for (int e = tid; e < mq_scratch_floats(N); e += NT) {
        float v = 0.f;
        if (e < 16) v = x0f[e];
        else if (e < 16 + 172) { if (e < 16 + 169) v = Acd[e - 16]; }
        else if (e < 344) v = Bcd[e - 188];
        else if (e < 356) v = rf[30 + e - 344];
        else v = Mb[e - 356];
        mqs[e] = v;
      }
    }

    HMPC_STAMP(2);
    // ---------------- stage 3: Hessian prefix chains (one 1x6 leg tile per item) + gradient ----------------
    if (dump) {
      float* oF = ka.dbg_F + (size_t)inst * 192;
      for (int e = tid; e < 192; e += NT) oF[e] = Fblk[e];
      float* olb = ka.dbg_lb + (size_t)inst * 16 * N;
      float* oub = ka.dbg_ub + (size_t)inst * 16 * N;
      for (int e = tid; e < 16 * N; e += NT) {
        const int s = e / 16, r = e % 16, leg = r / 8, rr_ = r % 8;
        float lo = 0.f, hi = 0.f;
        if (rr_ < 4) hi = (float)5e10;
        else if (rr_ == 4) hi = 0.01f;
        else if (rr_ < 7) lo = (float)(-5e10);
        else hi = FM(ka.f_max, (float)gait[2 * s + leg]);
        olb[e] = lo;
        oub[e] = hi;
      }
    }
    {
      float wr[12];
#pragma unroll
      for (int r = 0; r < 12; r++) wr[r] = rf[30 + r];
      // item = (li, lj, delta, i): running sums G_delta(K)[i][leg lj's six columns] = sum_{e<=K} T_{e+delta}^T M_e;
      // block (a,b) of B'SB, b - a = delta, equals G_delta(N-1-b) — the oracle's own summation order.
      // 32-item chunks in list order (longest chains first) go to the warps round-robin.
      const int nitems = (!MQ || first) ? flags[6] * 6 : 0;  // (H does not depend on the trajectory)
      for (int chunk = wid; chunk * 32 < nitems; chunk += NW) {
        const int it = chunk * 32 + lane;
        if (it >= nitems) continue;
        const int cm = comb[it / 6], ci = it % 6;
        const int li = cm & 1, lj = (cm >> 1) & 1, delta = (cm >> 2) & 63, Kmax = cm >> 8;
        const unsigned need = stmask[li] & (stmask[lj] >> delta);  // bit a: block (a, a+delta) wanted
        const int ii = col12_of(li, ci);
        float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        // rows 6..8 of every M_e equal Bcd's (k-independent): their products are loop invariants.
        // rows 3..5 / 9..11 hold one force axis each: they only couple force variables of the same axis.
        float prod[3][6];
#pragma unroll
        for (int r = 0; r < 3; r++) {
          const float tv = FM(Bcd[(6 + r) * 12 + ii], wr[6 + r]);
#pragma unroll
          for (int c = 0; c < 6; c++) prod[r][c] = FM(tv, Bcd[(6 + r) * 12 + col12_of(lj, c)]);
        }
        const bool fax = ci < 3;
        const int rax = fax ? ci : 0;
        const float w3 = rf[30 + 3 + rax];
        const float prod9 = FM(FM(Bcd[(9 + rax) * 12 + ii], rf[30 + 9 + rax]), Bcd[(9 + rax) * 12 + col12_of(lj, rax)]);
        for (int K = 0; K <= Kmax; K++) {
          const float* Mi = Mb + (K + delta) * 72 + 6 * li + ci;
          const float2* Mj = reinterpret_cast<const float2*>(Mb + K * 72 + 6 * lj);
          // all shared-memory operands of this step first (one latency instead of one per use)
          float mi[3];
          float2 mj[3][3];
#pragma unroll
          for (int r = 0; r < 3; r++) {
            mi[r] = Mi[r * 12];
            mj[r][0] = Mj[r * 6];
            mj[r][1] = Mj[r * 6 + 1];
            mj[r][2] = Mj[r * 6 + 2];
          }
          const float m3i = Mi[(3 + rax) * 12];
          const float m3j = Mb[K * 72 + (3 + rax) * 12 + 6 * lj + rax];
#pragma unroll
          for (int r = 0; r < 3; r++) {
            const float tv = FM(mi[r], wr[r]);  // (B'S)(i,k) = B(k,i)*w(k)
            acc[0] = FA(acc[0], FM(tv, mj[r][0].x));
            acc[1] = FA(acc[1], FM(tv, mj[r][0].y));
            acc[2] = FA(acc[2], FM(tv, mj[r][1].x));
            acc[3] = FA(acc[3], FM(tv, mj[r][1].y));
            acc[4] = FA(acc[4], FM(tv, mj[r][2].x));
            acc[5] = FA(acc[5], FM(tv, mj[r][2].y));
          }
          if (fax) {  // row 3+axis
            const float t3 = FM(FM(m3i, w3), m3j);
#pragma unroll
            for (int c = 0; c < 3; c++) acc[c] = (c == rax) ? FA(acc[c], t3) : acc[c];
          }
#pragma unroll
          for (int r = 0; r < 3; r++)
#pragma unroll
            for (int c = 0; c < 6; c++) acc[c] = FA(acc[c], prod[r][c]);
          if (fax) {  // row 9+axis
#pragma unroll
            for (int c = 0; c < 3; c++) acc[c] = (c == rax) ? FA(acc[c], prod9) : acc[c];
          }
          const int a = N - 1 - K - delta, b = a + delta;
          if ((need >> a) & 1u) {
            if (!dump && delta > 0) {  // block (b,a) strictly below the diagonal: element (cj, ci), no alpha
              // six consecutive rows of one column: at most two tiles, addresses by increments (hput, specialised)
              const int col = 6 * sl_blk[2 * a + li] + ci, row0 = 6 * sl_blk[2 * b + lj];
              const int I0 = row0 >> 3, r0 = row0 & 7, Jc = col >> 3, cb = col & 7;
              float* t0 = Hf + toff(I0, Jc);
              float* t1 = t0 + (I0 + 1) * 64;  // tile (I0 + 1, Jc)
#pragma unroll
              for (int cj = 0; cj < 6; cj++) {
                const float hv = FM(2.f, FA(acc[cj], 0.f));
                const int r = r0 + cj;
                float* t = (r < 8) ? t0 : t1;
                t[((r & 7) << 3) + cb] = hv;
                if (((r < 8) ? I0 : I0 + 1) == Jc) t[(cb << 3) + (r & 7)] = hv;  // diagonal tile: both triangles
              }
            } else {
              const int ka_ = dump ? 0 : sl_blk[2 * a + li], kb_ = dump ? 0 : sl_blk[2 * b + lj];
#pragma unroll
              for (int cj = 0; cj < 6; cj++) {
                const int jj = col12_of(lj, cj);
                if (delta == 0 && ii > jj) continue;  // the reference's solver reads the upper triangle only
                const float alpha = (delta == 0 && ii == jj) ? rf[42 + ii] : 0.f;
                const float hv = FM(2.f, FA(acc[cj], alpha));  // qH = 2*(B'SB + Alpha_rep)
                if (dump) {
                  float* oH = ka.dbg_H + (size_t)inst * (144 * N * N);
                  oH[(size_t)(12 * a + ii) * (12 * N) + 12 * b + jj] = hv;
                  oH[(size_t)(12 * b + jj) * (12 * N) + 12 * a + ii] = hv;
                } else {
                  const int gi = 6 * ka_ + ci, gj = 6 * kb_ + cj;
                  hput(Hf, gi > gj ? gi : gj, gi > gj ? gj : gi, hv);
                }
              }
            }
          }
        }
      }
    HMPC_STAMP(7);
      // gradient: g(a,ii) = sum_{s>=a} sum_r (T_{s-a}[r][ii]*2) * d_s[r]
      for (int e = tid; e < N * 12; e += NT) {
        const int a = e / 12, ii = e % 12, li = leg_of(ii);
        if (!((stmask[li] >> a) & 1u)) continue;
        float acc = 0.f;
        float t6[6];
#pragma unroll
        for (int r = 0; r < 6; r++) t6[r] = FM(FM(Bcd[(6 + r) * 12 + ii], wr[6 + r]), 2.f);
        for (int s = a; s < N; s++) {
          const float* Mi = Mb + (s - a) * 72 + 6 * li + loc_of(ii);
          const float* dk = dd + 12 * s;
          float mi[6], dkr[12];
#pragma unroll
          for (int r = 0; r < 6; r++) mi[r] = Mi[r * 12];
#pragma unroll
          for (int r = 0; r < 12; r++) dkr[r] = dk[r];
#pragma unroll
          for (int r = 0; r < 6; r++) acc = FA(acc, FM(FM(FM(mi[r], wr[r]), 2.f), dkr[r]));
#pragma unroll
          for (int r = 0; r < 6; r++) acc = FA(acc, FM(t6[r], dkr[6 + r]));
        }
        if (dump) ka.dbg_g[(size_t)inst * 12 * N + e] = acc;
        else gq[6 * sl_blk[2 * a + li] + loc_of(ii)] = (double)acc;
      }
    }
    __syncthreads();
    if (dump) continue;

    if (NB == 0) {
      if constexpr (MQ) {  // every candidate at once
        const size_t r0 = (size_t)inst * ka.mq_k + kq;
        for (int e = tid; e < (k1 - kq) * 12 * N; e += NT) {
          if (ka.wrench) ka.wrench[r0 * 12 * N + e] = 0.f;
          if (ka.wrench64) ka.wrench64[r0 * 12 * N + e] = 0.0;
        }
        for (int e = tid; e < k1 - kq; e += NT) ka.status[r0 + e] = ST_OK;
      } else {
        for (int e = tid; e < 12 * N; e += NT) {
          if (ka.wrench) ka.wrench[(size_t)inst * 12 * N + e] = 0.f;
          if (ka.wrench64) ka.wrench64[(size_t)inst * 12 * N + e] = 0.0;
        }
        if (ka.tau && tid < 10) ka.tau[(size_t)inst * 10 + tid] = 0.f;
        if (tid == 0) {
          ka.status[inst] = ST_OK;
          if (ka.ws_state) ka.ws_state[(size_t)inst * WS_STATE_INTS] = 0;
        }
      }
      __syncthreads();
      continue;
    }
    if constexpr (CLS == 3) {
      // the exact QP data for the residuals of the refinement rounds: stage 4 inverts the tiles in place, gq becomes zb
      float* Hc = reinterpret_cast<float*>(smem + L.Hc);
      double* gc = reinterpret_cast<double*>(smem + L.gc);
      if (!MQ || first)
        for (int e = tid; e < tri(NT8) * 64; e += NT) Hc[e] = Hf[e];
      for (int e = tid; e < n; e += NT) gc[e] = gq[e];
    }

    HMPC_STAMP(3);
    // ---------------- stage 4: blocked sweep inversion on the fp64 tensor pipe ----------------
    // The symmetric matrix is cut into 8x8 tiles (rows/columns beyond n: identity).  Sweeping the diagonal tile k
    //   A_kk <- -D^-1,  A_ik <- A_ik D^-1,  A_kj <- D^-1 A_kj,  A_ij <- A_ij - A_ik D^-1 A_kj        (D = A_kk)
    // for k = 0..NT8-1 leaves -H^-1 (Goodnight's sweep operator, block form; every D is a Schur complement of an SPD
    // matrix, so no pivoting).  Each warp keeps the lower tiles of two tile rows in mma accumulator fragments for the
    // whole stage.  Per block step: ONE barrier.  During step k the owners of panel k+1 update those tiles first and
    // publish them (the diagonal one already inverted, in-register) in fragment order, so that in step k+1 every
    // operand of W_I = P_I D^-1 and of the rank-8 updates A_IJ -= W_I P_J' is one conflict-free 8-byte load.
    if (!MQ || first) {
      // accumulator slots: tile J of row rB in c[J], tile J of row rA in c[2NW - J] (rA + rB = NT8 - 1 <= 2NW - 1, so the
      // two never meet) — every slot index is a compile-time constant of the unrolled loops
      constexpr int TS = 2 * NW + 1;
      const int rA = wid, rB = NT8 - 1 - wid;
      const bool hasA = rA <= rB, hasB = rA < rB;
      const int g = lane >> 2, t4 = lane & 3;
      const int fp = frag_pair(lane);
      const int ft = frag_elem(2 * t4, g);  // transposed element (2t, g); (2t+1, g) is 4 further
      double c0[TS], c1[TS];
#pragma unroll
      for (int t = 0; t < TS; t++) { c0[t] = 0.0; c1[t] = 0.0; }
      // the diagonal of H survives the stage (in x0, not live yet): stage 5 checks H_ii (H^-1)_ii against it
      for (int i = tid; i < n; i += NT) x0[i] = (double)Hf[toff(i >> 3, i >> 3) + (i & 7) * 9];
      {
        const int i = 8 * rB + g, j = 2 * t4;
        const float* src = Hf + toff(rB, 0) + g * 8 + 2 * t4;
#pragma unroll
        for (int J = 0; J < 2 * NW; J++)
          if (hasB && J <= rB) {
            const float2 v = *reinterpret_cast<const float2*>(src + J * 64);
            c0[J] = (i < n && 8 * J + j < n) ? (double)v.x : (i == 8 * J + j ? 1.0 : 0.0);
            c1[J] = (i < n && 8 * J + j + 1 < n) ? (double)v.y : (i == 8 * J + j + 1 ? 1.0 : 0.0);
          }
      }
      {
        const int i = 8 * rA + g, j = 2 * t4;
        const float* src = Hf + toff(rA, 0) + g * 8 + 2 * t4;
#pragma unroll
        for (int J = 0; J < NW; J++)
          if (hasA && J <= rA) {
            const float2 v = *reinterpret_cast<const float2*>(src + J * 64);
            c0[TS - 1 - J] = (i < n && 8 * J + j < n) ? (double)v.x : (i == 8 * J + j ? 1.0 : 0.0);
            c1[TS - 1 - J] = (i < n && 8 * J + j + 1 < n) ? (double)v.y : (i == 8 * J + j + 1 ? 1.0 : 0.0);
          }
      }
      double* Pbuf = reinterpret_cast<double*>(smem + L.Pb);
      double* WsA = reinterpret_cast<double*>(smem + L.Ws) + wid * 128;  // -W of row rA / rB, fragment order
      double* WsB = WsA + 64;
      bool bad = false;
      __syncthreads();  // the panel buffers may overlay the float32 tiles just read
      // panel 0: column 0 of every row; tile (0,0) (warp 0, row rA = 0) inverted
      if (hasB) *reinterpret_cast<double2*>(Pbuf + rB * 64 + fp) = make_double2(c0[0], c1[0]);
      if (hasA) {
        double d0 = c0[TS - 1], d1 = c1[TS - 1];
        if (rA == 0) bad |= tile_inverse_spd(d0, d1, lane);
        *reinterpret_cast<double2*>(Pbuf + rA * 64 + fp) = make_double2(d0, d1);
      }
      __syncthreads();
      for (int k = 0; k < NT8; k++) {
        const double* pbl = Pbuf + (k & 1) * NT8 * 64 + lane;  // operand fragments of panel tile I: pbl[I*64], pbl[I*64+32]
        double* Pn = Pbuf + ((k + 1) & 1) * NT8 * 64;
        const int kn = k + 1;  // the panel prepared for the next step (look-ahead)
        const bool genA = hasA && rA != k, genB = hasB && rB != k;
        double wA0 = 0.0, wA1 = 0.0, wB0 = 0.0, wB1 = 0.0;
        HMPC_WSTAMP(0);
        {
          // W_R = P_R D^-1 for the warp's rows, negated: stashed in fragment order (it is also the new column-k tile
          // of the row) and reloaded as the A operand of the rank-8 updates A_RJ -= W_R P_J'
          const double di0 = pbl[k * 64], di1 = pbl[k * 64 + 32];
          if (genA) {
            double W0 = 0.0, W1 = 0.0;
            dmma884(W0, W1, pbl[rA * 64], di0);
            dmma884(W0, W1, pbl[rA * 64 + 32], di1);
            *reinterpret_cast<double2*>(WsA + fp) = make_double2(-W0, -W1);
          }
          if (genB) {
            double W0 = 0.0, W1 = 0.0;
            dmma884(W0, W1, pbl[rB * 64], di0);
            dmma884(W0, W1, pbl[rB * 64 + 32], di1);
            *reinterpret_cast<double2*>(WsB + fp) = make_double2(-W0, -W1);
          }
          __syncwarp();
          if (genA) { wA0 = WsA[lane]; wA1 = WsA[32 + lane]; }
          if (genB) { wB0 = WsB[lane]; wB1 = WsB[32 + lane]; }
        }
        if (k == 1) HMPC_STAMP(20);
        HMPC_WSTAMP(1);
        // look-ahead: the next diagonal tile first — its inversion is the longest chain of the step.  It is an ordinary
        // tile in step k: rank-8 update (on a copy; the slot itself is updated below with the others), then its
        // in-register inverse goes to the next panel.
        if (kn < NT8 && ((hasA && rA == kn) || (hasB && rB == kn))) {
          const bool inA = hasA && rA == kn;
          double d0 = 0.0, d1 = 0.0;
#pragma unroll
          for (int J = 0; J < 2 * NW; J++)
            if (J == kn) {
              if (J < NW && inA) { d0 = c0[TS - 1 - (J < NW ? J : 0)]; d1 = c1[TS - 1 - (J < NW ? J : 0)]; }
              else { d0 = c0[J]; d1 = c1[J]; }
            }
          dmma884(d0, d1, inA ? wA0 : wB0, pbl[kn * 64]);
          dmma884(d0, d1, inA ? wA1 : wB1, pbl[kn * 64 + 32]);
          bad |= tile_inverse_spd(d0, d1, lane);
          *reinterpret_cast<double2*>(Pn + kn * 64 + fp) = make_double2(d0, d1);
        }
        if (k == 1) HMPC_STAMP(21);
        HMPC_WSTAMP(2);
        {
          // rank-8 updates of both rows (they share the P_J fragments); the column-k tile becomes W_R; the column-kn
          // tile goes to the next panel
          const int limA = genA ? rA : -1, limB = genB ? rB : -1;
          const int pubA = (hasA && rA > kn) ? kn : -1, pubB = (hasB && rB > kn) ? kn : -1;
          double* PnA = Pn + rA * 64 + fp;
          double* PnB = Pn + rB * 64 + fp;
#pragma unroll
          for (int J = 0; J < 2 * NW; J++) {
            if (J > limB && J > limA) break;
            const double p0 = pbl[J * 64], p1 = pbl[J * 64 + 32];
            if (J <= limB) {
              if (J == k) {
                const double2 d = *reinterpret_cast<const double2*>(WsB + fp);
                c0[J] = -d.x;
                c1[J] = -d.y;
              } else {
                dmma884(c0[J], c1[J], wB0, p0);
                dmma884(c0[J], c1[J], wB1, p1);
              }
              if (J == pubB) *reinterpret_cast<double2*>(PnB) = make_double2(c0[J], c1[J]);
            }
            if (J < NW && J <= limA) {
              constexpr int dummy = 0;
              const int sa = TS - 1 - (J < NW ? J : dummy);
              if (J == k) {
                const double2 d = *reinterpret_cast<const double2*>(WsA + fp);
                c0[sa] = -d.x;
                c1[sa] = -d.y;
              } else {
                dmma884(c0[sa], c1[sa], wA0, p0);
                dmma884(c0[sa], c1[sa], wA1, p1);
              }
              if (J == pubA) *reinterpret_cast<double2*>(PnA) = make_double2(c0[sa], c1[sa]);
            }
          }
        }
        if (k == 1) HMPC_STAMP(22);
        HMPC_WSTAMP(3);
        // pivot row k (one warp of the CTA): A_kJ <- D^-1 P_J' for J < k, A_kk <- -D^-1
        if ((hasB && rB == k) || (hasA && rA == k)) {
          const bool inA = hasA && rA == k;
          const double di0 = pbl[k * 64], di1 = pbl[k * 64 + 32];
          const double2 dk = *reinterpret_cast<const double2*>(Pbuf + (k & 1) * NT8 * 64 + k * 64 + fp);
#pragma unroll
          for (int J = 0; J < 2 * NW; J++) {
            if (J > k) break;
            double v0 = -dk.x, v1 = -dk.y;
            if (J < k) {
              v0 = 0.0;
              v1 = 0.0;
              dmma884(v0, v1, di0, pbl[J * 64]);
              dmma884(v0, v1, di1, pbl[J * 64 + 32]);
            }
            if (J < NW && inA) { c0[TS - 1 - (J < NW ? J : 0)] = v0; c1[TS - 1 - (J < NW ? J : 0)] = v1; }
            else { c0[J] = v0; c1[J] = v1; }
          }
        }
        // row kn of the next panel, transposed: P_J = A_kn,J'
        if (kn < NT8 && ((hasB && rB == kn) || (hasA && rA == kn))) {
          const bool inA = hasA && rA == kn;
#pragma unroll
          for (int J = 0; J < 2 * NW; J++) {
            if (J >= kn) break;
            const double v0 = (J < NW && inA) ? c0[TS - 1 - (J < NW ? J : 0)] : c0[J];
            const double v1 = (J < NW && inA) ? c1[TS - 1 - (J < NW ? J : 0)] : c1[J];
            Pn[J * 64 + ft] = v0;
            Pn[J * 64 + ft + 4] = v1;
          }
        }
        if (k == 1) HMPC_STAMP(23);
        HMPC_WSTAMP(4);
        __syncthreads();
        HMPC_WSTAMP(5);
        if (k == 1) HMPC_STAMP(24);
        if (k == 0) HMPC_STAMP(19);
      }
      {
        double* dstB = Hd + toff(rB, 0) + g * 8 + 2 * t4;
        double* dstA = Hd + toff(rA, 0) + g * 8 + 2 * t4;
#pragma unroll
        for (int J = 0; J < 2 * NW; J++) {
          if (hasB && J <= rB) *reinterpret_cast<double2*>(dstB + J * 64) = make_double2(-c0[J], -c1[J]);
          if (J < NW && hasA && J <= rA)
            *reinterpret_cast<double2*>(dstA + J * 64) = make_double2(-c0[TS - 1 - (J < NW ? J : 0)], -c1[TS - 1 - (J < NW ? J : 0)]);
        }
      }
      if (__any_sync(0xffffffffu, bad) && lane == 0) flags[3] = ST_NOT_SPD;
      __syncthreads();
    }

    HMPC_STAMP(4);
    // ---------------- stage 5: dual active-set iterations (Goldfarb-Idnani) ----------------
    // Thread e < m owns constraint row e (slack s_e in a register), thread NT-1-i owns variable i.  A working-set slot
    // keeps t_j = H^-1 a_j; the Schur complement inverse (A_W H^-1 A_W')^-1 is held explicitly (rank-1 up/downdates).
    // One working-set change = selection | t_p = H^-1 a_p | warp 0: step direction, ratio test, update | x, slacks:
    // four barriers.
    // rows: three blocks (30 lanes) per warp, so that a block's ten rows share a warp; row id = 10 * block + type
    const int vi = NT - 1 - tid;
    const int ke = 3 * wid + lane / 10;
    const bool isvar = vi < n, iscon = lane < 30 && ke < NB;
    const int erow = iscon ? 10 * ke + (lane - 10 * (lane / 10)) : 0x7fffffff;
    double xreg = 0.0;
    // Conditioning check.  The sweep inversion (Gauss-Jordan without pivoting, in place) loses accuracy like the SQUARE of
    // the scaled condition number: measured against an fp64 referee the optimum is off by ~1e-13 kappa^2, kappa = max_i
    // H_ii (H^-1)_ii (2e2 ... 1e4 on every workload of BASELINE.json, 3e5 for a robot lying on its side, where the answer
    // is 8e-3 off).  Beyond ka.kappa_max the 1e-4 contract cannot be promised: such an instance is reported as not solved
    // (ST_NOT_SPD: "Hessian not positive definite enough") instead of returning a wrong wrench with a clean status.
    bool illc = false;
    if (isvar) {
      xreg = -hinv_rowdot(Hd, vi, NT8, gq);
      if (!MQ || first) illc_h = x0[vi] * Hd[toff(vi >> 3, vi >> 3) + (vi & 7) * 9] > ka.kappa_max;
      illc = illc_h;
      x0[vi] = xreg;
    }
    {
      const unsigned key = __float_as_uint(fabsf((float)xreg));  // non-negative floats order like their bit patterns
      const unsigned kmax = __reduce_max_sync(0xffffffffu, key);
      if (lane == 0) redk[16 + wid] = kmax;  // upper half: the selection below reuses redk[0..NW) without a barrier in between
    }
    if (tid < 8) amask[tid] = 0u;
    if (tid == 0) { flags[7] = 0; flags[8] = 0; flags[9] = 0; flags[11] = 0; }
    const int ill = __syncthreads_or((int)illc);
    double tol;
    {
      unsigned kx = redk[16];
      for (int w = 1; w < NW; w++) kx = redk[16 + w] > kx ? redk[16 + w] : kx;
      tol = ka.tol_kkt * fmax(1.0, (double)__uint_as_float(kx));
    }
    // per-row constants: normal, right-hand side, slack at the unconstrained minimiser
    double ne[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    double se = 0.0, rhs_e = 0.0;
    int nie = 0, myslot = -1;
    bool act = false;
    if (iscon) {
      const int te = lane - 10 * (lane / 10);
      nie = (blk_sl[ke] & 1) * 10 + te;
      const double* nn = nrm + nie * 6;
#pragma unroll
      for (int c = 0; c < 6; c++) ne[c] = nn[c];
      rhs_e = (te == 5) ? -(double)0.01f : ((te == 9) ? -fz[ke] : 0.0);
      se = dot6(ne, x0 + 6 * ke) - rhs_e;
    }

    int q = 0, iters = 0;
    int code = flags[3];
    if (ill && code == ST_OK) code = ST_NOT_SPD;

    // ---- block start ----------------------------------------------------------------------------------------------
    // Rounds of: take the most violated inactive row of EVERY block, solve on the enlarged working set (all multipliers
    // at once through the explicit Schur complement S = A_W H^-1 A_W'), drop rows whose multiplier is not positive.
    // What a round leaves — x minimises the QP on the rows of W held as equalities, all multipliers positive — is an
    // S-pair, exactly the invariant of the dual iteration below, which therefore continues from it (and, when no row is
    // violated any more, stops at its first selection).  A walking gait ends with about one active row per stance step:
    // one to three rounds instead of ~N sequential working-set changes.  Every thread works in every phase: the block
    // minimum is a masked REDUX over the block's ten lanes, each entry of [S | b] lives in one thread's register during a
    // Gauss-Jordan sweep with one barrier per pivot.  Any doubt (capacity, a non-positive pivot) falls back to the plain
    // iteration from the unconstrained minimiser.
    if (qmax <= 31 && tcap > 0) {
      int* newslot = reinterpret_cast<int*>(rr);       // [nadd] slots of the entering rows (rr is not live yet)
      // slots a block round may use: those with a cached column, as many as one S entry per thread allows (tri(q) <= NT)
      int slot_cap = (int)((sqrtf(8.f * (float)NT + 1.f) - 1.f) * 0.5f);
      while (tri(slot_cap + 1) <= NT) slot_cap++;
      while (tri(slot_cap) > NT) slot_cap--;
      slot_cap = slot_cap < tcap ? slot_cap : tcap;
      double* colb = dvs;                              // [2][qmax + 3] pivot column, b_p and 1/d, double-buffered
      const int cst = qmax + 3;
      // Warm start (closed loop): the rows that were active at the previous tick's optimum, moved with the horizon, are
      // proposed as round 0's entering rows instead of the most violated ones; the round solves on them, prunes the ones
      // whose multiplier is not positive, and the following rounds / the dual iteration repair what changed.
      bool warm = false;
      unsigned* wmark = reinterpret_cast<unsigned*>(redi + 16);  // [16] bitmap over the rows
      if (ka.warm_start && ka.ws_state) {
        const int* ws = ka.ws_state + (size_t)inst * WS_STATE_INTS;
        const int cnt = ws[0];
        const int shift = ka.ws_shifts ? ka.ws_shifts[inst] : ka.ws_shift;  // < 0 (e.g. a reset robot): a cold start
        if (shift >= 0 && cnt > 0 && cnt < WS_STATE_INTS) {
          if (tid < 16) wmark[tid] = 0u;
          __syncthreads();
          if (tid < cnt) {
            const int ent = ws[1 + tid];
            const int sl = (ent >> 8) - 2 * shift;  // (step, leg): one MPC step later it sits one step earlier
            if (sl >= 0 && sl < 2 * N) {
              const int kb = sl_blk[sl];
              if (kb >= 0) {
                const int e = 10 * kb + (ent & 0xff) % 10;
                atomicOr(&wmark[e >> 5], 1u << (e & 31));
              }
            }
            // the steps that entered the horizon have no history: they inherit the rows of the old last step
            if ((ent >> 8) >= 2 * (N - 1)) {
              for (int sn = sl + 2; sn >= 0 && sn < 2 * N; sn += 2) {
                const int kb = sl_blk[sn];
                if (kb >= 0) {
                  const int e = 10 * kb + (ent & 0xff) % 10;
                  atomicOr(&wmark[e >> 5], 1u << (e & 31));
                }
              }
            }
          }
          __syncthreads();
          warm = true;
        }
      }
      for (int round = 0; code == ST_OK && round < ka.block_rounds; round++) {
        if (round == 0) HMPC_STAMP(8);
        // most violated inactive row of every block (round 0 of a warm start: the proposed rows)
        const unsigned gm = (lane < 30) ? (0x3ffu << (10 * (lane / 10))) : (1u << lane);
        const float sf = (iscon && !act) ? (float)se : 3.0e38f;
        const unsigned key = fkey(sf);
        const unsigned kmin = __reduce_min_sync(gm, key);
        const unsigned tie = __ballot_sync(0xffffffffu, key == kmin) & gm;
        bool cand = iscon && !act && se < -tol && key == kmin && (__ffs(tie) - 1) == lane;
        if (warm) cand = iscon && ((wmark[erow >> 5] >> (erow & 31)) & 1u);
        const bool warm_round = warm;
        warm = false;
        const unsigned cm = __ballot_sync(0xffffffffu, cand);
        if (lane == 0) redi[wid] = __popc(cm);
        __syncthreads();
        int nadd = 0, rank = __popc(cm & ((1u << lane) - 1u));  // row order: the earliest steps first
        for (int w = 0; w < NW; w++) {
          const int c = redi[w];
          nadd += c;
          if (w < wid) rank += c;
        }
        const unsigned am0 = amask[0];
        __syncthreads();  // everybody has read the counts and the slot mask
        // Every slot of a block round needs its cached column and one thread per entry of S: rows enter only while free
        // slots below slot_cap remain (the first candidates in row order take them, the others wait for the next round or
        // for the dual iteration).  No violated row: the iteration below confirms and stops.
        if (nadd == 0 || (am0 >> slot_cap) != 0u) break;
        // after the first round, few entering rows are cheaper one by one in the dual iteration than as another solve
        if (round > 0 && nadd < ka.block_min) break;
        const int room = slot_cap - __popc(am0);
        if (nadd > room) nadd = room;
        if (nadd <= 0) break;
        if (rank >= nadd) cand = false;
        unsigned mybit = 0u;
        if (cand) {  // the rank-th entering row takes the rank-th free slot
          unsigned fm = ~am0;
          for (int r = 0; r < rank; r++) fm &= fm - 1;
          const int sl = __ffs(fm) - 1;
          myslot = sl;
          wsl[sl] = ws_pack(ke, nie);
          newslot[rank] = sl;
          mybit = 1u << sl;
        }
        mybit = __reduce_or_sync(0xffffffffu, mybit);  // one shared-memory atomic per warp, not per row
        if (lane == 0 && mybit) atomicOr(&amask[0], mybit);
        __syncthreads();
        if (round == 0) HMPC_STAMP(9);
        if (isvar) {
          for (int r = 0; r < nadd; r++) {
            const int sl = newslot[r], w = wsl[sl];
            T[sl * n + vi] = hinv_dot6(Hd, vi, 6 * (w >> 8), nrm + (w & 0xff) * 6);
          }
        }
        __syncthreads();
        if (round == 0) HMPC_STAMP(10);
        // solve S lam = b on the working set; rows with a non-positive multiplier leave and the solve is repeated.
        // Thread e2 < tri(qh) holds entry (i, j), j <= i, of S; the diagonal owners also hold b_i.
        int verdict = 0;  // 0: all multipliers positive, 1: gave up
        for (int attempt = 0; attempt < 4; attempt++) {
          const unsigned am = amask[0];
          const int qh = 32 - __clz(am);
          const bool own = tid < tri(qh);
          int i = 0, j = 0;
          double a = 0.0, bi = 0.0;
          if (own) {
            i = (int)((sqrtf(8.f * (float)tid + 1.f) - 1.f) * 0.5f);
            while (tri(i + 1) <= tid) i++;
            while (tri(i) > tid) i--;
            j = tid - tri(i);
            const bool ui = (am >> i) & 1u, uj = (am >> j) & 1u;
            a = (i == j) ? 1.0 : 0.0;  // free slots: identity rows
            if (ui && uj) {
              const int w = wsl[i], ki = w >> 8;
              const double* ni = nrm + (w & 0xff) * 6;
              a = dot6(ni, T + j * n + 6 * ki);
              if (i == j) {
                const int te = (w & 0xff) % 10;
                bi = ((te == 5) ? -(double)0.01f : ((te == 9) ? -fz[ki] : 0.0)) - dot6(ni, x0 + 6 * ki);
              }
            } else if (ui != uj) {
              a = 0.0;
            }
          }
          const bool diag = own && i == j;
          // publish pivot column 0: S(.,0), b_0, 1/S(0,0)
          bool sing = false;
          if (own && j == 0) {
            colb[i] = a;
            if (i == 0) {
              colb[qh] = bi;
              colb[qh + 1] = fast_rcp(a);
              sing = !(a > 1e-13);
            }
          }
          if (round == 0 && attempt == 0) HMPC_STAMP(11);
          __syncthreads();
          for (int pv = 0; pv < qh; pv++) {
            if (own) {
              const double* cc = colb + (pv & 1) * cst;
              double* cn = colb + ((pv + 1) & 1) * cst;
              const double inv = cc[qh + 1];
              const double ci = cc[i], cj = cc[j];
              if (diag) bi = (i == pv) ? cc[qh] * inv : fma(-ci * inv, cc[qh], bi);
              if (i == pv) a = (j == pv) ? -inv : cj * inv;
              else if (j == pv) a = ci * inv;
              else a = fma(-ci * inv, cj, a);
              // next pivot's column: row pv+1 left of the diagonal and column pv+1 from the diagonal down
              const int pn = pv + 1;
              if (pn < qh) {
                if (j == pn) cn[i] = a;
                else if (i == pn) cn[j] = a;
                if (diag && i == pn) {
                  cn[qh] = bi;
                  cn[qh + 1] = fast_rcp(a);
                  sing |= !(a > 1e-13);
                }
              }
            }
            __syncthreads();
          }
          if (round == 0 && attempt == 0) HMPC_STAMP(12);
          // -S^-1 and lam = S^-1 b are in the registers: store them for the dual iteration / the x update
          bool neg = false;
          if (own) {
            Sv[tid] = -a;  // packed lower rows: index tri(i) + j = tid
            if (diag) {
              const bool used = (am >> i) & 1u;
              lam[i] = used ? bi : 0.0;
              neg = used && !(bi > 0.0);
            }
          }
          const int anyneg = __syncthreads_or((int)neg | ((int)sing << 1));
          if (anyneg & 2) { verdict = 1; break; }
          if (!(anyneg & 1)) break;
          if (attempt == 3) { verdict = 1; break; }
          // drop the rows with non-positive multipliers (their owner threads clear the slot) and solve again
          if (myslot >= 0 && !(lam[myslot] > 0.0)) {
            atomicAnd(&amask[0], ~(1u << myslot));
            myslot = -1;
            act = false;
            atomicAdd(&flags[11], 1);
          }
          __syncthreads();
        }
        if (round == 0) HMPC_STAMP(13);
        if (verdict != 0 || amask[0] == 0u) {
          // dependent rows / no progress: forget the guess, the plain iteration starts from x0
          __syncthreads();
          if (tid == 0) { amask[0] = 0u; flags[7] = 0; flags[8] = 0; flags[9] = 0; }
          q = 0;
          act = false;
          myslot = -1;
          if (isvar) xreg = x0[vi];
          if (iscon) se = dot6(ne, x0 + 6 * ke) - rhs_e;
          __syncthreads();
          break;
        }
        const unsigned amf = amask[0];
        const int qhf2 = 32 - __clz(amf);
        if (iscon) act = myslot >= 0;
        q = __popc(amf);
        if (!warm_round) iters += nadd;  // proposals of a warm start are not changes; what the solve drops of them is
        if (tid == 0) {
          flags[9] = qhf2;
          flags[7] = __ffs(~amf) - 1;
        }
        if (isvar) {
          double acc = x0[vi];
          for (int j = 0; j < qhf2; j++)
            if ((amf >> j) & 1u) acc = fma(lam[j], T[j * n + vi], acc);
          xreg = acc;
          zb[vi] = acc;
        }
        __syncthreads();
        if (round == 0) HMPC_STAMP(14);
        if (iscon) se = dot6(ne, zb + 6 * ke) - rhs_e;
        if (round == 0) HMPC_STAMP(15);
      }
      iters += flags[11];
    }
    HMPC_STAMP(16);
    bool noise_stop = false;
    while (code == ST_OK) {
      // ---- most violated inactive row (selection in float, value in double) ----
      const float sf = (iscon && !act) ? (float)se : 3.0e38f;
      const unsigned key = fkey(sf);
      const unsigned kmin = __reduce_min_sync(0xffffffffu, key);
      const int imin = __reduce_min_sync(0xffffffffu, key == kmin ? erow : 0x7fffffff);
      if (iscon && erow == imin) redv[wid] = se;
      if (lane == 0) { redk[wid] = kmin; redi[wid] = imin; }
      __syncthreads();
      unsigned kb = redk[0];
      int p = redi[0], wb = 0;
      for (int w = 1; w < NW; w++) {
        const unsigned ok = redk[w];
        if (ok < kb) { kb = ok; p = redi[w]; wb = w; }  // ties: the lower warp holds the lower row index
      }
      if (kb == fkey(3.0e38f)) break;  // every row is in the working set
      double sp = redv[wb];
      if (!(sp < -tol)) break;         // KKT point reached
      const int kp = p / 10, nip = (blk_sl[kp] & 1) * 10 + (p - 10 * kp);
      const double* np_ = nrm + nip * 6;
      const int f = flags[7];  // slot the entering row will take
      double* Tf = T + (f < tcap ? f : tcap) * n;  // a slot beyond the cache uses the spare column
      if (isvar) Tf[vi] = hinv_dot6(Hd, vi, 6 * kp, np_);
      __syncthreads();

      // ---- add row p (possibly after dropping blocking ones) ----
      double lam_p = 0.0;
      while (true) {
        iters++;
        if (iters > ka.max_iter) { code = ST_ITER_CAP; break; }
        if (wid == 0) {
          const int qhi = flags[9];
          for (int s2 = lane; s2 < qhi; s2 += 32) {
            double d = 0.0;
            if ((amask[s2 >> 5] >> (s2 & 31)) & 1u) {
              const int w = wsl[s2];
              d = dot6(nrm + (w & 0xff) * 6, Tf + 6 * (w >> 8));
            }
            dvs[s2] = d;
          }
          const double cHc = dot6(np_, Tf + 6 * kp);
          __syncwarp();
          // step direction in the dual space r = S^-1 d, curvature, ratio test
          double part = 0.0, tloc = __longlong_as_double(0x7ff0000000000000ll);
          int lloc = 0x7fffffff;
          for (int s2 = lane; s2 < qhi; s2 += 32) {
            const int rs = tri(s2);
            double a0 = 0.0, a1 = 0.0;
            int j = 0;
            for (; j + 1 < qhi; j += 2) {
              a0 = fma((j <= s2) ? Sv[rs + j] : Sv[tri(j) + s2], dvs[j], a0);
              a1 = fma((j + 1 <= s2) ? Sv[rs + j + 1] : Sv[tri(j + 1) + s2], dvs[j + 1], a1);
            }
            if (j < qhi) a0 = fma((j <= s2) ? Sv[rs + j] : Sv[tri(j) + s2], dvs[j], a0);
            const double acc = a0 + a1;
            rr[s2] = acc;
            part = fma(dvs[s2], acc, part);
            if (acc > 0.0) {
              const double ratio = lam[s2] * fast_rcp(acc);
              if (ratio < tloc) { tloc = ratio; lloc = s2; }
            }
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
          const double zn = cHc - part;
          // exact minimum of the non-negative ratios: high word, then low word among the lanes that hold it
          const unsigned thi = (unsigned)__double2hiint(tloc), tlo = (unsigned)__double2loint(tloc);
          const unsigned mhi = __reduce_min_sync(0xffffffffu, thi);
          const unsigned mlo = __reduce_min_sync(0xffffffffu, thi == mhi ? tlo : 0xffffffffu);
          const int l1 = __reduce_min_sync(0xffffffffu, (thi == mhi && tlo == mlo) ? lloc : 0x7fffffff);
          const double t1 = (l1 == 0x7fffffff) ? 1e300 : __hiloint2double((int)mhi, (int)mlo);
          const bool dependent = !(zn > ka.tol_dep * cHc);
          const double t2 = dependent ? 1e300 : fmax(0.0, -sp * fast_rcp(zn));
          const double t = fmin(t1, t2);
          int decision;  // 0 = full step (p joins W), 1 = partial step (drop l1, retry), 2 = infeasible, 3 = W full, 4 = see below
          if (!(t < 1e299)) decision = (-sp <= 100.0 * tol) ? 4 : 2;
          else if (t2 <= t1) decision = (q >= qmax) ? 3 : 0;
          else decision = 1;
          __syncwarp();
          if (decision < 2) {
            for (int s2 = lane; s2 < qhi; s2 += 32) lam[s2] = fmax(0.0, lam[s2] - t * rr[s2]);
          }
          int qhn = qhi;
          if (decision == 0) {
            // bordered inverse: S^-1 <- [S^-1 + r r'/zn, -r/zn; -r'/zn, 1/zn] with the new row in slot f
            const double izn = fast_rcp(zn);
            qhn = (f + 1 > qhi) ? f + 1 : qhi;
            for (int s2 = lane; s2 < qhn; s2 += 32) {
              const int rs = tri(s2);
              if (s2 == f) {
                for (int j = 0; j < f; j++) Sv[rs + j] = -rr[j] * izn;
                Sv[rs + f] = izn;
              } else {
                const double rs_ = rr[s2] * izn;
                for (int j = 0; j <= s2; j++) Sv[rs + j] = (j == f) ? -rs_ : fma(rs_, rr[j], Sv[rs + j]);
              }
            }
            __syncwarp();  // the multiplier update above also touched slot f (if it lies below qhi)
            if (lane == 0) {
              wsl[f] = ws_pack(kp, nip);
              lam[f] = lam_p + t;
              amask[f >> 5] |= 1u << (f & 31);
            }
          } else if (decision == 1) {
            // drop slot l1: S^-1 <- S^-1 - c c'/c_l without row/column l1 (c = column l1), which is then cleared
            lam_p += t;
            for (int s2 = lane; s2 < qhi; s2 += 32) dvs[s2] = (s2 >= l1) ? Sv[tri(s2) + l1] : Sv[tri(l1) + s2];
            __syncwarp();
            const double ipv = fast_rcp(dvs[l1]);
            for (int s2 = lane; s2 < qhi; s2 += 32) {
              const int rs = tri(s2);
              const double cs = dvs[s2] * ipv;
              for (int j = 0; j <= s2; j++) Sv[rs + j] = (j == l1 || s2 == l1) ? 0.0 : fma(-cs, dvs[j], Sv[rs + j]);
            }
            if (lane == 0) {
              const int w = wsl[l1];
              flags[5] = (w >> 8) * 10 + ((w & 0xff) % 10);
              lam[l1] = 0.0;
              amask[l1 >> 5] &= ~(1u << (l1 & 31));
            }
          }
          __syncwarp();
          if (lane == 0) {
            flags[4] = decision;
            flags[8] = qhi;
            flags[9] = qhn;
            dsc[0] = dependent ? 0.0 : t;
            int fn = 0;  // lowest free slot (at most qmax rows are in use: fn <= qmax, a valid slot)
            if (qmax <= 31) fn = __ffs(~amask[0]) - 1;
            else
              while (fn < qmax && ((amask[fn >> 5] >> (fn & 31)) & 1u)) fn++;
            flags[7] = fn;
          }
        }
        __syncthreads();
        const int decision = flags[4];
        if (decision >= 2) {
          // 4: "no step possible" for a row that is violated only at round-off level (at most 100 x the KKT tolerance): a
          // dependent row sitting on its bound (massively degenerate optima far outside the operating envelope,
          // tests/golden/stress_referee.npz).  It was the MOST violated row, so every row holds to that level: this is the
          // optimum, not an infeasible problem — whose violations are of the order of the data.
          if (decision == 4) { noise_stop = true; break; }
          code = (decision == 2) ? ST_INFEASIBLE : ST_WS_CAP;
          break;
        }
        const double t = dsc[0];
        // primal step direction z = t_p - sum_j r_j t_j, x += t z
        {
          // z = t_p - sum_j r_j t_j: cached columns directly, the slots beyond the cache through one H^-1 product of
          // A_W' r restricted to them (gq, padded to whole tiles, holds it; zb shares that memory: barriers in between)
          const int qhe = flags[8];
          const int qc = qhe < tcap ? qhe : tcap;
          double z = 0.0;
          if (isvar) {
            double z0 = Tf[vi], z1 = 0.0;
            int j = 0;
            for (; j + 1 < qc; j += 2) {
              z0 = fma(-rr[j], T[j * n + vi], z0);
              z1 = fma(-rr[j + 1], T[(j + 1) * n + vi], z1);
            }
            if (j < qc) z0 = fma(-rr[j], T[j * n + vi], z0);
            z = z0 + z1;
          }
          if (qhe > tcap) {
            if (isvar) {
              const int kb = vi / 6, c = vi - 6 * kb;
              double acc = 0.0;
              for (int j = tcap; j < qhe; j++) {
                const int w = wsl[j];
                if ((w >> 8) == kb) acc = fma(rr[j], nrm[(w & 0xff) * 6 + c], acc);
              }
              gq[vi] = acc;
            }
            __syncthreads();
            if (isvar) z -= hinv_rowdot(Hd, vi, NT8, gq);
            __syncthreads();
          }
          if (isvar) {
            zb[vi] = z;
            xreg = fma(t, z, xreg);
          }
        }
        __syncthreads();
        if (iscon && t != 0.0) se = fma(t, dot6(ne, zb + 6 * ke), se);
        if (decision == 0) {
          if (erow == p) { act = true; myslot = f; }
          q++;
          break;
        }
        // partial step: the blocking row left the working set; warp 0 needs the refreshed slack of p
        if (erow == flags[5]) { act = false; myslot = -1; }
        if (erow == p) dsc[1] = se;
        q--;
        __syncthreads();
        sp = dsc[1];
      }
      if (noise_stop) break;
    }

    HMPC_STAMP(5);
    // polish: x from scratch with the final multipliers, x = x0 + sum_j lam_j H^-1 a_j.
    // The explicit Schur-complement inverse drifts when many nearly dependent rows are active (massively degenerate
    // optima): large working sets get two rounds of refinement against the rows' own slacks at the composed x,
    // lam += S^-1 (d_W - A_W x), which vanish at the exact multipliers.  The usual ~N rows do not need it.
    __syncthreads();
    const int qhf = flags[9];
    // (after a noise-level stop the iterate itself is returned, like after a failure: the multipliers may lack the
    // partial one of the row that was being added, so x cannot be recomposed from them)
    const bool polish = code == ST_OK && !noise_stop;
    const int nref = (polish && q > 24) ? 2 : 0;
    for (int round = 0;; round++) {
      const bool beyond = polish && qhf > tcap;  // rows in slots without a cached column
      if (beyond) {
        if (isvar) {
          const int kb = vi / 6, c = vi - 6 * kb;
          double acc = 0.0;
          for (int j = tcap; j < qhf; j++) {
            const int w = wsl[j];
            if (((amask[j >> 5] >> (j & 31)) & 1u) && (w >> 8) == kb) acc = fma(lam[j], nrm[(w & 0xff) * 6 + c], acc);
          }
          gq[vi] = acc;
        }
        __syncthreads();
      }
      double xfin = xreg;
      if (isvar && polish) {
        xfin = x0[vi];
        const int qc = qhf < tcap ? qhf : tcap;
        for (int j = 0; j < qc; j++)
          if ((amask[j >> 5] >> (j & 31)) & 1u) xfin = fma(lam[j], T[j * n + vi], xfin);
        if (beyond) xfin += hinv_rowdot(Hd, vi, NT8, gq);
      }
      if (beyond) __syncthreads();  // zb shares gq's memory
      if (isvar) zb[vi] = xfin;
      __syncthreads();
      if (round == nref) break;
      if (wid == 0) {
        for (int s2 = lane; s2 < qhf; s2 += 32) {
          double acc = 0.0;
          if ((amask[s2 >> 5] >> (s2 & 31)) & 1u) {
            const int w = wsl[s2], ki = w >> 8, te = (w & 0xff) % 10;
            acc = ((te == 5) ? -(double)0.01f : ((te == 9) ? -fz[ki] : 0.0)) - dot6(nrm + (w & 0xff) * 6, zb + 6 * ki);
          }
          dvs[s2] = acc;
        }
        __syncwarp();
        for (int s2 = lane; s2 < qhf; s2 += 32) {
          if (!((amask[s2 >> 5] >> (s2 & 31)) & 1u)) continue;
          const int rs = tri(s2);
          double acc = 0.0;
          for (int j = 0; j < qhf; j++) acc = fma((j <= s2) ? Sv[rs + j] : Sv[tri(j) + s2], dvs[j], acc);
          lam[s2] = fmax(0.0, lam[s2] + acc);
        }
      }
      __syncthreads();
    }

    // working set for the next tick (closed loop): (step, leg) and normal index of every active row.  An instance that
    // overflowed this class's capacity is solved again (by the next class, or the host path's retry) from the same
    // proposal: it keeps the one it has.  The refinement class records an empty set: the next tick starts cold.
    if (ka.ws_state && wid == 0 && code != ST_WS_CAP) {
      int* ws = ka.ws_state + (size_t)inst * WS_STATE_INTS;
      const unsigned am = (code == ST_OK && qmax <= 31 && CLS != 3) ? amask[0] : 0u;
      if ((am >> lane) & 1u) {
        const int w = wsl[lane];
        ws[1 + __popc(am & ((1u << lane) - 1u))] = (blk_sl[w >> 8] << 8) | (w & 0xff);
      }
      if (lane == 0) ws[0] = __popc(am);
    }

    bool refined = false;
    if constexpr (CLS == 3) {
      // ---------------- refinement class: iterative refinement of the KKT solution against the stored Hessian ----------------
      // For a badly conditioned H the approximate operators of stages 4-5 (the sweep's H^-1, the explicit S^-1, x
      // recomposed from the multipliers) leave the optimum visibly off (DESIGN.md §2).  The float32 H and g are the QP's
      // exact data, so on the final working set W the KKT system  H x - A_W' lam = -g,  A_W x = d_W  is solved again by
      // iterative refinement: residuals in fp64 against the stored data, r_x = -(Hx + g - A_W' lam), r_lam = d_W - A_W x;
      // corrections through the same operators (range space): dlam = S^-1 (r_lam - A_W H^-1 r_x), dx = H^-1 (r_x + A_W' dlam).
      // At most four rounds; converged when a correction moves no component of x by more than the KKT tolerance.  The
      // answer is then accepted only at a KKT point: every multiplier >= -tol, every row feasible within tol.  Otherwise
      // (no convergence, or W itself is wrong) the instance keeps code 4.
      const float* Hc = reinterpret_cast<const float*>(smem + L.Hc);
      const double* gc = reinterpret_cast<const double*>(smem + L.gc);
      double* xr = x0;  // refined x (the unconstrained minimiser is spent)
      double* ub = gq;  // r_x, then r_x + A_W' dlam; zero-padded to whole tiles since stage 2 (zb, which shares it, moves to xr)
      double* yb = T;   // H^-1 r_x (the class has no column cache: T is one spare column of n)
      if (code == ST_OK) {
        if (isvar) xr[vi] = zb[vi];
        __syncthreads();
        bool conv = false, contracting = false;
        double dlast = 1e300;
        for (int round = 0; round < 4 && !conv; round++) {
          double rx = 0.0;
          if (isvar) {
            // row vi of the stored H (lower tiles, diagonal tiles complete) times x; A_W' lam restricted to the row's block
            const int I = vi >> 3, ir = vi & 7;
            double hx = 0.0;
            for (int j = 0; j < n; j++) {
              const int J = j >> 3;
              const float h = (J <= I) ? Hc[toff(I, J) + ir * 8 + (j & 7)] : Hc[toff(J, I) + (j & 7) * 8 + ir];
              hx = fma((double)h, xr[j], hx);
            }
            const int kb = vi / 6, c = vi - 6 * kb;
            double atl = 0.0;
            for (int j = 0; j < qhf; j++) {
              const int w = wsl[j];
              if (((amask[j >> 5] >> (j & 31)) & 1u) && (w >> 8) == kb) atl = fma(lam[j], nrm[(w & 0xff) * 6 + c], atl);
            }
            rx = DS(DS(atl, hx), gc[vi]);
            ub[vi] = rx;
          }
          if (wid == 0) {
            for (int s2 = lane; s2 < qhf; s2 += 32) {
              double acc = 0.0;
              if ((amask[s2 >> 5] >> (s2 & 31)) & 1u) {
                const int w = wsl[s2], ki = w >> 8, te = (w & 0xff) % 10;
                acc = ((te == 5) ? -(double)0.01f : ((te == 9) ? -fz[ki] : 0.0)) - dot6(nrm + (w & 0xff) * 6, xr + 6 * ki);
              }
              dvs[s2] = acc;  // r_lam
            }
          }
          __syncthreads();
          if (isvar) yb[vi] = hinv_rowdot(Hd, vi, NT8, ub);
          __syncthreads();
          if (wid == 0) {
            for (int s2 = lane; s2 < qhf; s2 += 32) {
              double acc = 0.0;
              if ((amask[s2 >> 5] >> (s2 & 31)) & 1u) {
                const int w = wsl[s2];
                acc = dvs[s2] - dot6(nrm + (w & 0xff) * 6, yb + 6 * (w >> 8));
              }
              rr[s2] = acc;  // r_lam - A_W H^-1 r_x
            }
            __syncwarp();
            for (int s2 = lane; s2 < qhf; s2 += 32) {
              double acc = 0.0;
              if ((amask[s2 >> 5] >> (s2 & 31)) & 1u) {
                const int rs = tri(s2);
                for (int j = 0; j < qhf; j++) acc = fma((j <= s2) ? Sv[rs + j] : Sv[tri(j) + s2], rr[j], acc);
              }
              dvs[s2] = acc;  // dlam
              lam[s2] += acc;
            }
          }
          __syncthreads();
          if (isvar) {
            const int kb = vi / 6, c = vi - 6 * kb;
            double acc = rx;
            for (int j = 0; j < qhf; j++) {
              const int w = wsl[j];
              if (((amask[j >> 5] >> (j & 31)) & 1u) && (w >> 8) == kb) acc = fma(dvs[j], nrm[(w & 0xff) * 6 + c], acc);
            }
            ub[vi] = acc;
          }
          __syncthreads();
          double dx = 0.0;
          if (isvar) {
            dx = hinv_rowdot(Hd, vi, NT8, ub);
            xr[vi] += dx;
          }
          {  // largest correction of the round (non-negative floats order like their bit patterns)
            const unsigned km = __reduce_max_sync(0xffffffffu, __float_as_uint((float)fabs(dx)));
            if (lane == 0) redk[16 + wid] = km;
          }
          __syncthreads();
          unsigned kx = redk[16];
          for (int w = 1; w < NW; w++) kx = redk[16 + w] > kx ? redk[16 + w] : kx;
          const double dmax = (double)__uint_as_float(kx);
          contracting = dmax <= 0.5 * dlast;
          dlast = dmax;
          conv = dmax <= tol;
        }
        // Accepted: converged, or after four rounds still contracting (each correction at most half the one before) with a
        // last correction below 1e-6 of the solution's scale — the error left is then smaller than that correction.  The
        // H^-1 of the sweep is the operator error that limits the rate: on h10_lying it contracts by ~0.08 per round.
        bool bad = !(conv || (contracting && dlast <= 1e3 * tol));
        if (iscon) bad |= dot6(ne, xr + 6 * ke) - rhs_e < -tol;
        if (wid == 0)
          for (int s2 = lane; s2 < qhf; s2 += 32) bad |= ((amask[s2 >> 5] >> (s2 & 31)) & 1u) && lam[s2] < -tol;
        refined = !__syncthreads_or((int)bad);
        if (isvar) zb[vi] = xr[vi];
        __syncthreads();
      }
      if (!refined) code = ST_NOT_SPD;  // not solved by refinement either: reported as today
    }

    // ---------------- stage 6: scatter (eliminated variables are exactly 0) ----------------
    for (int e = tid; e < 12 * N; e += NT) {
      const int s = e / 12, c12 = e % 12, leg = leg_of(c12);
      const int k = sl_blk[2 * s + leg];
      const double v = (k >= 0) ? zb[6 * k + loc_of(c12)] : 0.0;
      if (ka.wrench) ka.wrench[(size_t)row * 12 * N + e] = (float)v;
      if (ka.wrench64) ka.wrench64[(size_t)row * 12 * N + e] = v;
    }
    if (ka.tau && tid < 10) {
      // row f-2: tau = J_force_moment^T * f_ff, f_ff = -rBody [F; M] of the first-step wrench
      // (ConvexMPCLocomotion.cpp:419-440, LegController.cpp:57-63); swing legs get no feed-forward force
      const float* kp_ = reinterpret_cast<const float*>(smem + L.keep);
      const int leg = tid / 5, j = tid % 5;
      const double PI = 3.14159265359;
      double q5[5];
#pragma unroll
      for (int i = 0; i < 5; i++) q5[i] = (double)kp_[5 * leg + i];
      q5[2] -= 0.3 * PI;  // undo the caller's second offset: LegController's own angles
      q5[3] += 0.6 * PI;
      q5[4] -= 0.3 * PI;
      const double qw = kp_[10], qx = kp_[11], qy = kp_[12], qz = kp_[13];
      const double R[9] = {1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qw * qz), 2 * (qx * qz + qw * qy),
                           2 * (qx * qy + qw * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qw * qx),
                           2 * (qx * qz - qw * qy), 2 * (qy * qz + qw * qx), 1 - 2 * (qx * qx + qy * qy)};
      const int k0 = sl_blk[leg];  // step 0
      double fw[6] = {0, 0, 0, 0, 0, 0};
      if (k0 >= 0) {
        const double* w = zb + 6 * k0;
#pragma unroll
        for (int r = 0; r < 3; r++) {  // rBody = R^T
          fw[r] = -(R[0 * 3 + r] * (double)(float)w[0] + R[1 * 3 + r] * (double)(float)w[1] + R[2 * 3 + r] * (double)(float)w[2]);
          fw[3 + r] = -(R[0 * 3 + r] * (double)(float)w[3] + R[1 * 3 + r] * (double)(float)w[4] + R[2 * 3 + r] * (double)(float)w[5]);
        }
      }
      ka.tau[(size_t)inst * 10 + tid] = (float)leg_torque(q5, leg, j, fw);
    }
    HMPC_STAMP(6);
    if (tid == 0) {
      if (code == ST_WS_CAP && ka.esc_list) {  // hand over to the next class (larger working-set capacity)
        const int slot = atomicAdd(&ka.counts[ka.cls + 1], 1);
        ka.esc_list[slot] = row;
      }
      if (code == ST_NOT_SPD && flags[3] == ST_OK && ka.ref_list) {  // beyond the conditioning limit, every pivot positive
        const int slot = atomicAdd(ka.ref_count, 1);
        ka.ref_list[slot] = row;
      }
      int sw = (code & 0xff) | ((iters & 0xfff) << 8) | ((q & 0xff) << 20);
      if constexpr (CLS == 3) sw |= refined ? (1 << 28) : 0;  // HMPC_STATUS_REFINED
      ka.status[row] = sw;
    }
    __syncthreads();
    if constexpr (MQ) {
      if (++kq < k1) goto next_candidate;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Masked solve (hmpc_solve_device_masked): robot i is solved iff mask[i] != 0.  This kernel turns the mask into class 0's
// instance list, in ascending robot order, and its length word.  One CTA scans the mask in tiles of NT bytes: a ballot
// and popc inside each warp, the warp totals through shared memory across warps.  A single CTA writes the list in order
// without a second pass, and it runs as it is in the host emulation.  At 4096 robots it is 8 tiles.
// ------------------------------------------------------------------------------------------------
constexpr int SELECT_THREADS = 512;

template <int NT>
__global__ void __launch_bounds__(NT) hmpc_select_kernel(const unsigned char* mask, int batch, int* list, int* count)
{
  constexpr int NW = NT / 32;
  __shared__ int wtot[NW];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  pdl_trigger();  // class 0 may become resident; it waits for this kernel before it reads the list
  // The previous call's class-0 launch clears the length words this call uses, and the kernel before this one may have
  // written the mask: nothing is read or stored before both have completed.
  pdl_wait();
  int base = 0;
  for (int t0 = 0; t0 < batch; t0 += NT) {
    const int i = t0 + tid;
    const bool on = i < batch && mask[i] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, on);
    if (lane == 0) wtot[wid] = __popc(bal);
    __syncthreads();
    int off = base, tot = 0;
    for (int w = 0; w < NW; w++) {
      const int n = wtot[w];
      off += w < wid ? n : 0;
      tot += n;
    }
    if (on) list[off + __popc(bal & ((1u << lane) - 1u))] = i;
    base += tot;
    __syncthreads();  // the next tile rewrites wtot
  }
  if (tid == 0) *count = base;
}

// ------------------------------------------------------------------------------------------------
// Sharded masked calls (hmpc_solve_batch_sharded_warm): the gather sends every robot's latest float wrench row, but the
// solve writes only the listed rows of this tick's buffer.  This kernel copies the unlisted rows from the previous tick's
// buffer, one 16-byte vector per thread (a row of 12N floats is 3N vectors).  It writes no row the solve writes, so it
// needs no ordering against the solve chain.  Launch shape: hmpc_chain.h, carry_grid.
// ------------------------------------------------------------------------------------------------
constexpr int CARRY_THREADS = 256;

__global__ void __launch_bounds__(CARRY_THREADS) hmpc_carry_kernel(const unsigned char* mask, int batch, int row_vecs,
                                                                    const float4* prev, float4* cur)
{
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= (long long)batch * row_vecs) return;
  if (mask[v / row_vecs] == 0) cur[v] = prev[v];
}

// ------------------------------------------------------------------------------------------------
// The MPC's plan (hmpc_predict_device, hmpc_predict_batch): robot i's predicted states x_{k+1} = Acd x_k + Bcd u_k,
// k = 0..N-1, under the discrete model its QP was built from.  x_0, Acd and Bcd come from stage 1's own role_state and
// role_inertia (float32, bit for bit the solve kernel's); u_k is wrench row entries [12k, 12k+12).  One warp per robot: the
// roles run on the warp into its shared scratch, then lane r < 12 owns state component r through the N steps and reads the
// others by shuffle.  The recurrence is float64 with separately rounded operations in a fixed order, row r:
//   x_{k+1}[r] = x_k[r] + sum over the row's off-diagonal entries of Acd (ascending column, the gravity state last)
//                       + sum over the row's entries of Bcd (ascending column)
// where a row's entries are its structural ones: Acd is the identity plus dt*Rb (rows 0-2, columns 6-8), dt (rows 3-5,
// columns 9-11) and -dt (row 11, column 12); Bcd fills rows 6-8 and two entries (i, i+3) of rows 9-11.  The gravity state
// x[12] = 9.81f never changes and is not written.  Rows are read from `rows` with stride `row_stride`: only the first 19
// floats (p v q w r), which lie at the same offsets in a packed record and in an update_data_t.  T is the element type of
// the wrench in and the prediction out [B][N][12].  Robots with mask[i] == 0 (mask non-null) are skipped.  Launch shape:
// hmpc_chain.h, predict_grid.
// ------------------------------------------------------------------------------------------------
// One row of the plan's recurrence, x_{k+1}[r] = x_k[r] + (Acd x_k)[r] off the diagonal + (Bcd u_k)[r], on lane r < 12 of a
// warp whose lane j holds x_k[j] (j < 13) and u_k[j] (j < 12): nx entries of Acd on states xs[t], nu entries of Bcd on
// wrench entries us[t], in the order the comment of hmpc_predict_kernel gives.  ABS: the same sums over |Acd| and |Bcd|
// (the caller passes |x| and |u|), the magnitude of the terms a state is formed from.  step() is called by the whole warp.
template <bool ABS>
struct PlanRow {
  int nx, nu, xs[3], us[12];
  double ax[3], bu[12];
  __device__ __forceinline__ PlanRow(const float* Acd, const float* Bcd, int lane)
  {
    const int r = lane < 12 ? lane : 0;
    nx = r < 3 ? 3 : (r < 6 || r == 11) ? 1 : 0;
    nu = (r >= 6 && r < 9) ? 12 : (r >= 9 ? 2 : 0);
#pragma unroll
    for (int t = 0; t < 3; t++) {
      xs[t] = r < 3 ? 6 + t : (r < 6 ? r + 6 : 12);
      ax[t] = t < nx ? (double)Acd[r * 13 + xs[t]] : 0.0;
      if (ABS) ax[t] = fabs(ax[t]);
    }
#pragma unroll
    for (int t = 0; t < 12; t++) {
      us[t] = r < 9 ? t : (t == 0 ? r - 9 : r - 6);
      bu[t] = t < nu ? (double)Bcd[r * 12 + us[t]] : 0.0;
      if (ABS) bu[t] = fabs(bu[t]);
    }
  }
  __device__ __forceinline__ double step(double x, double u) const
  {
    double acc = x;
#pragma unroll
    for (int t = 0; t < 3; t++) {
      const double v = __shfl_sync(0xffffffffu, x, xs[t]);
      if (t < nx) acc = DA(acc, DM(ax[t], v));
    }
#pragma unroll
    for (int t = 0; t < 12; t++) {
      const double v = __shfl_sync(0xffffffffu, u, us[t]);
      if (t < nu) acc = DA(acc, DM(bu[t], v));
    }
    return acc;
  }
};

// The tracking cost of a plan, J = sum_k (x_{k+1} - traj_k)' S (x_{k+1} - traj_k) + u_k' alpha u_k, in float64 on lane r < 12:
// cost_step after each step of the recurrence (x = x_{k+1}[r], xd = traj_k[r], u = u_k[r]), then cost_total on the whole warp
// adds the twelve lanes' sums in lane order.  The certificate's cost and the multi-query call's cost are these.
__device__ __forceinline__ double cost_step(double cost, double S, double Al, double x, double xd, double u)
{
  const double e = DS(x, xd);
  cost = DA(cost, DM(DM(S, e), e));
  return DA(cost, DM(DM(Al, u), u));
}
__device__ __forceinline__ double cost_total(double cost)
{
  double J = 0.0;
  for (int r = 0; r < 12; r++) J = DA(J, __shfl_sync(0xffffffffu, cost, r));
  return J;
}

constexpr int PREDICT_THREADS = 128;
constexpr int PREDICT_WARP_BYTES = 1440;  // per warp: role scratch 64 B | x0 16 floats | Acd 169 | Bcd 156 floats

template <typename T>
__global__ void __launch_bounds__(PREDICT_THREADS) hmpc_predict_kernel(const unsigned char* rows, int row_stride, int batch,
                                                                        int N, float dt, const unsigned char* mask,
                                                                        const T* wrench, T* pred)
{
  constexpr int NW = PREDICT_THREADS / 32;
  __shared__ __align__(16) unsigned char scratch[NW * PREDICT_WARP_BYTES];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int i = blockIdx.x * NW + wid;
  if (i >= batch || (mask && mask[i] == 0)) return;  // (the whole warp)
  unsigned char* scr = scratch + wid * PREDICT_WARP_BYTES;
  float* x0f = reinterpret_cast<float*>(scr + 64);
  float* Acd = x0f + 16;
  float* Bcd = Acd + 169;  // (not zeroed: the roles write every entry read below)
  const float* rf = reinterpret_cast<const float*>(rows + (size_t)i * row_stride);
  role_state(rf, dt, x0f, Acd, lane, scr);
  if (lane == 31) role_inertia(rf, dt, Bcd);
  __syncwarp();
  const PlanRow<false> row(Acd, Bcd, lane);
  double x = lane < 13 ? (double)x0f[lane] : 0.0;
  const T* w = wrench + (size_t)i * 12 * N;
  T* out = pred + (size_t)i * 12 * N;
  for (int k = 0; k < N; k++) {
    const double u = lane < 12 ? (double)w[12 * k + lane] : 0.0;
    const double acc = row.step(x, u);
    if (lane < 12) {
      x = acc;
      out[12 * k + lane] = (T)acc;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// The certificate (hmpc_certify_device, hmpc_certify_batch): a first-order optimality check of robot i's wrench U for its
// row, independent of the solve.  One warp per robot, four per CTA (hmpc_chain.h: certify_grid).
//   1. Roles: stage 1's role_leg, role_state and role_inertia into the warp's scratch: Fblk, x0, Acd and Bcd, the solve's
//      float32 values bit for bit.
//   2. Plan and cost: the recurrence of hmpc_predict_kernel (PlanRow), lane r < 12 owning state r, and beside it the same
//      recurrence on |x0|, |Acd|, |Bcd|, |u|.  Lane r accumulates its cost terms in float64, step by step:
//        c_r += (S_r e) e,  then  c_r += (alpha_r u) u,     e = x_{k+1}[r] - traj_k[r],  u = u_k[r]
//      and J = c_0 + c_1 + ... + c_11 in that order: the QP objective 1/2 U'HU + g'U plus the constant d'Sd.
//   3. Gradient: the adjoint sweep from k = N down to 1, p_{N+1} = 0, lane j:
//        p_k[j] = p_{k+1}[j] + Acd[r][j] p_{k+1}[r] over column j's off-diagonal rows (ascending) + (2 S_j) e_k[j]
//        grad u_{k-1}[c] = 0 + Bcd[r][c] p_k[r] over column c's rows (ascending) + (2 alpha_c) u_{k-1}[c]
//      and the same sweep over the absolute values gives each entry the magnitude of its terms; the largest of them over
//      the stance legs' entries is the robot's gradient scale.
//   4. Multipliers: lane b < 2N owns block (step b/2, leg b%2).  A swing leg's six entries must be exactly 0.  A stance
//      leg's 8 rows of Fblk, with stage 1's bounds (friction >= 0; 0 <= Mx <= 0.01; line contact <= 0; 0 <= Fz <= f_max
//      gait; 5e10 means none), are candidates when their slack to a bound is within CERT_ACT_K eps P + CERT_ACT_ABS
//      (eps: float32's, the precision of the rows; P: the robot's row scale below).  The block's gradient is fitted by the candidate rows with sign-constrained multipliers (>= 0 at a
//      lower bound, <= 0 at an upper one) by Lawson-Hanson (cert_nnls), in float64 on the lane.
//   5. Measures: stationarity = max |grad - A'lambda| / gradient scale; primal = the worst bound violation or non-zero
//      swing entry / the largest sum |a||u| of the stance rows; complementarity = max |lambda| slack / (both scales).
//      Thresholds CERT_*_TOL (DESIGN.md §7): the pass bit needs all three under them and finite inputs.
// Rows are read through `lay` (hmpc_chain.h: packed_rows, update_rows).  T: wrench in and multipliers out (float: device
// call, double: host call).  cert [B]; lambda NULL or [B][N][2][8] (signed, zero off the candidate rows and on swing
// legs); grad NULL or [B][12N] (the gradient, for the kernel-source tests).  Robots with mask[i] == 0 are skipped.
// ------------------------------------------------------------------------------------------------
constexpr int CERT_THREADS = 128;
constexpr int CERT_NMAX = 16;
// per warp: role scratch 320 B | x0 16 floats | Acd 172 | Bcd 156 | Fblk 192 floats | plan, |plan|, gradient 3 x 192 doubles
constexpr int CERT_WARP_BYTES = 320 + 4 * (16 + 172 + 156 + 192) + 3 * 8 * 12 * CERT_NMAX;
// Candidate rows: slack <= CERT_ACT_K eps P + CERT_ACT_ABS, P the robot's row scale (the largest sum |a||u| of its stance
// rows) and eps the float32 epsilon whatever T is: the rows and bounds are float32, so a row's value is defined to that
// rounding whatever precision the wrench carries, and a solver holds its rows to its tolerance relative to the whole
// problem, not to each foot's force: a foot at zero force comes back at ~1e-12 N (DESIGN.md §7).
constexpr double CERT_EPS_ROWS = 1.1920928955078125e-07;
constexpr double CERT_ACT_K = 64.0;
constexpr double CERT_ACT_ABS = 1e-12;
constexpr double CERT_NNLS_DUAL = 1e-14;   // a row enters when its dual exceeds this times max |grad| of the block
constexpr int CERT_NNLS_ITERS = 64;        // Lawson-Hanson's outer iterations (a block has at most 6 independent rows)
constexpr double CERT_NNLS_PIVOT = 1e-10;  // a row whose pivot falls below this times its norm^2 is dependent: left out
constexpr double CERT_TINY = 1e-300;
constexpr double CERT_STAT_TOL = 2e-6;     // (DESIGN.md §7: margins over the measured floors)
constexpr double CERT_PRIMAL_TOL = 2e-7;
constexpr double CERT_COMPL_TOL = 1e-9;
enum : int { CERT_PASS = 1, CERT_NONFINITE = 2, CERT_SWING = 4, CERT_STATIONARITY = 8, CERT_PRIMAL = 16, CERT_COMPL = 32 };

// where a row's Alpha_K, traj and gait bytes lie (byte offsets; the first 42 floats are common to both layouts)
struct RowLayout {
  int stride, alpha, traj, gait;
};
// one robot's certificate (include/hector_mpc_b200.h: hmpc_certificate_t)
struct CertOut {
  double cost, stationarity, primal, complementarity;
  int n_active, flags;
};

__device__ __forceinline__ bool finite64(double x) { return fabs(x) <= 1.7976931348623157e308; }
__device__ __forceinline__ double warp_max64(double v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// min ||Z z - b|| over z restricted to the rows in bitmask P (Z: k rows of 6), by LDL' of the normal equations in a fixed
// order; false when a pivot falls below CERT_NNLS_PIVOT times its diagonal (the rows in P are dependent)
__device__ inline bool cert_ls(const double (*Z)[6], int k, unsigned P, const double* b, double* z)
{
  int p[8], np = 0;
  for (int t = 0; t < k; t++)
    if (P >> t & 1u) p[np++] = t;
  double L[8][8], D[8], h[8];
  for (int q = 0; q < np; q++) {
    double hq = 0.0;
    for (int c = 0; c < 6; c++) hq = DA(hq, DM(Z[p[q]][c], b[c]));
    h[q] = hq;
    for (int r = 0; r <= q; r++) {
      double g = 0.0;
      for (int c = 0; c < 6; c++) g = DA(g, DM(Z[p[q]][c], Z[p[r]][c]));
      for (int t = 0; t < r; t++) g = DS(g, DM(DM(L[q][t], L[r][t]), D[t]));
      if (r < q) {
        L[q][r] = g / D[r];
      } else {
        double gqq = 0.0;
        for (int c = 0; c < 6; c++) gqq = DA(gqq, DM(Z[p[q]][c], Z[p[q]][c]));
        if (!(g > DM(CERT_NNLS_PIVOT, gqq))) return false;
        D[q] = g;
      }
    }
  }
  for (int q = 0; q < np; q++) {
    double v = h[q];
    for (int t = 0; t < q; t++) v = DS(v, DM(L[q][t], h[t]));
    h[q] = v;
  }
  for (int q = 0; q < np; q++) h[q] = h[q] / D[q];
  for (int q = np - 1; q >= 0; q--) {
    double v = h[q];
    for (int t = q + 1; t < np; t++) v = DS(v, DM(L[t][q], h[t]));
    h[q] = v;
  }
  for (int t = 0; t < k; t++) z[t] = 0.0;
  for (int q = 0; q < np; q++) z[p[q]] = h[q];
  return true;
}

// Lawson-Hanson: y >= 0 minimising ||Z'y - b|| over the k <= 8 rows of Z (one block's sign-flipped candidate rows)
__device__ inline void cert_nnls(const double (*Z)[6], int k, const double* b, double* y)
{
  unsigned P = 0u, out = 0u;
  double bmax = 0.0;
  for (int c = 0; c < 6; c++) bmax = fmax(bmax, fabs(b[c]));
  const double tol = DM(CERT_NNLS_DUAL, bmax);
  for (int t = 0; t < 8; t++) y[t] = 0.0;
  for (int it = 0; it < CERT_NNLS_ITERS; it++) {
    double r[6];
    for (int c = 0; c < 6; c++) {
      double v = b[c];
      for (int t = 0; t < k; t++)
        if (P >> t & 1u) v = DS(v, DM(Z[t][c], y[t]));
      r[c] = v;
    }
    int best = -1;
    double wb = tol;
    for (int t = 0; t < k; t++) {
      if ((P | out) >> t & 1u) continue;
      double w = 0.0;
      for (int c = 0; c < 6; c++) w = DA(w, DM(Z[t][c], r[c]));
      if (w > wb) {
        wb = w;
        best = t;
      }
    }
    if (best < 0) break;
    P |= 1u << best;
    for (int inner = 0; inner < 8; inner++) {
      double z[8];
      // a row dependent on P, or one whose own multiplier comes out <= 0 (rounding), is left out until P changes
      if (!cert_ls(Z, k, P, b, z) || (inner == 0 && !(z[best] > 0.0))) {
        P &= ~(1u << best);
        out |= 1u << best;
        break;
      }
      out = 0u;
      bool pos = true;
      for (int t = 0; t < k; t++)
        if ((P >> t & 1u) && !(z[t] > 0.0)) pos = false;
      if (pos) {
        for (int t = 0; t < k; t++) y[t] = (P >> t & 1u) ? z[t] : 0.0;
        break;
      }
      double a = 2.0;
      int tmin = -1;
      for (int t = 0; t < k; t++)
        if ((P >> t & 1u) && !(z[t] > 0.0)) {
          const double at = y[t] / DS(y[t], z[t]);
          if (at < a) {
            a = at;
            tmin = t;
          }
        }
      if (tmin < 0) break;  // (non-finite z)
      for (int t = 0; t < k; t++)
        if (P >> t & 1u) y[t] = DA(y[t], DM(a, DS(z[t], y[t])));
      y[tmin] = 0.0;
      for (int t = 0; t < k; t++)
        if ((P >> t & 1u) && !(y[t] > 0.0)) {
          P &= ~(1u << t);
          y[t] = 0.0;
        }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(CERT_THREADS) hmpc_certify_kernel(const unsigned char* rows, RowLayout lay, int batch, int N,
                                                                     float dt, float f_max, const unsigned char* mask,
                                                                     const T* wrench, CertOut* cert, T* lambda, double* grad)
{
  constexpr int NW = CERT_THREADS / 32;
  __shared__ __align__(16) unsigned char scratch[NW * CERT_WARP_BYTES];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int i = blockIdx.x * NW + wid;
  if (i >= batch || (mask && mask[i] == 0)) return;  // (the whole warp)
  unsigned char* scr = scratch + wid * CERT_WARP_BYTES;
  float* x0f = reinterpret_cast<float*>(scr + 320);
  float* Acd = x0f + 16;
  float* Bcd = Acd + 172;
  float* Fblk = Bcd + 156;
  double* X = reinterpret_cast<double*>(Fblk + 192);  // [N][12] x_{k+1}
  double* XA = X + 12 * CERT_NMAX;                     // [N][12] the plan on absolute values
  double* G = XA + 12 * CERT_NMAX;                     // [N][12] the gradient
  const unsigned char* row = rows + (size_t)i * lay.stride;
  const float* rf = reinterpret_cast<const float*>(row);
  const float* alpha = reinterpret_cast<const float*>(row + lay.alpha);
  const float* traj = reinterpret_cast<const float*>(row + lay.traj);
  const unsigned char* gait = row + lay.gait;
  const T* w = wrench + (size_t)i * 12 * N;

  // ---- 1. the roles
  for (int e = lane; e < 192; e += 32) Fblk[e] = 0.f;
  __syncwarp();
  role_leg(rf, lane, Fblk, scr);
  __syncwarp();
  role_state(rf, dt, x0f, Acd, lane, scr + 256);
  if (lane == 31) role_inertia(rf, dt, Bcd);
  __syncwarp();

  // ---- 2. plan, its absolute-value twin and the cost
  const int j = lane < 12 ? lane : 0;
  const double S = (double)rf[30 + j], Al = (double)alpha[j];
  bool fin = true;
  double cost = 0.0;
  {
    const PlanRow<false> pr(Acd, Bcd, lane);
    const PlanRow<true> pa(Acd, Bcd, lane);
    double x = lane < 13 ? (double)x0f[lane] : 0.0, xa = fabs(x);
    for (int k = 0; k < N; k++) {
      const double u = lane < 12 ? (double)w[12 * k + lane] : 0.0;
      const double nx = pr.step(x, u), na = pa.step(xa, fabs(u));
      if (lane < 12) {
        x = nx;
        xa = na;
        X[12 * k + lane] = x;
        XA[12 * k + lane] = xa;
        cost = cost_step(cost, S, Al, x, (double)traj[12 * k + lane], u);
        fin = fin && finite64(u) && finite64(x);
      }
    }
  }
  const double J = cost_total(cost);
  __syncwarp();

  // ---- 3. the adjoint sweep and the gradient
  double gscale = 0.0;
  {
    const int pn = (j >= 6 && j < 9) ? 3 : (j >= 9 ? 1 : 0);  // column j of Acd off the diagonal: rows ps[t]
    const int bn = j < 6 ? 4 : 3;                               // column j of Bcd: rows bs[t]
    int ps[3], bs[4];
    double at[3], bt[4];
#pragma unroll
    for (int t = 0; t < 3; t++) {
      ps[t] = j < 9 ? t : j - 6;
      at[t] = t < pn ? (double)Acd[ps[t] * 13 + j] : 0.0;
    }
#pragma unroll
    for (int t = 0; t < 4; t++) {
      bs[t] = t < 3 ? 6 + t : 9 + j % 3;
      bt[t] = t < bn ? (double)Bcd[bs[t] * 12 + j] : 0.0;
    }
    const double S2 = DM(2.0, S), A2 = DM(2.0, Al);
    const int legj = leg_of(j);
    double p = 0.0, q = 0.0;
    for (int k = N; k >= 1; k--) {
      double acc = p, acca = q;
#pragma unroll
      for (int t = 0; t < 3; t++) {
        const double v = __shfl_sync(0xffffffffu, p, ps[t]), va = __shfl_sync(0xffffffffu, q, ps[t]);
        if (t < pn) {
          acc = DA(acc, DM(at[t], v));
          acca = DA(acca, DM(fabs(at[t]), va));
        }
      }
      const int o = 12 * (k - 1) + j;
      const double xd = (double)traj[o];
      p = DA(acc, DM(S2, DS(X[o], xd)));
      q = DA(acca, DM(fabs(S2), DA(XA[o], fabs(xd))));
      double g = 0.0, ga = 0.0;
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const double v = __shfl_sync(0xffffffffu, p, bs[t]), va = __shfl_sync(0xffffffffu, q, bs[t]);
        if (t < bn) {
          g = DA(g, DM(bt[t], v));
          ga = DA(ga, DM(fabs(bt[t]), va));
        }
      }
      const double u = (double)w[o];
      g = DA(g, DM(A2, u));
      ga = DA(ga, DM(fabs(A2), fabs(u)));
      if (lane < 12) {
        G[o] = g;
        if (grad) grad[(size_t)i * 12 * N + o] = g;
        const float fz = FM(f_max, (float)gait[2 * (k - 1) + legj]);
        if (!(fz < 0.0001f && fz > -0.0001f)) gscale = fmax(gscale, ga);
        fin = fin && finite64(g) && finite64(ga);
      }
    }
  }
  __syncwarp();

  // ---- 4. one lane per (step, leg) block: rows, candidates, multipliers
  double stat = 0.0, prim = 0.0, comp = 0.0, pscale = 0.0;
  int nact = 0;
  bool swing_bad = false;
  const bool blk = lane < 2 * N;
  const int s = lane >> 1, leg = lane & 1;
  const float fz = blk ? FM(f_max, (float)gait[2 * s + leg]) : 0.f;
  const bool stance = blk && !(fz < 0.0001f && fz > -0.0001f);
  double u[6], v[8];
  for (int c = 0; c < 6; c++) u[c] = blk ? (double)w[12 * s + col12_of(leg, c)] : 0.0;
  if (stance) {
    for (int t = 0; t < 8; t++) {
      double vt = 0.0, rs = 0.0;
      for (int c = 0; c < 6; c++) {
        const double a = (double)Fblk[(8 * leg + t) * 12 + col12_of(leg, c)];
        vt = DA(vt, DM(a, u[c]));
        rs = DA(rs, DM(fabs(a), fabs(u[c])));
      }
      fin = fin && finite64(vt) && finite64(rs);
      pscale = fmax(pscale, rs);
      v[t] = vt;
    }
  }
  pscale = warp_max64(pscale);
  const double tol = DA(DM(DM(CERT_ACT_K, CERT_EPS_ROWS), pscale), CERT_ACT_ABS);
  if (blk) {
    T* lam = lambda ? lambda + (((size_t)i * N + s) * 2 + leg) * 8 : nullptr;
    if (lam)
      for (int t = 0; t < 8; t++) lam[t] = (T)0;
    if (!stance) {
      for (int c = 0; c < 6; c++)
        if (u[c] != 0.0) {
          swing_bad = true;
          prim = fmax(prim, fabs(u[c]));
        }
    } else {
      double Z[8][6], y[8], sl[8], gb[6];
      int rowof[8], k = 0;
      bool up[8];
      for (int c = 0; c < 6; c++) gb[c] = G[12 * s + col12_of(leg, c)];
      for (int t = 0; t < 8; t++) {
        const bool haslo = t < 5 || t == 7, hashi = t >= 4;
        const double hi = t == 4 ? (double)0.01f : (t == 7 ? (double)fz : 0.0);
        const double slo = haslo ? v[t] : 1e300, shi = hashi ? DS(hi, v[t]) : 1e300;  // (lower bounds are 0)
        prim = fmax(prim, fmax(-slo, -shi));
        const bool atlo = slo <= tol, athi = shi <= tol;
        if (atlo || athi) {
          const bool upper = athi && (!atlo || shi < slo);
          for (int c = 0; c < 6; c++) {
            const double a = (double)Fblk[(8 * leg + t) * 12 + col12_of(leg, c)];
            Z[k][c] = upper ? -a : a;
          }
          sl[k] = fabs(upper ? shi : slo);
          up[k] = upper;
          rowof[k++] = t;
        }
      }
      cert_nnls(Z, k, gb, y);
      nact = k;
      double res[6];
      for (int c = 0; c < 6; c++) res[c] = gb[c];
      for (int t = 0; t < k; t++)
        for (int c = 0; c < 6; c++) res[c] = DS(res[c], DM(y[t], Z[t][c]));
      for (int c = 0; c < 6; c++) stat = fmax(stat, fabs(res[c]));
      for (int t = 0; t < k; t++) {
        comp = fmax(comp, DM(y[t], sl[t]));
        if (lam) lam[rowof[t]] = (T)(up[t] ? -y[t] : y[t]);
      }
    }
  }

  // ---- 5. the robot's measures
  gscale = warp_max64(gscale);
  stat = warp_max64(stat);
  prim = warp_max64(prim);
  comp = warp_max64(comp);
  for (int o = 16; o > 0; o >>= 1) nact += __shfl_xor_sync(0xffffffffu, nact, o);
  const bool any_swing = __any_sync(0xffffffffu, swing_bad);
  const bool all_fin = !__any_sync(0xffffffffu, !fin) && finite64(J);
  if (lane == 0) {
    CertOut c;
    const double gs = fmax(gscale, CERT_TINY), pss = fmax(pscale, CERT_TINY);
    c.cost = J;
    c.stationarity = stat / gs;
    c.primal = prim / pss;
    c.complementarity = comp / DM(gs, pss);
    c.n_active = nact;
    int f = 0;
    if (!all_fin) f |= CERT_NONFINITE;
    if (any_swing) f |= CERT_SWING;
    if (!(c.stationarity <= CERT_STAT_TOL)) f |= CERT_STATIONARITY;
    if (!(c.primal <= CERT_PRIMAL_TOL)) f |= CERT_PRIMAL;
    if (!(c.complementarity <= CERT_COMPL_TOL)) f |= CERT_COMPL;
    if (f == 0) f = CERT_PASS;
    c.flags = f;
    cert[i] = c;
  }
}

// ------------------------------------------------------------------------------------------------
// The cost of the multi-query call (hmpc_solve_device_multi, hmpc_solve_batch_multi): for row q = i*K + k, the certificate's
// tracking cost J (cost_step, cost_total; hmpc_certify_kernel, step 2) of wrench row q on robot i's row of `rows` (layout
// `lay`) with the reference trajectory traj[q] [12N] in place of the row's own.  One warp per row: stage 1's role_state and
// role_inertia, then the plan's recurrence (PlanRow), as hmpc_predict_kernel runs them.  Robots with mask[i] == 0 (mask
// non-null) are skipped.  T: the wrench's element type.  Launch shape: hmpc_chain.h, multi_cost_grid.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(PREDICT_THREADS) hmpc_multi_cost_kernel(const unsigned char* rows, RowLayout lay, int batch,
                                                                           int K, int N, float dt, const unsigned char* mask,
                                                                           const float* traj, const T* wrench, double* cost)
{
  constexpr int NW = PREDICT_THREADS / 32;
  __shared__ __align__(16) unsigned char scratch[NW * PREDICT_WARP_BYTES];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long q = (long long)blockIdx.x * NW + wid;
  if (q >= (long long)batch * K) return;  // (the whole warp)
  const int i = (int)(q / K);
  if (mask && mask[i] == 0) return;
  unsigned char* scr = scratch + wid * PREDICT_WARP_BYTES;
  float* x0f = reinterpret_cast<float*>(scr + 64);
  float* Acd = x0f + 16;
  float* Bcd = Acd + 169;  // (not zeroed: the roles write every entry read below)
  const unsigned char* row = rows + (size_t)i * lay.stride;
  const float* rf = reinterpret_cast<const float*>(row);
  const float* alpha = reinterpret_cast<const float*>(row + lay.alpha);
  const float* xd = traj + (size_t)q * 12 * N;
  const T* w = wrench + (size_t)q * 12 * N;
  role_state(rf, dt, x0f, Acd, lane, scr);
  if (lane == 31) role_inertia(rf, dt, Bcd);
  __syncwarp();
  const PlanRow<false> pr(Acd, Bcd, lane);
  const int j = lane < 12 ? lane : 0;
  const double S = (double)rf[30 + j], Al = (double)alpha[j];
  double x = lane < 13 ? (double)x0f[lane] : 0.0, c = 0.0;
  for (int k = 0; k < N; k++) {
    const double u = lane < 12 ? (double)w[12 * k + lane] : 0.0;
    const double nx = pr.step(x, u);
    if (lane < 12) {
      x = nx;
      c = cost_step(c, S, Al, x, (double)xd[12 * k + lane], u);
    }
  }
  const double J = cost_total(c);
  if (lane == 0) cost[q] = J;
}

// ------------------------------------------------------------------------------------------------
// The pick of a multi-command states call (hmpc_solve_states_device_multi), behind its cost kernel: per robot i, best[i] =
// the k with the smallest cost[i][k] among the candidates whose status code is 0 and whose cost is finite, the lowest such k
// on ties, or -1 when there is none.  Then robot i's torque row: joint_torque on the record's joint angles and quaternion and
// the chosen candidate's step-0 wrench, what the solve's epilogue gives that candidate's expanded row (zeros for -1).  Last
// the record's traj is set to the chosen candidate's, traj[i][best] (candidate 0 for -1), so the record is the one
// hmpc_prepare_kernel writes for the chosen command.  One warp per robot; robots with mask[i] == 0 (mask non-null) are
// skipped; tau may be null.  T: the wrench's element type.  Launch shape: hmpc_chain.h, pick_grid.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(PREDICT_THREADS) hmpc_pick_kernel(unsigned char* records, int rec_stride, int batch, int K,
                                                                     int N, float f_max, const unsigned char* mask,
                                                                     const float* traj, const T* wrench, const int* status,
                                                                     const double* cost, int* best, float* tau)
{
  constexpr int NW = PREDICT_THREADS / 32;
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * NW + (threadIdx.x >> 5);
  if (i >= batch || (mask && mask[i] == 0)) return;  // (the whole warp)
  const size_t r0 = (size_t)i * K;
  double bc = 0.0;
  int bk = -1;
  for (int k = lane; k < K; k += 32)  // (ascending k: a tie keeps the lower one)
    if ((status[r0 + k] & 0xff) == 0 && finite64(cost[r0 + k]) && (bk < 0 || cost[r0 + k] < bc)) bc = cost[r0 + k], bk = k;
  for (int o = 16; o > 0; o >>= 1) {
    const double oc = __shfl_xor_sync(0xffffffffu, bc, o);
    const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
    if (ok >= 0 && (bk < 0 || oc < bc || (oc == bc && ok < bk))) bc = oc, bk = ok;
  }
  float* f = reinterpret_cast<float*>(records + (size_t)i * rec_stride);
  const float* src = traj + (r0 + (bk < 0 ? 0 : bk)) * 12 * N;
  if (tau && lane < 10) {
    float t = 0.f;
    if (bk >= 0) {
      const int leg = lane / 5, j = lane % 5;
      const float ub = FM(f_max, (float)(records + (size_t)i * rec_stride + (54 + 12 * N) * 4)[leg]);  // step 0's gait byte
      const T* w = wrench + (r0 + bk) * 12 * N;
      T w6[6];
      for (int c = 0; c < 6; c++) w6[c] = w[col12_of(leg, c)];
      t = joint_torque(f + 19, f + 6, leg, j, (ub < 0.0001f && ub > -0.0001f) ? nullptr : w6);  // (stage 1's swing test)
    }
    tau[(size_t)i * 10 + lane] = t;
  }
  __syncwarp();  // (the torques read the record's floats 6-28, the copy below writes 54 on)
  for (int e = lane; e < 12 * N; e += 32) f[54 + e] = src[e];
  if (lane == 0) best[i] = bk;
}

}  // namespace hmpc
