/*
 * hector_mpc_b200.h — C-ABI of libhector_mpc_b200.so
 *
 * An H100 (sm_90a) batched force-and-moment MPC solver that is a drop-in for the
 * C boundary of DRCL-USC/Hector_Simulation's convex MPC:
 *
 *   reference boundary : hector_control/ConvexMPC/convexMPC_interface.h:11-43
 *   reference caller   : hector_control/ConvexMPC/ConvexMPCLocomotion.cpp:410,415,428-429
 *
 * Part 1 re-exports the four reference symbols with identical signatures and semantics
 * (one robot, blocking solve, result held by the library).  Part 2 is the additive batched
 * interface (thousands of independent robots per launch).  Plain pointers and sizes only:
 * no C++/torch types cross this boundary.
 *
 * There is NO CPU fallback behind these entry points: if no CUDA device / kernel image is
 * usable, every entry point reports HMPC_ERR_CUDA (batched API) or aborts with a message
 * (reference API, which has no error channel — convexMPC_interface.h:39-43).
 */
#ifndef HECTOR_MPC_B200_H
#define HECTOR_MPC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
#define HMPC_EXTERNC extern "C"
#else
#define HMPC_EXTERNC
#endif

/* ------------------------------------------------------------------------------------------
 * Part 0 — POD records, byte-compatible with the reference
 * ---------------------------------------------------------------------------------------- */

#define K_MAX_GAIT_SEGMENTS 36 /* convexMPC_interface.h:3 */

/* convexMPC_interface.h:11-17.  `mu` is carried but ignored by the solver, exactly like the
 * reference (SolverMPC.cpp:488 shadows it with a local 2.0). */
struct problem_setup
{
  float dt;
  float mu;
  float f_max;
  int horizon;
};

/* convexMPC_interface.h:19-37 — same member order, types and padding (sizeof == 3016). */
struct update_data_t
{
  float p[3];                          /* CoM position, world                               */
  float v[3];                          /* CoM velocity, world                               */
  float q[4];                          /* orientation quaternion (w,x,y,z)                  */
  float w[3];                          /* angular velocity, world                           */
  float r[6];                          /* foot - CoM, layout [x0,x1,y0,y1,z0,z1]            */
  float joint_angles[10];              /* leg0 q0..q4, leg1 q0..q4 (before the solver's offset) */
  float yaw;
  float weights[12];                   /* state tracking weights (rpy, p, w, v)             */
  float traj[12 * K_MAX_GAIT_SEGMENTS];/* reference trajectory, 12 per horizon step         */
  float Alpha_K[12];                   /* input regularisation [F0 F1 M0 M1]                */
  unsigned char gait[K_MAX_GAIT_SEGMENTS]; /* contact table, [step][leg], 0/1             */
  unsigned char hack_pad[1000];
  int max_iterations;
  double rho, sigma, solver_alpha, terminate;
};

/* ------------------------------------------------------------------------------------------
 * Part 1 — the reference's own entry points (convexMPC_interface.h:39-43)
 *
 *   setup_problem        replaces convexMPC_interface.cpp:42-66  (+ resize_qp_mats, SolverMPC.cpp:196-299)
 *   update_problem_data  replaces convexMPC_interface.cpp:83-103 (+ solve_mpc, SolverMPC.cpp:371-738,
 *                         + qpOASES QProblem::init, SolverMPC.cpp:702-712)
 *   get_solution         replaces convexMPC_interface.cpp:105-110
 *   update_solver_settings replaces convexMPC_interface.cpp:112-118 (stored, otherwise unused)
 *
 * Semantics kept: update_problem_data blocks until the wrench is available; get_solution(i),
 * i in [0, 12*horizon), is step-major [F0(3) F1(3) M0(3) M1(3)] in the world frame and returns
 * 0.0 before the first solve; swing-leg entries are exactly 0.0.  Single caller thread.
 * Difference (documented in INTEGRATION.md): horizon > 19 aborts with a message instead of
 * letting a C++ exception escape (SolverMPC.cpp:140-143).
 * ---------------------------------------------------------------------------------------- */
HMPC_EXTERNC void setup_problem(double dt, int horizon, double mu, double f_max);
HMPC_EXTERNC double get_solution(int index);
HMPC_EXTERNC void update_solver_settings(int max_iter, double rho, double sigma, double solver_alpha,
                                         double terminate, double use_jcqp);
HMPC_EXTERNC void update_problem_data(double* p, double* v, double* q, double* w, double* r,
                                      double* joint_angles, double yaw, double* weights,
                                      double* state_trajectory, double* Alpha_K, int* gait);

/* The boundary above has no error channel (its functions return void / a double).  Two additive calls give a 1 kHz
 * controller one without changing the reference's call sites:
 *   hmpc_reference_last_status  the status word of the last update_problem_data (HMPC_STATUS_* macros below): code,
 *                               working-set changes, active rows — what "failed to solve!" (SolverMPC.cpp:714-715) hides.
 *   hmpc_reference_last_rc      HMPC_OK, HMPC_ERR_NOT_CONVERGED, or the error of the last tick.  A tick that fails at run
 *                               time (a CUDA error after a successful setup_problem) does NOT end the process: the error is
 *                               printed once per episode, get_solution keeps returning the last tick's wrench, and this call
 *                               (with hmpc_last_error()) tells the controller, which can fall back to its stand-still
 *                               behaviour.  HMPC_REFERENCE_ABORT=1 in the environment restores "abort on any failure".
 * Misuse and start-up failures stay fatal with a message: horizon > 19 (the reference throws), update_problem_data before
 * setup_problem, no usable GPU at setup_problem. */
HMPC_EXTERNC int hmpc_reference_last_status(void);
HMPC_EXTERNC int hmpc_reference_last_rc(void);

/* ------------------------------------------------------------------------------------------
 * Part 2 — batched interface (additive; SURVEY.md §8b "batched extension")
 * ---------------------------------------------------------------------------------------- */

typedef struct hmpc_ctx hmpc_ctx;

/* return codes */
#define HMPC_OK 0
#define HMPC_ERR_ARG 1      /* bad argument (null pointer, batch > capacity, horizon out of range) */
#define HMPC_ERR_CUDA 2     /* CUDA runtime error / no device / no sm_90a device; hmpc_last_error() has text */
#define HMPC_ERR_NOT_CONVERGED 3 /* at least one instance did not reach a KKT point; see status[] */

/* per-instance status word written with every result (never silently stale — contrast
 * SolverMPC.cpp:714-715, which prints and carries on with stale data):
 *   bits  0..7  : termination code  (0 = optimal, 1 = iteration cap, 2 = working-set capacity,
 *                                    3 = infeasible/degenerate step, 4 = Hessian not positive definite ENOUGH: a
 *                                    non-positive pivot, or max_i H_ii (H^-1)_ii above the conditioning limit of the
 *                                    fp64 sweep inversion (1.5e5; 2e2 ... 1e4 on the workloads of BASELINE.json, 3e5
 *                                    for a robot lying on its side) — the wrench of such an instance is not trusted)
 *   bits  8..19 : working-set changes performed (comparable to qpOASES nWSR)
 *   bits 20..27 : number of active constraints at the solution
 *   bit  28     : solved by the refinement class (hmpc_set_refinement; code 0).  Only with refinement on.
 * With refinement on, an instance whose scaled condition number is above 1.5e4 (and below 1e9), with every pivot positive,
 * is solved again by the refinement class; it returns code 0 with bit 28 set, or code 4 as above.
 */
#define HMPC_STATUS_CODE(s) ((s) & 0xff)
#define HMPC_STATUS_ITERS(s) (((s) >> 8) & 0xfff)
#define HMPC_STATUS_NACTIVE(s) (((s) >> 20) & 0xff)
#define HMPC_STATUS_REFINED(s) (((s) >> 28) & 1)

#define HMPC_MAX_HORIZON 16 /* dense fp64 working set of one QP must fit one SM's shared memory */

/* Packed device record (HBM layout, one per robot).  Only the bytes that change per tick:
 *   float state[30]  = p3 v3 q4 w3 r6 joint10 yaw1
 *   float weights[12], float alpha[12]
 *   float traj[12*N]
 *   u8    gait[2*N]   (+ zero padding to a multiple of 16 bytes)
 * hmpc_record_bytes(N) gives the stride.  N=10: 216 + 98*N = 1196 algorithmic bytes per QP
 * in+out (SURVEY.md §8d), 720-byte input stride. */
HMPC_EXTERNC size_t hmpc_record_bytes(int horizon);
/* pack n reference records into the device layout (host side helper, pure byte shuffling) */
HMPC_EXTERNC int hmpc_pack_records(const struct update_data_t* in, int n, int horizon, void* out);

/* create a context on `device` able to hold `max_batch` robots of `horizon` steps */
HMPC_EXTERNC hmpc_ctx* hmpc_create(int max_batch, int horizon, int device);
HMPC_EXTERNC void hmpc_destroy(hmpc_ctx* ctx);
HMPC_EXTERNC const char* hmpc_last_error(void);

/* dt / f_max of problem_setup (mu is ignored like the reference).  Defaults 0.04 / 500. */
HMPC_EXTERNC int hmpc_set_problem(hmpc_ctx* ctx, const struct problem_setup* setup);

/* Host-buffer path (the reference-facing call: H2D + solve + D2H inside).
 *   in         : B reference records (host)
 *   wrench_out : [B][12*horizon] doubles, same layout as get_solution (host)
 *   status     : [B] status words (host), may be NULL
 * Blocks until results are in host memory. */
HMPC_EXTERNC int hmpc_solve_batch(hmpc_ctx* ctx, const struct update_data_t* in, int B,
                                  double* wrench_out, int* status);

/* Device-resident path: `d_records` = B packed records already in HBM, `d_wrench`
 * [B][12*horizon] float, `d_status` [B] int, all device pointers; enqueued on `stream`
 * (a cudaStream_t passed as void*), returns without synchronising. */
/* d_records must be 16-byte aligned (the kernels stage records with a bulk copy); B <= the context's capacity. */
HMPC_EXTERNC int hmpc_solve_device(hmpc_ctx* ctx, const void* d_records, int B, float* d_wrench,
                                   int* d_status, void* stream);

/* Row f-2 (SURVEY.md §8f): the same solves with the leg-controller epilogue fused in — joint torques of the
 * first-step wrench, tau[leg*5+j] = (J_force_moment^T * f_ff)[j], f_ff = -rBody * [F; M]
 * (replaces LegController.cpp:57-63 + :108-166 and ConvexMPCLocomotion.cpp:419-440 for stance legs; swing legs 0).
 * tau_out [B][10] doubles (host) / d_tau [B][10] floats (device); pass NULL to skip. */
HMPC_EXTERNC int hmpc_solve_batch_ex(hmpc_ctx* ctx, const struct update_data_t* in, int B, double* wrench_out,
                                     double* tau_out, int* status);
HMPC_EXTERNC int hmpc_solve_device_ex(hmpc_ctx* ctx, const void* d_records, int B, float* d_wrench, int* d_status,
                                      float* d_tau, void* stream);

/* In-place mode of hmpc_solve_batch(_ex).  A control loop reuses the same record / result arrays every tick; register
 * them once (cudaHostRegister underneath) and hmpc_solve_batch lets the GPU read the update_data_t records where they
 * lie and write the double wrenches (and status) where the caller wants them: no packing, no staging copies, no
 * float->double pass on the host.  It is used whenever `in`, `wrench_out` and `status` (if given) of a call all lie
 * inside pinned ranges; results are identical to the staged path.  The caller keeps the memory allocated until
 * hmpc_unpin_host_buffer / hmpc_destroy.  (The reference-style entry points pin their own globals.) */
/* Registration is page-granular: the pages that hold [ptr, ptr + bytes) are pinned whole.  Give the arrays their own pages
 * (posix_memalign to the page size, size rounded up): an unrelated host buffer that shares such a page only partly cannot be
 * the source / destination of a later cudaMemcpy (cudaErrorInvalidValue). */
HMPC_EXTERNC int hmpc_pin_host_buffer(hmpc_ctx* ctx, void* ptr, size_t bytes);
HMPC_EXTERNC int hmpc_unpin_host_buffer(hmpc_ctx* ctx, void* ptr);

/* Row f-1 (SURVEY.md §8f): the caller's data preparation on the device.  `hmpc_state_t` is what
 * ConvexMPCLocomotion::updateMPCIfNeeded reads before it builds the MPC inputs (ConvexMPCLocomotion.cpp:279-346),
 * in double precision as the reference holds it; hmpc_prepare_device turns B of them into packed records (joint
 * offsets + fmod, foot positions r, weights, the 12 x horizon reference trajectory, double -> float narrowing:
 * ConvexMPCLocomotion.cpp:283-406 + convexMPC_interface.cpp:87-99) with one GPU thread per robot, so a tick moves
 * 352 bytes per robot to the device instead of a 720-byte record.  hmpc_solve_batch_states = H2D of the states +
 * hmpc_prepare_device + the solve of hmpc_solve_batch_ex; with the states, wrench_out and status pinned
 * (hmpc_pin_host_buffer) it runs in place, as hmpc_solve_batch does: the same solve, with the wrenches stored as the
 * solver's doubles rather than their float rounding, as in hmpc_solve_batch's in-place mode.  The warm and masked calls on
 * states follow hmpc_solve_batch_masked below. */
struct hmpc_state_t
{
  double position[3];              /* seResult.position */
  double vWorld[3];
  double orientation[4];           /* (w,x,y,z) */
  double omegaWorld[3];
  double rpy[3];                   /* seResult.rpy */
  double leg_q[10];                /* _legController->data[leg].q (LegController's own offset already applied) */
  double leg_p[6];                 /* _legController->data[leg].p, [leg][xyz] */
  double state_des[5];             /* stateDes[3], [4] (roll, pitch), [6], [7] (body-frame vx, vy), [11] (yaw rate) */
  double world_position_desired[2];
  unsigned char gait[K_MAX_GAIT_SEGMENTS]; /* mpcTable, [step][leg] */
  unsigned char pad[4];
};
/* dtMPC is the caller's double `dt * iterationsBetweenMPC` (ConvexMPCLocomotion.cpp:20) used for the trajectory;
 * the QP itself keeps the float dt of hmpc_set_problem, exactly as the reference splits the two. */
HMPC_EXTERNC int hmpc_prepare_device(hmpc_ctx* ctx, const struct hmpc_state_t* d_states, int B, double dtMPC,
                                     void* d_records, void* stream);
HMPC_EXTERNC int hmpc_solve_batch_states(hmpc_ctx* ctx, const struct hmpc_state_t* in, int B, double dtMPC,
                                         double* wrench_out, double* tau_out, int* status);

/* Row f-3 (SURVEY.md §8f): the closed loop on the device — BASELINE config 5 (consecutive ticks of the same robots).
 * One tick = hmpc_prepare_device -> the solve -> hmpc_advance, all enqueued on one stream, no host in the loop:
 *   - the next tick's contact table is Gait::mpc_gait of the advanced iteration counter (GaitGenerator.cpp:85-103);
 *   - the body is integrated one forward-Euler step of the single rigid body the MPC predicts with
 *     (SolverMPC.cpp:145-146, 312-331: x+ = x + dt f(x,u)), feet pinned in the world, first-step wrench fed back;
 *   - a leg that touches down is placed by the heuristic of ConvexMPCLocomotion.cpp:119-160 (hip projection +
 *     0.5 v T_stance + 0.02 (v - v_des), clamped, z = 0) — the swing trajectory itself is out of scope (row f-4);
 *   - world_position_desired integrates the commanded velocity with the clamp write-back of :338-346.
 * hmpc_rollout_t is the per-robot loop state that lives next to hmpc_state_t. */
struct hmpc_rollout_t
{
  double feet_world[6];   /* [leg][xyz]: where each foot is pinned (stance) or was last pinned (swing) */
  int gait_offset[2];     /* Gait(nIterations = horizon, offsets, durations)  (ConvexMPCLocomotion.cpp:16-17) */
  int gait_duration[2];
  int iteration;          /* MPC tick counter; Gait::_iteration = iteration % horizon */
  int failures;           /* ticks whose solver status code was not 0 (accumulated) */
  int iters_total;        /* working-set changes, accumulated */
  int ticks;              /* ticks advanced so far */
};
/* Warm start: every tick after the first proposes the previous tick's optimal working set, moved one step with the
 * horizon, to the active-set stage (the reference cold-starts every tick, SolverMPC.cpp:702-709; BASELINE.json
 * configs[4] names the warm start).  The optimum is the same point either way — the working set only decides how many
 * changes the solver makes to reach it; the status word then counts the changes relative to the proposal.  The sets live in
 * the context; hmpc_reset_warm_start forgets them (a new loop on the same context).  HMPC_WARM_START=0 in the environment
 * at hmpc_create keeps every tick a cold start. */
HMPC_EXTERNC int hmpc_reset_warm_start(hmpc_ctx* ctx, void* stream);

/* Warm start in the caller's own loop (a batched simulator, an RL environment, a host program).  The same working-set memory
 * as the rollout: slot i belongs to robot i of the batch, every warm call records each robot's optimal working set there and
 * proposes it to that robot's next warm call.  shift[i] = MPC steps robot i's horizon moved since its last warm call on this
 * context: NULL = every robot 1 (one call per MPC tick), 0 = the same horizon again, < 0 = no history (e.g. an environment
 * reset: a cold solve whose working set is still recorded).  The optimum is the same point as a cold solve's; bits 8..19 of
 * the status count changes relative to the proposal.  The proposal feeds the block start of the active-set stage, which
 * runs for working-set capacities of up to 31 rows: horizons up to 13 in the single-support class, up to 10 in the
 * double-support class.  Beyond that a warm call is a cold solve, bit for bit.  HMPC_WARM_START=0 at hmpc_create makes
 * every warm call a cold solve.
 *   hmpc_solve_device_warm: as hmpc_solve_device_ex; d_shift NULL or device int [B].  Same argument checks.
 *   hmpc_solve_batch_warm : as hmpc_solve_batch_ex (all three host-buffer modes); shift NULL or host int [B]. */
HMPC_EXTERNC int hmpc_solve_device_warm(hmpc_ctx* ctx, const void* d_records, int B, float* d_wrench, int* d_status,
                                        float* d_tau, const int* d_shift, void* stream);
HMPC_EXTERNC int hmpc_solve_batch_warm(hmpc_ctx* ctx, const struct update_data_t* in, int B, double* wrench_out,
                                       double* tau_out, int* status, const int* shift);
/* Solving part of the batch.  A reference-style controller runs its MPC only every iterationsBetweenMPC control ticks
 * of each robot's own counter (ConvexMPCLocomotion.cpp:277), and robots that stand, lie or wait for a reset need none,
 * so in a batch of robots reset at different times only a changing subset is due in any tick.  The masked calls solve
 * robot i iff mask[i] != 0 (a torch.bool tensor can be passed as it is), with the arrays sized for the whole batch:
 * records, outputs, mask[B] and shift[B], B <= the context's capacity.
 *   - A listed robot's wrench row, status word, torque row and working-set slot are written exactly as the _warm call
 *     writes them.  An unlisted robot's keep their bytes, on the host arrays too in every host-buffer mode.
 *   - Warm start as in the _warm calls: slot i is robot i, whatever other robots are listed; shift[i] (read for listed
 *     robots only) is the MPC steps robot i's horizon moved since its last solve on this context.  NULL = 1 for every
 *     listed robot, 0 = the same horizon, < 0 = a cold solve that records the set.  HMPC_WARM_START=0 and
 *     hmpc_set_refinement act as in the other calls.
 *   - An empty mask is valid: nothing is written.  The host call returns HMPC_ERR_NOT_CONVERGED for listed robots only.
 *   - Argument checks as in the _warm calls, plus a NULL mask is HMPC_ERR_ARG; B = 0 is a no-op.
 *   hmpc_solve_device_masked: as hmpc_solve_device_warm; d_mask device bytes [B].  The mask is read on the device, by one
 *                             more launch ahead of the chain, so the call needs no host synchronisation and one captured
 *                             graph serves every mask written into the captured buffer.
 *   hmpc_solve_batch_masked : as hmpc_solve_batch_warm (all three host-buffer modes); mask host bytes [B]. */
HMPC_EXTERNC int hmpc_solve_device_masked(hmpc_ctx* ctx, const void* d_records, int B, const unsigned char* d_mask,
                                          float* d_wrench, int* d_status, float* d_tau, const int* d_shift, void* stream);
HMPC_EXTERNC int hmpc_solve_batch_masked(hmpc_ctx* ctx, const struct update_data_t* in, int B, const unsigned char* mask,
                                         double* wrench_out, double* tau_out, int* status, const int* shift);
/* The same calls with robot states (hmpc_state_t) in: the data preparation of hmpc_prepare_device, then the solve.
 *   hmpc_solve_states_device_masked: one chain on `stream`, the selection kernel, then the preparation of the listed robots
 *                             only, then the solve of hmpc_solve_device_masked.  d_records [B][hmpc_record_bytes] (16-byte
 *                             aligned) receives the listed robots' records, what the solver saw; unlisted rows keep their
 *                             bytes.  Capturable, as hmpc_solve_device_masked.
 *   hmpc_solve_batch_states_warm / _masked: hmpc_solve_batch_warm / _masked on states, in all three host-buffer modes.
 * Like hmpc_solve_batch_states, these calls run in place when the states array, wrench_out and status (if given) lie in
 * pinned ranges (hmpc_pin_host_buffer): the preparation kernel reads the states where they lie, the records stay in the
 * context, and double wrenches and status words are written straight into the caller's arrays. */
HMPC_EXTERNC int hmpc_solve_states_device_masked(hmpc_ctx* ctx, const struct hmpc_state_t* d_states, int B,
                                                 const unsigned char* d_mask, double dtMPC, void* d_records, float* d_wrench,
                                                 int* d_status, float* d_tau, const int* d_shift, void* stream);
HMPC_EXTERNC int hmpc_solve_batch_states_warm(hmpc_ctx* ctx, const struct hmpc_state_t* in, int B, double dtMPC,
                                              double* wrench_out, double* tau_out, int* status, const int* shift);
HMPC_EXTERNC int hmpc_solve_batch_states_masked(hmpc_ctx* ctx, const struct hmpc_state_t* in, int B, const unsigned char* mask,
                                                double dtMPC, double* wrench_out, double* tau_out, int* status,
                                                const int* shift);
/* The MPC's plan: robot i's predicted states under the discrete model its QP was built from, pred[i][k] = x_{k+1} =
 * Acd x_k + Bcd u_k for k = 0 .. N-1, with x_0, Acd and Bcd the float32 ones of the solve (the same code computes them) and
 * u_k = wrench row entries [12k, 12k+12).  A row of 12 is rpy, p, omega, v: the layout of update_data_t::traj, so pred - traj
 * is the tracking error; the gravity state is not returned.  dt is the context's problem dt (hmpc_set_problem), as in the
 * QP, not the caller's dtMPC.  The recurrence runs in float64 with separately rounded operations in a fixed order
 * (DESIGN.md §3); hmpc_predict_device returns its float rounding.
 *   - The plan is computed for whatever wrench row is passed.  A robot whose status code is not 0 has an untrusted wrench,
 *     so its plan is untrusted too.
 *   - A mask (NULL: every robot) skips robots with mask[i] == 0: their prediction rows keep their bytes.  Pass the mask of
 *     the masked solve the wrenches came from.
 *   - Argument checks: a NULL context or pointer and B > capacity are HMPC_ERR_ARG; B = 0 is a no-op.
 *   hmpc_predict_device: d_records B packed records (or any rows whose first 19 floats are p v q w r) with row stride
 *                        hmpc_record_bytes(horizon); d_wrench [B][12N] float; d_mask NULL or device bytes [B]; d_pred
 *                        [B][N][12] float.  One launch on `stream`, no host synchronisation.  Capturable.
 *   hmpc_predict_batch : in B update_data_t, wrench [B][12N] double as the host solves return them, mask NULL or host bytes
 *                        [B], pred_out [B][N][12] double.  In place when in, wrench and pred_out lie in pinned ranges
 *                        (hmpc_pin_host_buffer), else staged through the context's pinned memory; the same plans either way. */
HMPC_EXTERNC int hmpc_predict_device(hmpc_ctx* ctx, const void* d_records, int B, const unsigned char* d_mask,
                                     const float* d_wrench, float* d_pred, void* stream);
HMPC_EXTERNC int hmpc_predict_batch(hmpc_ctx* ctx, const struct update_data_t* in, int B, const unsigned char* mask,
                                    const double* wrench, double* pred_out);
/* The certificate: a first-order optimality (KKT) check of robot i's wrench for its row, made on the device without the
 * solve, so it judges any wrench: the solver's, qpOASES', a learned policy's.  The status word is not read.  From the row
 * and the context's dt and f_max (hmpc_set_problem) it rebuilds the solve's float32 x0, Acd, Bcd and constraint rows
 * (the same code computes them), runs the plan in float64, and takes the gradient of the QP objective by an adjoint sweep
 * over it.  Per stance (step, leg) the rows within rounding of a bound are fitted to the gradient with sign-constrained
 * multipliers; a swing leg's entries must be exactly 0.  DESIGN.md §3 gives the operations, §7 the thresholds.
 *   cost              J = sum_k (x_k - traj_k)' S (x_k - traj_k) + u_k' Alpha_K u_k: the QP objective 1/2 U'HU + g'U plus
 *                     the constant d'Sd of the record, float64 in a fixed order;
 *   stationarity      max |grad J - A'lambda| over the largest gradient entry formed from absolute values (|x|, |u|, |S|,
 *                     |Acd|, |Bcd|) of the stance legs;
 *   primal            the worst bound violation or non-zero swing entry over the largest sum |a||u| of the stance rows;
 *   complementarity   max |lambda| slack over the product of both scales;
 *   n_active          the rows taken as active (candidates for a multiplier);
 *   flags             HMPC_CERT_PASS alone when the inputs are finite, no swing entry is non-zero and each measure is
 *                     within its threshold; otherwise the bits of what failed.
 *   - lambda (NULL: not written) [B][N][2][8]: one per row of Fblk, >= 0 at a lower bound, <= 0 at an upper one, 0 on the
 *     other rows and on swing legs: how hard each foot presses on its friction rows and force limit, the sensitivity of
 *     the optimum to those bounds.  Where several rows are active at one point (a foot at zero force) it is one of many.
 *   - A mask (NULL: every robot) skips robots with mask[i] == 0: their certificates and multipliers keep their bytes.
 *   - Argument checks: a NULL context or pointer (lambda may be NULL) and B > capacity are HMPC_ERR_ARG; B = 0 is a no-op.
 *   hmpc_certify_device: d_records B packed records, d_wrench [B][12N] float, d_mask NULL or device bytes [B], d_cert [B],
 *                        d_lambda float.  One launch on `stream`, no host synchronisation.  Capturable.
 *   hmpc_certify_batch : in B update_data_t, wrench [B][12N] double as the host solves return them, mask NULL or host bytes,
 *                        lambda_out double.  In place when in, wrench, cert_out and lambda_out lie in pinned ranges
 *                        (hmpc_pin_host_buffer), else staged through the context's pinned memory; the same results. */
typedef struct hmpc_certificate_t {
  double cost, stationarity, primal, complementarity;
  int n_active, flags;
} hmpc_certificate_t;
#define HMPC_CERT_PASS 1          /* the wrench is a KKT point of its record's QP to the thresholds below */
#define HMPC_CERT_NONFINITE 2     /* a non-finite wrench entry, state, gradient or row */
#define HMPC_CERT_SWING 4         /* a swing leg's wrench entry is not 0 */
#define HMPC_CERT_STATIONARITY 8  /* stationarity > HMPC_CERT_STATIONARITY_TOL */
#define HMPC_CERT_PRIMAL 16       /* primal > HMPC_CERT_PRIMAL_TOL */
#define HMPC_CERT_COMPLEMENTARITY 32  /* complementarity > HMPC_CERT_COMPLEMENTARITY_TOL */
#define HMPC_CERT_STATIONARITY_TOL 2e-6
#define HMPC_CERT_PRIMAL_TOL 2e-7
#define HMPC_CERT_COMPLEMENTARITY_TOL 1e-9
HMPC_EXTERNC int hmpc_certify_device(hmpc_ctx* ctx, const void* d_records, int B, const unsigned char* d_mask,
                                     const float* d_wrench, hmpc_certificate_t* d_cert, float* d_lambda, void* stream);
HMPC_EXTERNC int hmpc_certify_batch(hmpc_ctx* ctx, const struct update_data_t* in, int B, const unsigned char* mask,
                                    const double* wrench, hmpc_certificate_t* cert_out, double* lambda_out);
/* Several reference trajectories per robot: robot i's MPC solved for K candidate trajectories traj[i][k] [12N] (laid out
 * like update_data_t::traj) at once.  The record's own traj bytes are not read; everything else in it is shared by the K
 * candidates, so the QP's constraints, its Hessian and the sweep inversion are computed once per robot and only the
 * gradient and the active-set stage run per candidate (DESIGN.md §3).
 *   - Let the expanded batch be the B*K records in which row i*K + k is robot i's record with traj replaced by candidate k.
 *     Candidate (i, k) gets, bit for bit, the wrench and status word hmpc_solve_device gives row i*K + k of the expanded
 *     batch, in every size class and with hmpc_set_refinement on, and the cost hmpc_certify_device gives for that row and
 *     that wrench.  Results: wrench [B][K][12N], status [B][K], cost NULL or double [B][K].
 *   - cost: J = sum_k (x_k - traj_k)' S (x_k - traj_k) + u_k' Alpha_K u_k including the constant d'Sd, so candidates can be
 *     ranked by it.  A candidate whose status code is not 0 has no trusted wrench, hence no trusted cost.
 *   - Calls are cold: no working set is proposed or recorded, and the warm-start memory is not touched.
 *   - A mask (NULL: every robot) skips robots with mask[i] == 0: their K rows of every output keep their bytes.
 *   - Argument checks: a NULL context, records, traj, wrench or status pointer, K < 1 and B*K > capacity are HMPC_ERR_ARG;
 *     B = 0 is a no-op.
 *   hmpc_solve_device_multi: d_records B packed records, float traj and wrench, device mask.  One chain on `stream`, no
 *                            host synchronisation.  Capturable.
 *   hmpc_solve_batch_multi : in B update_data_t, host arrays, double wrenches (the solver's own: they round to the device
 *                            call's floats).  In place when in, traj, wrench_out, status and cost_out lie in pinned ranges
 *                            (hmpc_pin_host_buffer), else staged through the context's pinned memory; the same results.
 *                            Its cost is hmpc_certify_batch's for the expanded row and the double wrench.  Returns
 *                            HMPC_ERR_NOT_CONVERGED when a listed candidate did not reach a KKT point. */
HMPC_EXTERNC int hmpc_solve_device_multi(hmpc_ctx* ctx, const void* d_records, int B, int K, const float* d_traj,
                                         const unsigned char* d_mask, float* d_wrench, int* d_status, double* d_cost,
                                         void* stream);
HMPC_EXTERNC int hmpc_solve_batch_multi(hmpc_ctx* ctx, const struct update_data_t* in, int B, int K, const float* traj,
                                        const unsigned char* mask, double* wrench_out, int* status, double* cost_out);
/* test hook: 1 when the last hmpc_solve_batch_multi that launched ran in place, 0 when it staged, -1 before any */
HMPC_EXTERNC int hmpc_debug_last_multi_in_place(void);
/* Candidate commands per robot, from its state: robot i's MPC solved for K commands cmd[i][k] at once, the cheapest
 * converged one picked on the device.  A command is the part of hmpc_state_t the reference trajectory is built from
 * (ConvexMPCLocomotion.cpp:331-399); every other field of the state is shared by the K candidates.  The chain prepares robot
 * i's record once and its K trajectories, then runs hmpc_solve_device_multi's solve and cost on them, then a pick kernel
 * (DESIGN.md §3).
 *   - Let the expanded state batch be the B*K states in which row i*K + k is state i with its 56 command bytes replaced by
 *     cmd[i][k].  Bit for bit, in every size class and with hmpc_set_refinement on:
 *       traj[i][k]          the traj hmpc_prepare_device writes for expanded row i*K + k;
 *       wrench[i][k],       what hmpc_solve_device gives the expanded prepared row (hmpc_solve_device_multi on robot i's record
 *       status[i][k]        with those K trajectories);
 *       cost[i][k]          what hmpc_certify_device reports as the cost of that row and wrench;
 *       best[i]             the k of the smallest cost among the candidates with status code 0 and a finite cost, the lowest k
 *                           on ties; -1 when there is none;
 *       tau[i]              the torque row hmpc_solve_device_ex gives expanded row i*K + best[i]; zeros when best[i] = -1;
 *       records row i       the record hmpc_prepare_device writes for expanded row i*K + best[i] (i*K when best[i] = -1), so
 *                           hmpc_predict_device / hmpc_certify_device on (records, the chosen wrench) work directly.
 *   - Calls are cold: no working set is proposed or recorded, and the warm-start memory is not touched.
 *   - A mask (NULL: every robot) skips robots with mask[i] == 0: every output row of theirs keeps its bytes, records
 *     included.
 *   - Argument checks: a NULL context or required pointer (d_mask / mask and d_tau / tau_out may be NULL), K < 1 and
 *     B*K > capacity are HMPC_ERR_ARG; B = 0 is a no-op.
 *   hmpc_solve_states_device_multi: device arrays; d_records [B][hmpc_record_bytes] (16-byte aligned), d_traj float
 *                            [B][K][12N], d_wrench float [B][K][12N], d_status [B][K], d_cost [B][K], d_best [B], d_tau float
 *                            [B][10] or NULL.  One chain on `stream`, no host synchronisation.  Capturable.
 *   hmpc_solve_batch_states_multi: host arrays, double wrenches and torques (the solver's own: they round to the device
 *                            call's floats).  In place when in, cmd, wrench_out, status, cost_out and best lie in pinned ranges
 *                            (hmpc_pin_host_buffer), else staged through the context's pinned memory; the same results.  The
 *                            records and trajectories stay in the context.  Returns HMPC_ERR_NOT_CONVERGED when a listed robot
 *                            has best == -1. */
struct hmpc_command_t {            /* bytes [256, 312) of hmpc_state_t, same order */
  double state_des[5];             /* roll, pitch, body vx, vy, yaw rate */
  double world_position_desired[2];
};
HMPC_EXTERNC int hmpc_solve_states_device_multi(hmpc_ctx* ctx, const struct hmpc_state_t* d_states, int B, int K,
                                                const struct hmpc_command_t* d_cmd, const unsigned char* d_mask, double dtMPC,
                                                void* d_records, float* d_traj, float* d_wrench, int* d_status, double* d_cost,
                                                int* d_best, float* d_tau, void* stream);
HMPC_EXTERNC int hmpc_solve_batch_states_multi(hmpc_ctx* ctx, const struct hmpc_state_t* in, int B, int K,
                                               const struct hmpc_command_t* cmd, const unsigned char* mask, double dtMPC,
                                               double* wrench_out, int* status, double* cost_out, int* best, double* tau_out);
/* test hook: 1 when the last hmpc_solve_batch_states_multi that launched ran in place, 0 when it staged, -1 before any */
HMPC_EXTERNC int hmpc_debug_last_states_multi_in_place(void);
/* The reference boundary warm-started: after hmpc_reference_set_warm_start(1), every update_problem_data proposes the
 * previous call's working set moved one step (a hmpc_solve_batch_warm with shift NULL on the one-robot context).
 * setup_problem with another dt, f_max or horizon forgets it.  Default 0: every tick a cold start, like the reference. */
HMPC_EXTERNC void hmpc_reference_set_warm_start(int on);
/* ticks >= 1.  d_wrench_log: NULL or float [ticks][B][12] (first-step wrench of every tick); d_record_log: NULL or
 * [ticks][B][hmpc_record_bytes] (the packed records the solver saw, for after-the-fact parity checks). */
HMPC_EXTERNC int hmpc_rollout_device(hmpc_ctx* ctx, struct hmpc_state_t* d_states, struct hmpc_rollout_t* d_loop, int B,
                                     int ticks, double dtMPC, float* d_wrench_log, void* d_record_log, void* stream);

/* ---------------------------------------------------------------------------------------------------------------------
 * Multi-GPU (SURVEY.md §8e; the reference has nothing here: one robot per process).  Robots are independent, so a batch
 * larger than one device is cut into contiguous slices, one process per GPU, identical kernels, no data-path collective.
 * Every rank gets ITS slice back on the host exactly like hmpc_solve_batch (in place when the arrays are pinned); when a
 * consumer needs the whole batch on every device, `d_all` (device, float [world * B_local][12 * horizon], rank-major)
 * receives ONE ncclAllGather of the float wrenches, enqueued behind the solve on a side stream so that it overlaps the
 * next tick (results are double-buffered); hmpc_shard_wait blocks until the last gather has landed.  NCCL is loaded at run
 * time (libnccl.so.2), only by these calls.
 *   rank 0: hmpc_shard_unique_id(id)  ->  ship the 128 bytes to every rank  ->  all: hmpc_shard_init(ctx, rank, world, id)
 * B_local must be the same on every rank (pad the last slice).  The gather is a collective of the context's own NCCL
 * communicator: call hmpc_shard_wait before another communicator (e.g. torch.distributed's) runs a collective on the same
 * device, as with any two NCCL communicators. */
#define HMPC_SHARD_ID_BYTES 128
HMPC_EXTERNC int hmpc_shard_unique_id(void* id128);
HMPC_EXTERNC int hmpc_shard_init(hmpc_ctx* ctx, int rank, int world, const void* id128);
HMPC_EXTERNC int hmpc_solve_batch_sharded(hmpc_ctx* ctx, const update_data_t* in_local, int B_local, double* wrench_local,
                                          int* status_local, float* d_all);
HMPC_EXTERNC int hmpc_shard_wait(hmpc_ctx* ctx);
/* Sharded calls warm-started, masked and on robot states: each rank solves only its due robots, and the gather still
 * carries every robot's last wrench.
 *   - mask_local NULL: hmpc_solve_batch_warm (hmpc_solve_batch_states_warm) on the local slice; non-NULL: the slice's
 *     hmpc_solve_batch_masked (hmpc_solve_batch_states_masked).  The slice's results come back on the rank's own arrays in
 *     all three host-buffer modes, in place when the arrays are pinned.  tau_local and shift_local may be NULL.
 *   - Warm start: slot i is local robot i of this rank's context; shift_local as in the other warm calls.
 *     hmpc_reset_warm_start and HMPC_WARM_START=0 act as elsewhere.
 *   - HMPC_ERR_NOT_CONVERGED is returned for listed robots only.  Argument checks as in hmpc_solve_batch_sharded
 *     (hmpc_shard_init first, 1 <= B_local <= capacity) plus those of the warm and masked calls.  An all-zero mask is
 *     valid: nothing is solved, and the gather still runs.
 *   - Gather: row r * B_local + i of d_all on every rank is the float wrench of robot i of rank r — this call's result
 *     for a listed robot, else its row from the last sharded call of that context that solved it, or zeros if none has.
 *     This holds whatever the caller's host arrays contain and whether or not earlier calls passed d_all: every sharded
 *     call, hmpc_solve_batch_sharded included, keeps the context's gather buffers current, gathering or not.  A small
 *     kernel behind the solve copies the unlisted rows from the previous tick's buffer. */
HMPC_EXTERNC int hmpc_solve_batch_sharded_warm(hmpc_ctx* ctx, const struct update_data_t* in_local, int B_local,
                                               const unsigned char* mask_local, double* wrench_local, double* tau_local,
                                               int* status_local, const int* shift_local, float* d_all);
HMPC_EXTERNC int hmpc_solve_batch_states_sharded_warm(hmpc_ctx* ctx, const struct hmpc_state_t* in_local, int B_local,
                                                      const unsigned char* mask_local, double dtMPC, double* wrench_local,
                                                      double* tau_local, int* status_local, const int* shift_local,
                                                      float* d_all);

/* Row f-4 (SURVEY.md §8f): the swing-leg controller, batched — swingLegController::updateSwingLeg
 * (src/common/SwingLegController.cpp:46-219): foot position, swing sub-phase (Gait::getSwingSubPhase,
 * GaitGenerator.cpp:54-80), swing-time countdown, touch-down placement (:98-128), Bezier swing trajectory
 * (FootSwingTrajectory.cpp:17-36, Interpolation.h:53-74) and the approximate 5-DoF inverse kinematics (:160-193), one GPU
 * thread per robot, fp64.  hmpc_swing_t is the controller's per-robot memory (swingLegController's members);
 * hmpc_swing_cmd_t is what setDesiredJointState (:198-219) hands to the leg controller for the legs in swing
 * (zeros and swing[leg] = 0 for stance legs).  `d_phase[i]` is Gait::_phase of robot i (GaitGenerator.cpp:112); the
 * gait's offsets/durations come from hmpc_rollout_t (nIterations = the context's horizon). */
struct hmpc_swing_t
{
  double p0[6];          /* footSwingTrajectory[leg]._p0, world */
  double swing_time[2];  /* swingTimes[leg] */
  int first_swing[2];    /* firstSwing[leg] (initially 1, 1) */
};
struct hmpc_swing_cmd_t
{
  double pf[6];          /* planned touch-down position of each leg, world (footSwingTrajectory[leg]._pf) */
  double p_des[6];       /* commands[leg].pDes = pFoot_b, body frame */
  double v_des[6];       /* commands[leg].vDes = vFoot_b */
  double q_des[10];      /* commands[leg].qDes from computeIK */
  int swing[2];          /* swingStates[leg] > 0 */
};
/* dt = the controller's own period (0.001, SwingLegController.h:79), dtSwing = dtMPC (ConvexMPCLocomotion.cpp:70).
 * One call = one updateSwingLeg.  Note that the reference's ConvexMPCLocomotion::run calls updateSwingLeg inside its
 * per-foot loop (ConvexMPCLocomotion.cpp:218), i.e. TWICE per control tick, so its swing-time countdown runs at 2*dt per
 * tick; a caller reproducing that controller calls this function twice per tick (tests/test_reference_tick.py does). */
HMPC_EXTERNC int hmpc_swing_device(hmpc_ctx* ctx, const struct hmpc_state_t* d_states, const struct hmpc_rollout_t* d_loop,
                                   const double* d_phase, struct hmpc_swing_t* d_swing, int B, double dt, double dtSwing,
                                   struct hmpc_swing_cmd_t* d_cmd, void* stream);

/* CUDA graphs.  The device-resident calls can be recorded into a CUDA graph by stream capture (cudaStreamBeginCapture,
 * torch.cuda.graph, ...) on the stream they are given: hmpc_solve_device, hmpc_solve_device_ex, hmpc_solve_device_warm,
 * hmpc_solve_device_masked, hmpc_solve_states_device_masked, hmpc_prepare_device, hmpc_rollout_device, hmpc_swing_device,
 * hmpc_predict_device, hmpc_certify_device, hmpc_solve_device_multi, hmpc_solve_states_device_multi and
 * hmpc_reset_warm_start.  Each
 * launch of the graph gives the results an eager call on the same inputs gives, bit for bit.
 *   - A replay is a real call.  A captured warm solve proposes and records working sets, a captured rollout advances
 *     d_states and d_loop, a captured hmpc_reset_warm_start clears the working sets, every time the graph is launched.
 *   - A context's calls, eager ones and graph launches alike, must be ordered on one stream (or by events).  All chains
 *     a context records share one set of class lists, so two graphs of one context, or one graph launched twice, must not
 *     run concurrently.
 *   - The pointers and B are frozen into the graph: to solve other inputs, write them into the captured buffers.
 *   - A graph must not be launched after hmpc_destroy of its context.
 *   - A call that returns an error while its stream is capturing may have recorded part of its work: end the capture
 *     and discard the graph.  Argument errors are found before anything is enqueued.
 * The host-buffer calls (hmpc_solve_batch, _ex, _warm, _masked, _states, _states_warm, _states_masked,
 * hmpc_solve_batch_sharded, hmpc_predict_batch, hmpc_certify_batch, hmpc_solve_batch_multi, hmpc_solve_batch_states_multi)
 * and the reference boundary
 * (update_problem_data) wait for their own streams and cannot be captured. */

/* Robots beyond the conditioning limit (INTEGRATION.md).  The fp64 sweep inversion of the solve is accurate up to a scaled
 * condition number max_i H_ii (H^-1)_ii of about 1e5; above 1.5e5 an instance returns code 4 with no trusted wrench — a
 * robot lying on its side (about 3e5) is the common case.  hmpc_set_refinement(ctx, 1) hands every instance above 1.5e4 whose
 * pivots are all positive to the refinement class, one more launch at the end of the solve: it solves the QP again from
 * the unconstrained minimiser, then refines the KKT solution of the final working set against the stored Hessian (up to
 * four rounds, residuals in fp64) and accepts it only at a KKT point (code 0 and HMPC_STATUS_REFINED); otherwise the
 * instance keeps code 4.  Above 1e9, with a non-positive pivot, or with more stance blocks than the class holds (double
 * support up to horizon 14, single support up to 16) it keeps code 4 as well.  The class records an empty working set: a
 * warm call after it starts cold.  Default 0: every call, status word and launch as without this switch.  Applies to every
 * solve of the context (device-resident, host-buffer, rollout).  hmpc_reference_set_refinement does the same for the
 * reference boundary's one-robot context. */
HMPC_EXTERNC int hmpc_set_refinement(hmpc_ctx* ctx, int on);
HMPC_EXTERNC void hmpc_reference_set_refinement(int on);

/* number of kernel launches hmpc_solve_device enqueues per call (one per size class, + the refinement class when on) */
HMPC_EXTERNC int hmpc_launches_per_solve(const hmpc_ctx* ctx);
/* launch configuration of size class `cls` (0, 1, 2, or HMPC_REFINEMENT_CLASS): out[0..5] = threads per CTA, dynamic shared
 * memory bytes, working-set capacity, resident-grid cap (CTAs), max blocks of 6 variables, sweep strip width */
#define HMPC_REFINEMENT_CLASS 3
HMPC_EXTERNC int hmpc_class_config(const hmpc_ctx* ctx, int cls, int* out);

/* Debug/parity hook: run only the assembly stage for B packed device records and write the
 * full (un-reduced) fp32 QP data per instance: H [n*n] row-major (upper triangle valid,
 * mirrored), g [n], the 16x12 constraint block [192], lb/ub [16N].  n = 12*horizon. */
HMPC_EXTERNC int hmpc_assemble_device(hmpc_ctx* ctx, const void* d_records, int B, float* d_H,
                                      float* d_g, float* d_Fblk, float* d_lb, float* d_ub,
                                      void* stream);

#endif /* HECTOR_MPC_B200_H */
