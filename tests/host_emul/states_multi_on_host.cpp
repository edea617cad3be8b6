// tests/host_emul/states_multi_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only): candidate commands per robot, solved
// from its state (hmpc_solve_states_device_multi).
//
// Built by tests/test_states_multi.py with the same host-buildable device header and flags as kernel_source_on_host.cpp.  It
// includes multi_on_host.cpp (and through it certify_on_host.cpp and kernel_source_on_host.cpp) whole, so one library holds
// the single preparation (emul_prepare), the single solve (emul_solve), the certificate (emul_certify), the multi-query chain
// (emul_solve_multi) and
//   * emul_prepare_traj: the trajectory launch (hmpc_prepare_traj_kernel), over every robot or a list;
//   * emul_solve_states_multi: hmpc_capi.cu's multi-command states chain: the selection kernel over the robot mask, the
//     preparation and the trajectories over its list, the multi-query classes and the cost kernel (emul_solve_multi's, with
//     the same mask: its selection kernel builds the same list again in a slot of its own), then the pick kernel.
// Every launch's arguments and grid come from the library's own hmpc_chain.h (prepare_args, prepare_traj_args, prepare_grid,
// pick_grid).
// Built with -DHMPC_STATES_MULTI_MAIN (and -fsanitize=thread) it is a program that runs the chain on the states of a file.
#include "multi_on_host.cpp"

namespace {
// hmpc_capi.cu's launch_prepare and launch_prepare_traj: every thread of the grid, one at a time
template <class F>
void run_threads(int grid, F fn)
{
  const unsigned NT = hmpc::PREPARE_THREADS;
  for (int t = 0; t < grid * hmpc::PREPARE_THREADS; t++) {
    blockDim = {NT, 1, 1};
    blockIdx = {(unsigned)t / NT, 0, 0};
    threadIdx = {(unsigned)t % NT, 0, 0};
    gridDim = {(unsigned)grid, 1, 1};
    fn();
  }
}
void run_prepare(const hmpc::PrepareArgs& pa)
{
  run_threads(hmpc::prepare_grid(pa.batch), [&] {
    hmpc::hmpc_prepare_kernel(pa.states, pa.batch, pa.N, pa.dtMPC, pa.records, pa.rec_stride, pa.list, pa.count);
  });
}
void run_prepare_traj(const hmpc::PrepareTrajArgs& pa)
{
  run_threads(hmpc::prepare_grid(pa.batch * pa.K), [&] {
    hmpc::hmpc_prepare_traj_kernel(pa.states, pa.batch, pa.K, pa.cmd, pa.N, pa.dtMPC, pa.traj, pa.list, pa.count);
  });
}

// hmpc_capi.cu's launch_pick: each CTA of its grid on PREDICT_THREADS OS threads
void run_pick(unsigned char* records, int B, int K, int N, float f_max, const unsigned char* mask, const float* traj,
              const float* wrench, const int* status, const double* cost, int* best, float* tau)
{
  const int grid = hmpc::pick_grid(B);
  const unsigned NT = hmpc::PREDICT_THREADS;
  for (int b = 0; b < grid; b++) {
    hmpc_emul::Cta* cta = new hmpc_emul::Cta;
    cta->bar.count = NT;
    for (int w = 0; w < 32; w++) cta->warps[w].bar.count = 32;
    std::vector<std::thread> th;
    th.reserve(NT);
    for (unsigned t = 0; t < NT; t++)
      th.emplace_back([=] {
        threadIdx = {t, 0, 0};
        blockIdx = {(unsigned)b, 0, 0};
        blockDim = {NT, 1, 1};
        gridDim = {(unsigned)grid, 1, 1};
        hmpc_emul_cta = cta;
        hmpc::hmpc_pick_kernel<float>(records, hmpc::record_stride(N), B, K, N, f_max, mask, traj, wrench, status, cost, best,
                                      tau);
        hmpc_emul_cta = nullptr;
      });
    for (auto& x : th) x.join();
    delete cta;
  }
}

hmpc::SolveIO states_io(const unsigned char* states, double dtMPC, unsigned char* records, int B)
{
  hmpc::SolveIO io;
  io.states = states;
  io.dt_mpc = dtMPC;
  io.records = records;
  io.batch = B;
  return io;
}
}  // namespace

extern "C" {

/* the trajectories of B states' K commands cmd [B][K][7] into traj [B][K][12N], over every robot or over `list` [*count]
 * when list is not NULL */
void emul_prepare_traj(const unsigned char* states, int B, int K, const double* cmd, int N, double dtMPC, float* traj,
                       const int* list, const int* count)
{
  hmpc::ChainLists lists;
  lists.counts = const_cast<int*>(count);
  lists.list[0] = const_cast<int*>(list);
  hmpc::MultiIO mq;
  mq.traj = traj;
  mq.K = K;
  mq.cmd = cmd;
  run_prepare_traj(hmpc::prepare_traj_args(N, states_io(states, dtMPC, nullptr, B), lists, mq));
}

/* The multi-command states chain on B robots with K commands each (B*K <= 4096): states [B] hmpc_state_t, cmd [B][K][7],
 * refine: hmpc_set_refinement, mask NULL or [B].  Outputs: records [B][stride], traj [B][K][12N], wrench [B*K][12N] floats,
 * status and cost [B*K], best [B], tau [B][10] or NULL, launched[4] as in emul_solve_multi (or NULL).  Returns 0, or what
 * emul_solve_multi returns. */
int emul_solve_states_multi(const unsigned char* states, const double* cmd, double dtMPC, unsigned char* records, float* traj,
                            int B, int K, int N, int refine, const unsigned char* mask, float* wrench, int* status,
                            double* cost, int* best, float* tau, int* launched)
{
  if (B < 1 || K < 1 || B * K > 4096 || !states || !cmd || !records || !traj) return 1;
  std::vector<int> mem(hmpc::ClassSlot::cls_slot_ints(B), 0);
  const hmpc::ClassSlot slot{mem.data(), B, 0};
  const hmpc::ChainLists lists = hmpc::slot_lists(slot, mask != nullptr, refine != 0);
  if (mask) run_select(mask, B, slot.list0(), slot.counts());
  hmpc::MultiIO mq;
  mq.traj = traj;
  mq.K = K;
  mq.cmd = cmd;
  const hmpc::SolveIO io = states_io(states, dtMPC, records, B);
  run_prepare(hmpc::prepare_args(N, io, lists));
  run_prepare_traj(hmpc::prepare_traj_args(N, io, lists, mq));
  if (int rc = emul_solve_multi(records, nullptr, B, K, N, refine, mask, traj, wrench, nullptr, status, cost, launched)) return rc;
  run_pick(records, B, K, N, settings(refine).f_max, mask, traj, wrench, status, cost, best, tau);
  return 0;
}

}  // extern "C"

#ifdef HMPC_STATES_MULTI_MAIN
// usage: states_multi_tsan <file> <horizon> <K> [refine] — the file holds hmpc_state_t rows; command k of robot i is the
// state's own with body vx moved by 0.1 k and the yaw rate by 0.05 k.  Prints best and the status words and exits non-zero
// when a robot has no converged candidate.
int main(int argc, char** argv)
{
  if (argc < 4) return 2;
  const int N = atoi(argv[2]), K = atoi(argv[3]);
  const bool refine = argc > 4 && strcmp(argv[4], "refine") == 0;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<unsigned char> buf(1 << 20);
  const size_t n = fread(buf.data(), 1, buf.size(), f);
  fclose(f);
  const int B = (int)(n / 352), nw = 12 * N;
  std::vector<double> cmd((size_t)B * K * 7);
  for (int i = 0; i < B; i++)
    for (int k = 0; k < K; k++) {
      double* c = cmd.data() + ((size_t)i * K + k) * 7;
      memcpy(c, buf.data() + (size_t)i * 352 + 32 * 8, 7 * sizeof(double));
      c[2] += 0.1 * k;
      c[4] += 0.05 * k;
    }
  std::vector<unsigned char> rec((size_t)B * hmpc::record_stride(N));
  std::vector<float> traj((size_t)B * K * nw), w((size_t)B * K * nw), tau((size_t)B * 10);
  std::vector<int> st((size_t)B * K, -1), best(B, -2);
  std::vector<double> cost((size_t)B * K);
  int launched[4] = {0, 0, 0, 0};
  const int rc = emul_solve_states_multi(buf.data(), cmd.data(), 0.04, rec.data(), traj.data(), B, K, N, refine, nullptr, w.data(),
                                         st.data(), cost.data(), best.data(), tau.data(), launched);
  int none = 0;
  for (int i = 0; i < B; i++) none += best[i] < 0;
  printf("rc %d B %d K %d launched %d %d %d %d no_best %d best", rc, B, K, launched[0], launched[1], launched[2], launched[3], none);
  for (int i = 0; i < B; i++) printf(" %d", best[i]);
  printf(" status");
  for (int r = 0; r < B * K; r++) printf(" %08x", (unsigned)st[r]);
  printf("\n");
  return rc || none;
}
#endif
