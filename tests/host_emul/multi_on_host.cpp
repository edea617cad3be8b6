// tests/host_emul/multi_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only): the multi-query solve (several reference
// trajectories per robot).
//
// Built by tests/test_multi_query.py with the same host-buildable device header and flags as kernel_source_on_host.cpp.  It
// includes certify_on_host.cpp (and through it kernel_source_on_host.cpp) whole, so one library holds the single solve
// (emul_solve), the certificate (emul_certify) and emul_solve_multi: hmpc_capi.cu's multi-query chain, the selection kernel
// over the robot mask, class 0 over the robots, the later classes and the refinement class over the lists the kernels
// build, then the cost kernel.  Variants, class shapes and every launch's arguments come from the library's own
// hmpc_chain.h (plan_classes with mq, multi_launch_args, multi_cost_grid).  Each launch runs on one emulated CTA, so every
// class's scratch is one row.  Built with -DHMPC_MULTI_MAIN (and -fsanitize=thread) it is a program that solves the records
// of a file for K candidates each.
#include "certify_on_host.cpp"

namespace {
void run_class_mq(const hmpc::SolverSettings& S, int N, int ncls, int cls, const hmpc::ClassCfg& k, const hmpc::SolveIO& io,
                  const hmpc::ChainLists& lists, const hmpc::MultiIO& mq)
{
  const hmpc::KernelArgs ka = hmpc::multi_launch_args(S, N, ncls, cls, k, io, lists, mq);
  switch (k.variant) {
#define HMPC_RUN_MQ(ID, NT, MB, NF, CL) \
  case ID: run_cta(NT, [=] { hmpc::hmpc_solve_kernel<NT, MB, NF, CL, true>(ka); }); return;
    HMPC_MQ_VARIANTS(HMPC_RUN_MQ)
#undef HMPC_RUN_MQ
  }
  hmpc_emul::die("no such multi-query kernel variant");
}

template <typename T>
void run_multi_cost(const unsigned char* rows, hmpc::RowLayout lay, int B, int K, int N, float dt, const unsigned char* mask,
                    const float* traj, const T* wrench, double* cost)
{
  const int grid = hmpc::multi_cost_grid((long long)B * K);
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
        hmpc::hmpc_multi_cost_kernel<T>(rows, lay, B, K, N, dt, mask, traj, wrench, cost);
        hmpc_emul_cta = nullptr;
      });
    for (auto& x : th) x.join();
    delete cta;
  }
}
}  // namespace

extern "C" {

/* hmpc_solve_device_multi (packed `records`, float `wrench`) or hmpc_solve_batch_multi's chain (update_data_t `raw` read in
 * place, double `wrench64`) on B robots with K candidate trajectories each, traj [B][K][12N] floats.  refine:
 * hmpc_set_refinement.  mask NULL or [B].  Outputs [B*K] rows: wrench / wrench64 [.][12N], status, cost (NULL: no cost
 * launch; the cost kernel reads the wrench the call stores).  launched[4] = the entries of the lists of classes 0-2 and of
 * the refinement class (class 0: robots), or NULL.  Returns 0, 1 on bad arguments, 2 when class 0 did not clear the next
 * call's length words. */
int emul_solve_multi(const unsigned char* records, const unsigned char* raw, int B, int K, int N, int refine,
                     const unsigned char* mask, const float* traj, float* wrench, double* wrench64, int* status, double* cost,
                     int* launched)
{
  if (B < 1 || K < 1 || B * K > 4096 || (!records && !raw) || (!wrench && !wrench64)) return 1;
  const hmpc::SolverSettings S = settings(refine);
  hmpc::ClassCfg cls[3], ref;
  const int ncls = hmpc::plan_classes(N, cls, ref, true);
  if (ncls == 0) return 1;
  hmpc::SolveIO io;
  io.records = records;
  io.raw = raw;
  io.batch = B;
  io.wrench = wrench;
  io.wrench64 = wrench64;
  io.status = status;
  io.mask = mask;
  std::vector<float> scratch(4 * (size_t)hmpc::mq_scratch_floats(N), 0.f);
  hmpc::MultiIO mq;
  mq.traj = traj;
  mq.K = K;
  for (int i = 0; i < 4; i++) mq.scratch[i] = scratch.data() + (size_t)i * hmpc::mq_scratch_floats(N);
  std::vector<int> mem(hmpc::ClassSlot::cls_slot_ints(B * K), 0);
  const hmpc::ClassSlot slot{mem.data(), B * K, 0};
  int* next = slot.counts_next();
  for (int w = 0; w < 5; w++) next[w] = 0x55;  // the class-0 launch must clear them
  const hmpc::ChainLists lists = hmpc::slot_lists(slot, mask != nullptr, S.refine);
  if (mask) run_select(mask, B, slot.list0(), slot.counts());
  int la[4] = {0, 0, 0, 0};
  for (int i = 0; i < ncls; i++) {
    const int n = (i == 0 && !mask) ? B : lists.counts[i];
    if (n == 0) continue;
    run_class_mq(S, N, ncls, i, cls[i], io, lists, mq);
    la[i] = n;
    if (i == 0 && (next[0] | next[1] | next[2] | next[3] | next[4])) return 2;
  }
  if (S.refine && (la[3] = *lists.ref_count) > 0) run_class_mq(S, N, ncls, hmpc::REFINE_CLASS, ref, io, lists, mq);
  if (launched) memcpy(launched, la, sizeof la);
  if (cost) {
    const float dt = S.dt;
    if (raw)
      run_multi_cost<double>(raw, hmpc::update_rows(), B, K, N, dt, mask, traj, wrench64, cost);
    else
      run_multi_cost<float>(records, hmpc::packed_rows(N), B, K, N, dt, mask, traj, wrench, cost);
  }
  return 0;
}

int emul_mq_variant() { return hmpc::MQ_VARIANT; }

}  // extern "C"

#ifdef HMPC_MULTI_MAIN
// usage: multi_tsan <file> <horizon> <K> [refine] — the file holds packed records; candidate k of robot i is the record's own
// trajectory with entry (step k % N, component k % 12) moved by 0.05 k.  Prints the status words and exits non-zero when a
// candidate did not converge.
int main(int argc, char** argv)
{
  if (argc < 4) return 2;
  const int N = atoi(argv[2]), K = atoi(argv[3]);
  const bool refine = argc > 4 && strcmp(argv[4], "refine") == 0;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<unsigned char> buf(1 << 22);
  const size_t n = fread(buf.data(), 1, buf.size(), f);
  fclose(f);
  const int rs = hmpc::record_stride(N), B = (int)(n / rs), nw = 12 * N;
  std::vector<float> traj((size_t)B * K * nw), w((size_t)B * K * nw);
  std::vector<int> st((size_t)B * K, -1);
  std::vector<double> cost((size_t)B * K);
  for (int i = 0; i < B; i++)
    for (int k = 0; k < K; k++) {
      float* t = traj.data() + ((size_t)i * K + k) * nw;
      memcpy(t, buf.data() + (size_t)i * rs + 54 * 4, nw * sizeof(float));
      t[12 * (k % N) + k % 12] += 0.05f * (float)k;
    }
  int launched[4] = {0, 0, 0, 0};
  const int rc = emul_solve_multi(buf.data(), nullptr, B, K, N, refine, nullptr, traj.data(), w.data(), nullptr, st.data(),
                                  cost.data(), launched);
  int bad = 0;
  for (int r = 0; r < B * K; r++) bad += (st[r] & 0xff) != 0;
  printf("rc %d B %d K %d launched %d %d %d %d not_converged %d status", rc, B, K, launched[0], launched[1], launched[2],
         launched[3], bad);
  for (int r = 0; r < B * K; r++) printf(" %08x", (unsigned)st[r]);
  printf("\n");
  return rc || bad;
}
#endif
