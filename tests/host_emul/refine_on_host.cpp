// tests/host_emul/refine_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only): the device-resident solve with refinement on
// (hmpc_set_refinement: classes 0-2 hand instances beyond the conditioning limit to the refinement class at the end of the
// chain) on the host.
//
// Built by tests/test_refinement.py exactly like kernel_source_on_host.cpp, whose CTA emulation, kernel variants and class
// configuration it reuses by inclusion (same translation unit); everything that library exports stays available.  With
// -DREFINE_RACE_MAIN it is a command-line driver for the ThreadSanitizer build (packed records in a file).
#include "kernel_source_on_host.cpp"

#include <cstdio>

namespace {
// hmpc_capi.cu HMPC_FOR_VARIANT, variants 20 + b: the refinement class
void launch_refine(int variant, const hmpc::KernelArgs& ka)
{
  switch (variant) {
    case 20: run_cta(64, [=] { hmpc::hmpc_solve_kernel<64, 1, 0, 3>(ka); }); break;
    case 21: run_cta(128, [=] { hmpc::hmpc_solve_kernel<128, 1, 0, 3>(ka); }); break;
    case 22: run_cta(192, [=] { hmpc::hmpc_solve_kernel<192, 1, 0, 3>(ka); }); break;
    case 23: run_cta(256, [=] { hmpc::hmpc_solve_kernel<256, 1, 0, 3>(ka); }); break;
    default: run_cta(384, [=] { hmpc::hmpc_solve_kernel<384, 1, 0, 3>(ka); }); break;
  }
}
// hmpc_capi.cu build_refine_class, minus the CUDA occupancy calls
ClassCfg refine_class(int N)
{
  ClassCfg k{};
  const int rs = hmpc::record_stride(N);
  for (int nb = 2 * N;; nb = N) {
    const int n = 6 * nb, nt8 = (n + 7) / 8;
    const int w_sweep = (nt8 + 1) / 2, w_rows = (nb + 2) / 3, warps = w_sweep > w_rows ? w_sweep : w_rows;
    int bucket = 0;
    while (bucket < 4 && kBucketThreads[bucket] < 32 * warps) bucket++;
    k.nb_cap = nb;
    k.variant = 20 + bucket;
    k.tcap = 0;
    k.qmax = n;
    k.L = hmpc::refine_layout(N, nb, k.qmax, rs, kBucketThreads[bucket] / 32);
    while (k.L.total > 226 * 1024 && k.qmax > 4) {
      k.qmax -= 4;
      k.L = hmpc::refine_layout(N, nb, k.qmax, rs, kBucketThreads[bucket] / 32);
    }
    if (nb == N || (k.L.total <= 226 * 1024 && k.qmax >= hmpc::class_qmax(N, 1))) break;
  }
  return k;
}
}  // namespace

extern "C" {

/* refinement class of horizon N: out[0..4] = threads, shared-memory bytes, working-set capacity, blocks of 6 variables,
 * variant */
void emul_refine_config(int N, int* out)
{
  const ClassCfg k = refine_class(N);
  out[0] = kBucketThreads[k.variant - 20];
  out[1] = k.L.total;
  out[2] = k.qmax;
  out[3] = k.nb_cap;
  out[4] = k.variant;
}

/* The device-resident chain of hmpc_capi.cu (enqueue_solve) on B <= 1024 packed records: class 0 over every robot
 * (classifying on the way), class 1 and class 2 through the escalation lists, then — refine != 0 — the refinement class over
 * the instances classes 0-2 handed over.  refine != 0: classes 0-2 hand over above kappa_refine, the refinement class's own
 * limit is kappa_max_refined; refine == 0: classes 0-2 stop at kappa_max (hmpc_capi.cu's default 1.5e5) and nothing is
 * handed over.  ws [B][WS_STATE_INTS] (written back; proposed when warm != 0) or NULL.
 * Outputs: wrench [B][12N] floats, wrench64 [B][12N] doubles or NULL, status [B], launched[4] = instances class 0 kept,
 * class 1, class 2, the refinement class (NULL to skip). */
int emul_solve_refine(const unsigned char* records, int B, int N, float dt, float f_max, int refine, double kappa_max,
                      double kappa_refine, double kappa_max_refined, int* ws, int warm, float* wrench, double* wrench64,
                      int* status, int* launched)
{
  if (B < 1 || B > 1024 || !records) return 1;
  ClassCfg cls[3];
  const int ncls = build_classes(N, cls);
  std::vector<int> block(16 + 4 * (size_t)B, 0);
  int* counts = block.data();      // [8] words of this call (lengths, wave barrier, refinement length), [8] the next call's
  int* lists = counts + 16;        // lists + i * B: class i's list, i = 1, 2; i = 3: the refinement class's
  for (int e = 8; e < 16; e++) counts[e] = 0x55;  // the class-0 launch must clear words 8..12 (the next call's)
  counts[0] = B;
  hmpc::KernelArgs base{};
  base.records = records;
  base.rec_stride = hmpc::record_stride(N);
  base.batch = B;
  base.horizon = N;
  base.dt = dt;
  base.f_max = f_max;
  base.max_iter = 500;
  base.tol_kkt = 1e-9;  // hmpc_capi.cu's defaults
  base.tol_dep = 1e-11;
  base.block_min = 2;
  base.block_rounds = 4;
  base.wrench = wrench;
  base.wrench64 = wrench64;
  base.status = status;
  base.ws_state = ws;
  base.ws_shift = 1;
  for (int i = 0; i < ncls; i++) {
    if (launched) launched[i] = counts[i];
    if (counts[i] == 0) continue;
    hmpc::KernelArgs ka = base;
    ka.kappa_max = refine ? kappa_refine : kappa_max;
    ka.warm_start = (ws && warm) ? 1 : 0;
    ka.list = i == 0 ? nullptr : lists + (size_t)i * B;
    ka.split_nb = i == 0 ? cls[0].nb_cap : -1;
    ka.counts_next = i == 0 ? counts + 8 : nullptr;
    ka.wave_sync = i == 0 ? reinterpret_cast<unsigned*>(counts + 3) : nullptr;
    ka.counts = counts;
    ka.cls = i;
    ka.esc_list = i + 1 < ncls ? lists + (size_t)(i + 1) * B : nullptr;
    if (refine) {
      ka.ref_list = lists + (size_t)3 * B;
      ka.ref_count = counts + 4;
    }
    ka.nb_cap = cls[i].nb_cap;
    ka.qmax = cls[i].qmax;
    ka.tcap = cls[i].tcap;
    ka.L = cls[i].L;
    launch_variant(cls[i].variant, ka);
    if (i == 0) {
      if (counts[8] | counts[9] | counts[10] | counts[11] | counts[12]) return 2;  // the next call's words not cleared
      if (launched) launched[0] = B - counts[1];
    }
  }
  if (launched) launched[3] = refine ? counts[4] : 0;
  if (refine && counts[4] > 0) {
    const ClassCfg k = refine_class(N);
    hmpc::KernelArgs ka = base;  // hmpc_capi.cu refine_args
    ka.kappa_max = kappa_max_refined;
    ka.list = lists + (size_t)3 * B;
    ka.counts = counts + 4;
    ka.split_nb = -1;
    ka.nb_cap = k.nb_cap;
    ka.qmax = k.qmax;
    ka.tcap = 0;
    ka.L = k.L;
    launch_refine(k.variant, ka);
  }
  return 0;
}

}  // extern "C"

#ifdef REFINE_RACE_MAIN
int main(int argc, char** argv)
{
  // usage: refine_race_driver <packed records file> <horizon>: refinement on; prints the status words
  if (argc < 3) return 2;
  const int N = atoi(argv[2]);
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<unsigned char> buf(1 << 22);
  const size_t nbytes = fread(buf.data(), 1, buf.size(), f);
  fclose(f);
  const int B = (int)(nbytes / hmpc::record_stride(N));
  std::vector<float> w((size_t)B * 12 * N);
  std::vector<int> st(B), ws((size_t)B * hmpc::WS_STATE_INTS, 0);
  int launched[4] = {0, 0, 0, 0};
  const int rc = emul_solve_refine(buf.data(), B, N, 0.04f, 500.f, 1, 1.5e5, 1.5e4, 1e9, ws.data(), 1, w.data(), nullptr, st.data(),
                                   launched);
  printf("rc %d B %d launched %d %d %d %d status", rc, B, launched[0], launched[1], launched[2], launched[3]);
  for (int i = 0; i < B; i++) printf(" %08x", (unsigned)st[i]);
  printf("\n");
  return rc;
}
#endif
