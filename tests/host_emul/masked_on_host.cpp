// tests/host_emul/masked_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only): the masked solve (hmpc_solve_device_masked:
// the selection kernel turns a per-robot mask into class 0's instance list, then the chain runs over it) on the host.
//
// Built by tests/test_masked_solve.py exactly like kernel_source_on_host.cpp, whose CTA emulation, kernel variants and class
// configuration it reuses by inclusion through warm_start_on_host.cpp (same translation unit, so emul_solve_warm, the full
// solve it is compared against, is exported too).  With -DMASKED_RACE_MAIN it is a command-line driver for the
// ThreadSanitizer build of the selection kernel.
#include "warm_start_on_host.cpp"

#include <cstdio>

namespace {
void run_select(const unsigned char* mask, int B, int* list, int* count)
{
  run_cta(hmpc::SELECT_THREADS, [=] { hmpc::hmpc_select_kernel<hmpc::SELECT_THREADS>(mask, B, list, count); });
}
}  // namespace

extern "C" {

int emul_select_threads() { return hmpc::SELECT_THREADS; }

/* the selection kernel on one emulated CTA: list[0 .. *count) = the robots i < B with mask[i] != 0 */
void emul_select(const unsigned char* mask, int B, int* list, int* count) { run_select(mask, B, list, count); }

/* The masked device-resident chain of hmpc_capi.cu (enqueue_solve with a mask) on B <= 1024 packed records: the selection
 * kernel, class 0 over its list (classifying on the way), class 1 and class 2 through the escalation lists.  Warm-started
 * from `ws` [B][WS_STATE_INTS] with `shifts` [B] per robot (NULL: 1 each), as hmpc_solve_device_masked passes them; ws NULL:
 * a cold solve.  Outputs: wrench [B][12N] floats, status [B], launched[3] = instances class 0 kept, class 1, class 2 (NULL to
 * skip).  Returns 2 when class 0 did not clear the next call's length words. */
int emul_solve_masked(const unsigned char* records, int B, int N, const unsigned char* mask, int* ws, const int* shifts,
                      float* wrench, int* status, int* launched)
{
  if (B < 1 || B > 1024 || !records || !mask) return 1;
  ClassCfg cls[3];
  const int ncls = build_classes(N, cls);
  std::vector<int> block(16 + 4 * (size_t)B, 0);
  int* counts = block.data();      // [8] words of this call, [8] the next call's (cleared by the class-0 launch)
  int* lists = counts + 16 - B;    // lists + i * B: class i's list, i = 1, 2; i = 4: class 0's
  int* list0 = lists + (size_t)4 * B;
  for (int e = 8; e < 13; e++) counts[e] = 0x55;
  counts[0] = 0x55;                // the selection kernel writes the length
  run_select(mask, B, list0, counts);
  for (int i = 0; i < ncls; i++) {
    if (launched) launched[i] = counts[i];
    if (counts[i] == 0) continue;
    hmpc::KernelArgs ka{};
    ka.records = records;
    ka.rec_stride = hmpc::record_stride(N);
    ka.batch = B;
    ka.horizon = N;
    ka.dt = 0.04f;
    ka.f_max = 500.f;
    ka.max_iter = 500;
    ka.tol_kkt = 1e-9;  // hmpc_capi.cu's defaults
    ka.tol_dep = 1e-11;
    ka.kappa_max = 1.5e5;
    ka.block_min = 2;
    ka.block_rounds = 4;
    ka.wrench = wrench;
    ka.status = status;
    ka.warm_start = ws ? 1 : 0;
    ka.ws_state = ws;
    ka.ws_shift = 1;
    ka.ws_shifts = shifts;
    ka.list = i == 0 ? list0 : lists + (size_t)i * B;
    ka.split_nb = i == 0 ? cls[0].nb_cap : -1;
    ka.counts_next = i == 0 ? counts + 8 : nullptr;
    ka.wave_sync = i == 0 ? reinterpret_cast<unsigned*>(counts + 3) : nullptr;
    ka.counts = counts;
    ka.cls = i;
    ka.esc_list = i + 1 < ncls ? lists + (size_t)(i + 1) * B : nullptr;
    ka.nb_cap = cls[i].nb_cap;
    ka.qmax = cls[i].qmax;
    ka.tcap = cls[i].tcap;
    ka.L = cls[i].L;
    launch_variant(cls[i].variant, ka);
    if (i == 0) {
      if (counts[8] | counts[9] | counts[10] | counts[11] | counts[12]) return 2;
      if (launched) launched[0] = counts[0] - counts[1];
    }
  }
  return 0;
}

}  // extern "C"

#ifdef MASKED_RACE_MAIN
int main()
{
  // the selection kernel on masks of several sizes and densities; prints "ok" when every list is the serial one
  unsigned rng = 12345u;
  const int sizes[] = {1, 37, 512, 1300};
  const int dens[] = {0, 20, 50, 100};
  int bad = 0;
  for (int B : sizes)
    for (int d : dens) {
      std::vector<unsigned char> mask(B);
      for (int i = 0; i < B; i++) {
        rng = rng * 1664525u + 1013904223u;
        mask[i] = (int)((rng >> 8) % 100) < d ? (unsigned char)(1 + (rng >> 24) % 255) : 0;
      }
      std::vector<int> list(B, -1);
      int count = -1;
      run_select(mask.data(), B, list.data(), &count);
      int n = 0;
      for (int i = 0; i < B; i++)
        if (mask[i]) bad += (n < count && list[n] == i) ? 0 : 1, n++;
      bad += (n == count) ? 0 : 1;
    }
  printf(bad ? "mismatch %d\n" : "ok\n", bad);
  return bad ? 1 : 0;
}
#endif
