// tests/host_emul/race_driver.cpp — TEST INFRASTRUCTURE (CPU suite only).
// Runs the host-compiled kernel source (kernel_source_on_host.cpp) from the command line.  Built with -fsanitize=thread by
// tests/test_kernel_source_on_host.py: every CUDA thread of the emulated CTA is an OS thread and __syncthreads / __syncwarp /
// the warp primitives are real synchronisation, so ThreadSanitizer reports any pair of conflicting shared-memory (or global)
// accesses that the kernel does not order with a barrier — a CPU-side racecheck of the kernel's source.  (It cannot see
// hazards specific to the GPU's async proxy; the PTX fences stay in the product.)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

extern "C" int emul_solve(const unsigned char* records, const unsigned char* raw, int B, int N, int hostlists, int refine,
                          const unsigned char* mask, int* ws, int warm, int shift, const int* shifts, float* wrench,
                          double* wrench64, int* status, float* tau, int* launched, float* dH, float* dg, float* dF, float* dlb,
                          float* dub);
extern "C" void emul_select(const unsigned char* mask, int B, int* list, int* count);
extern "C" int emul_record_stride(int N);
extern "C" int emul_ws_ints();

// the selection kernel on masks of several sizes and densities; prints "ok" when every list is the serial one
static int select_main()
{
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
      emul_select(mask.data(), B, list.data(), &count);
      int n = 0;
      for (int i = 0; i < B; i++)
        if (mask[i]) bad += (n < count && list[n] == i) ? 0 : 1, n++;
      bad += (n == count) ? 0 : 1;
    }
  printf(bad ? "mismatch %d\n" : "ok\n", bad);
  return bad ? 1 : 0;
}

int main(int argc, char** argv)
{
  // usage: race_driver select
  //        race_driver <file> <horizon> [raw] [warm] [refine]   (raw: the file holds update_data_t records, 3016 bytes each)
  if (argc == 2 && strcmp(argv[1], "select") == 0) return select_main();
  if (argc < 3) return 2;
  const int N = atoi(argv[2]);
  bool raw = false, warm = false, refine = false;
  for (int a = 3; a < argc; a++) {
    raw |= strcmp(argv[a], "raw") == 0;
    warm |= strcmp(argv[a], "warm") == 0;
    refine |= strcmp(argv[a], "refine") == 0;
  }
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<unsigned char> buf(1 << 22);
  const size_t n = fread(buf.data(), 1, buf.size(), f);
  fclose(f);
  const int B = (int)(n / (raw ? 3016 : emul_record_stride(N)));
  const unsigned char* rec = raw ? nullptr : buf.data();
  const unsigned char* in = raw ? buf.data() : nullptr;
  std::vector<float> w((size_t)B * 12 * N), tau((size_t)B * 10);
  std::vector<double> w64((size_t)B * 12 * N);
  std::vector<int> st(B), ws((size_t)B * emul_ws_ints(), 0);
  int launched[4] = {0, 0, 0, 0};
  int* wsp = (warm || refine) ? ws.data() : nullptr;  // working sets: recorded, and proposed by the second tick of `warm`
  int rc = emul_solve(rec, in, B, N, 0, refine, nullptr, wsp, refine, 0, nullptr, w.data(), w64.data(), st.data(), tau.data(),
                      launched, 0, 0, 0, 0, 0);
  if (warm && rc == 0) {  // second tick on the same records: the stored working sets are proposed to the block start
    rc = emul_solve(rec, in, B, N, 0, refine, nullptr, wsp, 1, 0, nullptr, w.data(), w64.data(), st.data(), tau.data(),
                    launched, 0, 0, 0, 0, 0);
    for (int i = 0; i < B; i++)
      if (((st[i] >> 8) & 0xfff) != 0) rc = 3;  // proposing the optimal set must need no change at all
  }
  int bad = 0;
  for (int i = 0; i < B; i++) bad += (st[i] & 0xff) != 0;
  printf("rc %d B %d launched %d %d %d %d not_converged %d status", rc, B, launched[0], launched[1], launched[2], launched[3], bad);
  for (int i = 0; i < B; i++) printf(" %08x", (unsigned)st[i]);
  printf("\n");
  return rc || bad;
}
