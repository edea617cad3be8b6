// tests/host_emul/carry_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only): the carry kernel of the sharded masked calls.
//
// Built by tests/test_sharded_warm.py with the same host-buildable device header and flags as kernel_source_on_host.cpp,
// which it includes whole, plus
//   * emul_carry: hmpc_carry_kernel over its whole grid, every CTA's threads on OS threads at once;
//   * with -DHMPC_CARRY_MAIN, a main() that checks the carry on a few shapes, for the ThreadSanitizer build: two threads
//     that touch the same bytes, one of them storing, are reported.
// The launch shape comes from the library's own hmpc_chain.h (carry_grid, carry_row_vecs).
#include "kernel_source_on_host.cpp"

namespace {
// hmpc_capi.cu's carry launch (launch_carry): the CTAs one after another, the CARRY_THREADS threads of each at once
void run_carry(const unsigned char* mask, int batch, int N, const float* prev, float* cur)
{
  const int grid = hmpc::carry_grid(batch, N);
  const unsigned NT = hmpc::CARRY_THREADS;
  for (int b = 0; b < grid; b++) {
    std::vector<std::thread> th;
    th.reserve(NT);
    for (unsigned t = 0; t < NT; t++)
      th.emplace_back([=] {
        threadIdx = {t, 0, 0};
        blockIdx = {(unsigned)b, 0, 0};
        blockDim = {NT, 1, 1};
        gridDim = {(unsigned)grid, 1, 1};
        hmpc::hmpc_carry_kernel(mask, batch, hmpc::carry_row_vecs(N), reinterpret_cast<const float4*>(prev),
                                reinterpret_cast<float4*>(cur));
      });
    for (auto& x : th) x.join();
  }
}
}  // namespace

extern "C" {

int emul_carry_threads() { return hmpc::CARRY_THREADS; }
int emul_carry_grid(int batch, int N) { return hmpc::carry_grid(batch, N); }

/* the carry of a sharded masked call: rows i < batch of `cur` ([batch][12N] floats, 16-byte aligned) with mask[i] == 0
 * get row i of `prev` */
void emul_carry(const unsigned char* mask, int batch, int N, const float* prev, float* cur) { run_carry(mask, batch, N, prev, cur); }

}  // extern "C"

#ifdef HMPC_CARRY_MAIN
#include <cstdio>

// usage: carry_tsan — prints "ok" when every listed row kept its bytes and every unlisted row equals the previous buffer's
int main()
{
  unsigned rng = 777u;
  int bad = 0;
  const int shapes[][2] = {{1, 5}, {37, 10}, {130, 16}};
  for (const auto& sh : shapes) {
    const int B = sh[0], N = sh[1], nw = 12 * N;
    std::vector<unsigned char> mask(B);
    std::vector<float> prev((size_t)B * nw), cur((size_t)B * nw), before;
    for (int i = 0; i < B; i++) {
      rng = rng * 1664525u + 1013904223u;
      mask[i] = (rng >> 16) % 3 == 0 ? (unsigned char)(1 + (rng >> 24) % 255) : 0;
    }
    for (size_t e = 0; e < prev.size(); e++) prev[e] = (float)e, cur[e] = -(float)e - 1.f;
    before = cur;
    run_carry(mask.data(), B, N, prev.data(), cur.data());
    for (int i = 0; i < B; i++)
      bad += memcmp(&cur[(size_t)i * nw], mask[i] ? &before[(size_t)i * nw] : &prev[(size_t)i * nw], nw * sizeof(float)) != 0;
  }
  printf(bad ? "mismatch %d\n" : "ok\n", bad);
  return bad ? 1 : 0;
}
#endif
