// tests/host_emul/predict_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only): the prediction kernel (the MPC's plan).
//
// Built by tests/test_prediction.py with the same host-buildable device header and flags as kernel_source_on_host.cpp,
// which it includes whole, plus emul_predict: hmpc_predict_kernel over its whole grid, one CTA after another, the threads
// of each on OS threads at once (its warps shuffle).  The launch shape comes from the library's own hmpc_chain.h
// (predict_grid), the kernel's arguments are those of hmpc_capi.cu's launch_predict.
#include "kernel_source_on_host.cpp"

namespace {
template <typename T>
void run_predict(const unsigned char* rows, int row_stride, int batch, int N, float dt, const unsigned char* mask,
                 const T* wrench, T* pred)
{
  const int grid = hmpc::predict_grid(batch);
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
        hmpc::hmpc_predict_kernel<T>(rows, row_stride, batch, N, dt, mask, wrench, pred);
        hmpc_emul_cta = nullptr;
      });
    for (auto& x : th) x.join();
    delete cta;
  }
}
}  // namespace

extern "C" {

int emul_predict_threads() { return hmpc::PREDICT_THREADS; }
int emul_predict_grid(int batch) { return hmpc::predict_grid(batch); }

/* the prediction kernel on B rows of `rows` (row_stride bytes apart; the first 19 floats of a row are p v q w r), the
 * problem dt `dt`, mask NULL or [B].  double64 != 0: wrench [B][12N] and pred [B][N][12] are doubles (the host call's
 * instantiation), else floats (the device call's). */
void emul_predict(const unsigned char* rows, int row_stride, int B, int N, float dt, const unsigned char* mask, int double64,
                  const void* wrench, void* pred)
{
  if (double64)
    run_predict<double>(rows, row_stride, B, N, dt, mask, static_cast<const double*>(wrench), static_cast<double*>(pred));
  else
    run_predict<float>(rows, row_stride, B, N, dt, mask, static_cast<const float*>(wrench), static_cast<float*>(pred));
}

}  // extern "C"
