// tests/host_emul/certify_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only): the certificate kernel.
//
// Built by tests/test_certificate.py with the same host-buildable device header and flags as kernel_source_on_host.cpp,
// which it includes whole, plus emul_certify: hmpc_certify_kernel over its whole grid, one CTA after another, the threads
// of each on OS threads at once (its warps shuffle).  The launch shape and the row layouts come from the library's own
// hmpc_chain.h (certify_grid, packed_rows, update_rows), the kernel's arguments are those of hmpc_capi.cu's launch_certify.
// Built with -DHMPC_CERTIFY_MAIN (and -fsanitize=thread) it is a program that certifies the rows of a file.
#include "kernel_source_on_host.cpp"

#include <cstdio>

namespace {
template <typename T>
void run_certify(const unsigned char* rows, hmpc::RowLayout lay, int batch, int N, float dt, float f_max,
                 const unsigned char* mask, const T* wrench, hmpc::CertOut* cert, T* lambda, double* grad)
{
  const int grid = hmpc::certify_grid(batch);
  const unsigned NT = hmpc::CERT_THREADS;
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
        hmpc::hmpc_certify_kernel<T>(rows, lay, batch, N, dt, f_max, mask, wrench, cert, lambda, grad);
        hmpc_emul_cta = nullptr;
      });
    for (auto& x : th) x.join();
    delete cta;
  }
}
}  // namespace

extern "C" {

int emul_certify_threads() { return hmpc::CERT_THREADS; }
int emul_certify_grid(int batch) { return hmpc::certify_grid(batch); }
int emul_certify_bytes() { return (int)sizeof(hmpc::CertOut); }
/* the kernel's constants: [act_k, act_abs, nnls_dual, nnls_pivot, tiny, stat_tol, primal_tol, compl_tol, eps_rows,
 * nnls_iters] */
void emul_certify_constants(double* out)
{
  const double c[10] = {hmpc::CERT_ACT_K, hmpc::CERT_ACT_ABS,    hmpc::CERT_NNLS_DUAL,  hmpc::CERT_NNLS_PIVOT,
                        hmpc::CERT_TINY,  hmpc::CERT_STAT_TOL,   hmpc::CERT_PRIMAL_TOL, hmpc::CERT_COMPL_TOL,
                        hmpc::CERT_EPS_ROWS, (double)hmpc::CERT_NNLS_ITERS};
  memcpy(out, c, sizeof c);
}

/* the certificate kernel on B rows of `rows`: update_rows != 0 the update_data_t layout, else packed records of horizon N;
 * dt, f_max the problem's; mask NULL or [B].  double64 != 0: wrench [B][12N] and lambda [B][N][2][8] are doubles (the host
 * call's instantiation), else floats (the device call's).  cert [B] (40-byte hmpc_certificate_t), lambda and grad
 * ([B][12N] doubles) may be NULL. */
void emul_certify(const unsigned char* rows, int update_rows, int B, int N, float dt, float f_max, const unsigned char* mask,
                  int double64, const void* wrench, void* cert, void* lambda, double* grad)
{
  const hmpc::RowLayout lay = update_rows ? hmpc::update_rows() : hmpc::packed_rows(N);
  hmpc::CertOut* c = static_cast<hmpc::CertOut*>(cert);
  if (double64)
    run_certify<double>(rows, lay, B, N, dt, f_max, mask, static_cast<const double*>(wrench), c, static_cast<double*>(lambda),
                        grad);
  else
    run_certify<float>(rows, lay, B, N, dt, f_max, mask, static_cast<const float*>(wrench), c, static_cast<float*>(lambda),
                       grad);
}

}  // extern "C"

#ifdef HMPC_CERTIFY_MAIN
// usage: certify_tsan <file> — the file holds int B, int N, then B update_data_t rows and B x 12N double wrenches; certifies
// them (problem dt 0.04, f_max 500) and prints "ok <passes>"
int main(int argc, char** argv)
{
  if (argc < 2) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int hdr[2];
  if (fread(hdr, sizeof hdr, 1, f) != 1) return 2;
  const int B = hdr[0], N = hdr[1];
  std::vector<unsigned char> rows((size_t)B * 3016);
  std::vector<double> w((size_t)B * 12 * N), lam((size_t)B * 16 * N);
  std::vector<hmpc::CertOut> cert(B);
  if (fread(rows.data(), 1, rows.size(), f) != rows.size() || fread(w.data(), sizeof(double), w.size(), f) != w.size()) return 2;
  fclose(f);
  emul_certify(rows.data(), 1, B, N, 0.04f, 500.f, nullptr, 1, w.data(), cert.data(), lam.data(), nullptr);
  int pass = 0;
  for (int i = 0; i < B; i++) pass += cert[i].flags == hmpc::CERT_PASS;
  printf("ok %d\n", pass);
  return 0;
}
#endif
