// tests/host_emul/warm_start_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only): the warm-started solve with per-robot
// shifts (KernelArgs::ws_shifts, what hmpc_solve_device_warm / hmpc_solve_batch_warm pass) on the host.
//
// Built by tests/test_warm_start_calls.py exactly like kernel_source_on_host.cpp, whose CTA emulation, kernel variants and
// class configuration it reuses by inclusion (same translation unit); everything that library exports stays available.
#include "kernel_source_on_host.cpp"

extern "C" {

/* The device-resident path of hmpc_capi.cu (enqueue_solve: class 0 over every robot, classifying on the way, then class 1
 * and class 2 through the escalation lists) on B <= 1024 packed records, warm-started from `ws` [B][WS_STATE_INTS]
 * (written back) with `shift` for every robot, or `shifts` [B] per robot when not NULL.  ws == NULL: a cold solve.
 * Outputs: wrench [B][12N] floats, status [B], launched[3] = instances each class kept (NULL to skip). */
int emul_solve_warm(const unsigned char* records, int B, int N, float dt, float f_max, int max_iter, int* ws, int shift,
                    const int* shifts, float* wrench, int* status, int* launched)
{
  if (B < 1 || B > 1024 || !records) return 1;
  ClassCfg cls[3];
  const int ncls = build_classes(N, cls);
  std::vector<int> block(8 + 3 * (size_t)B, 0);
  int* counts = block.data();  // [4] list lengths, [4] the next call's (cleared by the class-0 launch)
  int* lists = counts + 8;
  counts[0] = B;
  for (int i = 0; i < ncls; i++) {
    if (launched) launched[i] = counts[i];
    if (counts[i] == 0) continue;
    hmpc::KernelArgs ka{};
    ka.records = records;
    ka.rec_stride = hmpc::record_stride(N);
    ka.batch = B;
    ka.horizon = N;
    ka.dt = dt;
    ka.f_max = f_max;
    ka.max_iter = max_iter;
    ka.tol_kkt = 1e-9;   // hmpc_capi.cu's defaults
    ka.tol_dep = 1e-11;
    ka.kappa_max = 1.5e5;
    ka.block_min = 2;
    ka.block_rounds = 4;
    ka.wrench = wrench;
    ka.status = status;
    ka.warm_start = ws ? 1 : 0;
    ka.ws_state = ws;
    ka.ws_shift = shift;
    ka.ws_shifts = shifts;
    ka.list = i == 0 ? nullptr : lists + (size_t)i * B;
    ka.split_nb = i == 0 ? cls[0].nb_cap : -1;
    ka.counts_next = i == 0 ? counts + 4 : nullptr;
    ka.counts = counts;
    ka.cls = i;
    ka.esc_list = i + 1 < ncls ? lists + (size_t)(i + 1) * B : nullptr;
    ka.nb_cap = cls[i].nb_cap;
    ka.qmax = cls[i].qmax;
    ka.tcap = cls[i].tcap;
    ka.L = cls[i].L;
    launch_variant(cls[i].variant, ka);
    if (i == 0 && launched) launched[0] = B - counts[1];  // instances class 0 kept
  }
  return 0;
}

}  // extern "C"
