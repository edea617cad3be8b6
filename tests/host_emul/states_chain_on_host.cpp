// tests/host_emul/states_chain_on_host.cpp — TEST INFRASTRUCTURE (CPU suite only): the chain that starts from robot states.
//
// Built as its own host library by tests/test_states_masked.py, with the same host-buildable device header and flags as
// kernel_source_on_host.cpp, which it includes whole: every emul_* entry point of that library is here too, plus
//   * emul_prepare_list: the preparation launch over an instance list (hmpc_prepare_kernel's `list` / `count`);
//   * emul_solve_states: the states chain of hmpc_solve_states_device_masked and of the in-place mode of the state calls.
// The preparation launch's arguments and grid come from the library's own hmpc_chain.h (prepare_args, prepare_grid).
#include "kernel_source_on_host.cpp"

namespace {
// hmpc_capi.cu's preparation launch (launch_prepare): every thread of its grid, one at a time
void run_prepare(const hmpc::PrepareArgs& pa)
{
  const unsigned NT = hmpc::PREPARE_THREADS;
  const int threads = hmpc::prepare_grid(pa.batch) * hmpc::PREPARE_THREADS;
  for (int t = 0; t < threads; t++) {
    blockDim = {NT, 1, 1};
    blockIdx = {(unsigned)t / NT, 0, 0};
    threadIdx = {(unsigned)t % NT, 0, 0};
    gridDim = {(unsigned)hmpc::prepare_grid(pa.batch), 1, 1};
    hmpc::hmpc_prepare_kernel(pa.states, pa.batch, pa.N, pa.dtMPC, pa.records, pa.rec_stride, pa.list, pa.count);
  }
}
}  // namespace

extern "C" {

/* the preparation launch of hmpc_prepare_device (every robot), or over `list` [*count] (the states chain of a masked call)
 * when list is not NULL */
void emul_prepare_list(const unsigned char* states, int batch, int N, double dtMPC, unsigned char* records, const int* list,
                       const int* count)
{
  hmpc::SolveIO io;
  io.states = states;
  io.records = records;
  io.batch = batch;
  io.dt_mpc = dtMPC;
  hmpc::ChainLists lists;
  lists.counts = const_cast<int*>(count);
  lists.list[0] = const_cast<int*>(list);
  run_prepare(hmpc::prepare_args(N, io, lists));
}

/* The states chain on B <= 1024 robots: [the selection kernel over `mask`] -> the preparation of hmpc_state_t `states`
 * (dtMPC) over class 0's list, or every robot without a mask, into `records` [B][stride] -> class 0 over the same robots ->
 * class 1 -> class 2 -> [refinement].  The classes run as emul_solve's device-resident chain over `records` with the same
 * mask: its selection kernel builds the list again, the same list, in a slot of its own.  The other arguments as in
 * emul_solve (no assembly dump).  Returns what emul_solve returns, or 1 for a bad argument. */
int emul_solve_states(const unsigned char* states, double dtMPC, unsigned char* records, int B, int N, int refine,
                      const unsigned char* mask, int* ws, int warm, int shift, const int* shifts, float* wrench, double* wrench64,
                      int* status, float* tau, int* launched)
{
  if (B < 1 || B > 1024 || !states || !records) return 1;
  std::vector<int> mem(hmpc::ClassSlot::cls_slot_ints(B), 0);
  const hmpc::ClassSlot slot{mem.data(), B, 0};
  const hmpc::ChainLists lists = hmpc::slot_lists(slot, mask != nullptr, refine != 0);
  if (mask) run_select(mask, B, slot.list0(), slot.counts());
  hmpc::SolveIO io;
  io.states = states;
  io.dt_mpc = dtMPC;
  io.records = records;
  io.batch = B;
  run_prepare(hmpc::prepare_args(N, io, lists));
  return emul_solve(records, nullptr, B, N, 0, refine, mask, ws, warm, shift, shifts, wrench, wrench64, status, tau, launched,
                    nullptr, nullptr, nullptr, nullptr, nullptr);
}

}  // extern "C"
