// window_plan_host.cu -- the factor order and the window plan of dynosam_b200/csrc/window_plan.cuh compiled for the
// host, so that tests/test_window_plan.py can run them on a machine without a GPU.
#include "window_plan.cuh"

using namespace dynoba;

static WindowPlan last;     // the plan of the latest host_plan_windows call, read back by host_plan_copy

extern "C" {
// plans a block and returns the sizes of its arrays and its counters: [gwin, lvar, jobs, batches, chunk_batch, cvars,
// win_ctas, win_flushed, all_window] (jobs and batches in int4s)
void host_plan_windows(int NPs, int stride, int64_t NP, const int32_t* prow0, const int32_t* prow1, const int32_t* gp,
                       const int32_t* gl, int ng, int cap, int nseg, int64_t* out) {
  const int32_t* prow[2] = {prow0, prow1};
  last = plan_windows(NPs, stride, NP, prow, gp, gl, ng, cap, nseg);
  const int64_t v[9] = {(int64_t)last.gwin.size(), (int64_t)last.lvar.size(), (int64_t)last.jobs.size(), (int64_t)last.batches.size(),
                        (int64_t)last.chunk_batch.size(), (int64_t)last.cvars.size(), last.win_ctas, last.win_flushed, last.all_window};
  for (int i = 0; i < 9; i++) out[i] = v[i];
}
void host_plan_copy(unsigned char* gwin, unsigned char* lvar, int4* jobs, int4* batches, int32_t* chunk_batch, int32_t* cvars) {
  std::copy(last.gwin.begin(), last.gwin.end(), gwin);
  std::copy(last.lvar.begin(), last.lvar.end(), lvar);
  std::copy(last.jobs.begin(), last.jobs.end(), jobs);
  std::copy(last.batches.begin(), last.batches.end(), batches);
  std::copy(last.chunk_batch.begin(), last.chunk_batch.end(), chunk_batch);
  std::copy(last.cvars.begin(), last.cvars.end(), cvars);
}
// perm: sorted position -> factor of a block with group ranks frank and keys frank << 32 | pose position
void host_order_block_factors(int32_t* perm, const int32_t* frank, const int64_t* key, int64_t n, int64_t ngroups, int fast) {
  for (int64_t i = 0; i < n; i++) perm[i] = (int32_t)i;
  order_block_factors(perm, frank, key, n, (size_t)ngroups, fast != 0);
}
}
