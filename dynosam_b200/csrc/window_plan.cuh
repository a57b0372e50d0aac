// window_plan.cuh -- the symbolic decisions of finalize (api.cu) that need no device: the order of a factor block's
// factors, and the window plan of its landmark elimination (kernels_window.cu).  Plain host functions of host arrays,
// so that tests/capi/window_plan_host.cu can run them on a machine without a GPU.
#pragma once
#include <parallel/algorithm>
#include <omp.h>
#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>
#include "internal.cuh"

namespace dynoba {

// std::vector without the serial value-initialisation pass (the elements are written in parallel right after resize)
template <class T> struct NoInitAlloc : std::allocator<T> {
  template <class U> struct rebind { using other = NoInitAlloc<U>; };
  template <class U, class... A> void construct(U* p, A&&... a) {
    if constexpr (sizeof...(A) == 0) ::new ((void*)p) U; else ::new ((void*)p) U(std::forward<A>(a)...);
  }
};

// Factor order of a block: by (group rank, pose position), i.e. by key[i] = frank[i] << 32 | position of the first pose
// slot.  perm [n] holds the identity on entry and maps sorted position -> factor on return.  ngroups: landmark groups of
// the whole problem (a bound on the runs of distinct ranks).  fast = false skips the run sort (tests compare the two).
inline void order_block_factors(int32_t* perm, const int32_t* frank, const int64_t* key, int64_t n, size_t ngroups, bool fast = true) {
  int unsorted = 0;
#pragma omp parallel for schedule(static) reduction(|:unsorted)
  for (int64_t i = 1; i < n; i++) unsorted |= key[i-1] > key[i];
  if (!unsorted) return;
  // Fast path: the caller lists each landmark's factors contiguously with ascending poses (how DynOSAM's
  // formulations add them) and only the ORDER OF THE LANDMARKS differs from ours -- then sorting the runs (one per
  // landmark) replaces sorting the factors.  Anything else falls back to the general stable sort.
  std::vector<int64_t> run0;                                 // first factor of each run of equal group rank
  {
    const int nseg = std::max(1, std::min<int>(omp_get_max_threads(), (int)(n/65536) + 1));
    std::vector<std::vector<int64_t>> seg(nseg);
#pragma omp parallel for schedule(static, 1)
    for (int t = 0; t < nseg; t++) {
      const int64_t s0 = n*t/nseg, s1 = n*(t + 1)/nseg;
      for (int64_t i = s0; i < s1; i++) if (i == 0 || frank[i] != frank[i-1]) seg[t].push_back(i);
    }
    for (auto& v : seg) run0.insert(run0.end(), v.begin(), v.end());
  }
  const int64_t nrun = (int64_t)run0.size();
  int bad = 0;                                               // a rank in two runs, or poses not ascending inside a run
  std::vector<int64_t> order(nrun);
  if (fast && nrun <= (int64_t)ngroups) {
#pragma omp parallel for schedule(static) reduction(|:bad)
    for (int64_t r = 0; r < nrun; r++) {
      order[r] = r;
      const int64_t e = r + 1 < nrun ? run0[r + 1] : n;
      for (int64_t i = run0[r] + 1; i < e; i++) bad |= key[i-1] > key[i];
    }
    if (!bad) {
      __gnu_parallel::sort(order.begin(), order.end(), [&](int64_t a, int64_t c) { return frank[run0[a]] < frank[run0[c]]; });
#pragma omp parallel for schedule(static) reduction(|:bad)
      for (int64_t r = 1; r < nrun; r++) bad |= frank[run0[order[r-1]]] == frank[run0[order[r]]];
    }
  } else bad = 1;
  if (!bad) {
    std::vector<int64_t> dst(nrun + 1, 0);
    for (int64_t r = 0; r < nrun; r++) { const int64_t a = order[r]; dst[r + 1] = dst[r] + ((a + 1 < nrun ? run0[a + 1] : n) - run0[a]); }
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < nrun; r++) {
      const int64_t a = order[r], len = dst[r + 1] - dst[r];
      for (int64_t k = 0; k < len; k++) perm[dst[r] + k] = (int32_t)(run0[a] + k);
    }
  } else {
    __gnu_parallel::stable_sort(perm, perm + n, [&](int a, int c) { return key[a] < key[c]; });
  }
}

// The window plan of one factor block of a 3-dof landmark type: what kernels_window.cu's DevWindows holds, on the host.
struct WindowPlan {
  std::vector<unsigned char> gwin;                              // per group: 1 window path, 2 simple kernel, 0 general (gl < 0)
  std::vector<unsigned char, NoInitAlloc<unsigned char>> lvar;  // [NPs][stride] window slot of each pose slot (window factors only)
  std::vector<int4> jobs, batches;                              // as DevWindows
  std::vector<int32_t> chunk_batch, cvars;
  int64_t win_ctas = 0, win_flushed = 0;                        // accumulate-kernel CTAs and 6x6 blocks it flushes, per damped solve
  bool all_window = false;                                      // no group left for the per-landmark atomics kernel
};

// NPs: pose slots of the factor type (1 or 2), stride: the block's SoA stride, NP: pose-like variables of the problem,
// prow[k]: solver position of pose slot k of every sorted factor (rows of the block's index image), gp [ng + 1] / gl [ng]:
// first factor and landmark of each group in the symbolic order (gl < 0: a general group), cap: most variables of a chunk
// (a wider landmark gets a chunk of its own), nseg: host segments.
inline WindowPlan plan_windows(int NPs, int stride, int64_t NP, const int32_t* const prow[2], const int32_t* gp, const int32_t* gl,
                               int ng, int cap, int nseg) {
  WindowPlan w;
  std::vector<unsigned char>& gwin = w.gwin; gwin.assign(ng, 0);
  auto& lvar = w.lvar; lvar.resize((size_t)NPs*stride);        // only read for window-path factors
  // NP = 2: a variable keeps its window slot over the consecutive chunks that contain it, and the accumulate kernel
  // walks runs of chunks.  NP = 1 chunks (~1000 landmarks each) are runs of their own, slots in position order.
  const bool slide = NPs == 2;
  // greedy chunking, independently inside parallel segments of the group list (a chunk never crosses a segment)
  // per chunk: first group, slots spanned (highest occupied slot + 1), slot -> position row, first batch (+ end)
  struct SegOut { std::vector<int32_t> g0, nslot, cv, b0; std::vector<int4> bat; int64_t flushed = 0; };
  std::vector<SegOut> seg(nseg);
#pragma omp parallel for schedule(static, 1)
  for (int t = 0; t < nseg; t++) {
    const int ga = (int)((int64_t)ng*t/nseg), gb_ = (int)((int64_t)ng*(t + 1)/nseg);
    std::vector<int32_t> stamp(NP, -1), gstamp(NP, -1), inchunk(NP, -1), cur;   // indexed by solver position
    std::vector<int32_t> wslot(NP, -1), occ(WIN_NLOC_MAX, -1);                 // window slot of a position, occupant of a slot
    int cur_g0 = ga, chunk_id = 0; SegOut& out = seg[t];
    auto close_chunk = [&](int g_end) {
      std::vector<int32_t> sorted = cur; std::sort(sorted.begin(), sorted.end());
      std::vector<int32_t> row(WIN_NLOC_MAX, -1);
      if (slide) {     // variables that stay keep their slot; entering ones take the lowest free slots
        for (int32_t p_ : sorted) stamp[p_] = -2;
        for (int s_ = 0; s_ < WIN_NLOC_MAX; s_++) if (occ[s_] >= 0 && stamp[occ[s_]] != -2) occ[s_] = -1;
        for (int32_t p_ : sorted) if (wslot[p_] >= 0 && occ[wslot[p_]] == p_) stamp[p_] = wslot[p_];
        int fs = 0;
        for (int32_t p_ : sorted) if (stamp[p_] == -2) { while (occ[fs] >= 0) fs++; occ[fs] = p_; wslot[p_] = fs; stamp[p_] = fs; }
        row = occ;
      } else {
        for (size_t i = 0; i < sorted.size(); i++) { stamp[sorted[i]] = (int32_t)i; row[i] = sorted[i]; }   // position -> local index
      }
      for (int g = cur_g0; g < g_end; g++) if (gwin[g] == 1)
        for (int s_ = gp[g]; s_ < gp[g+1]; s_++) for (int k = 0; k < NPs; k++)
          lvar[(size_t)k*stride + s_] = (unsigned char)stamp[prow[k][s_]];
      for (size_t i = 0; i < sorted.size(); i++) stamp[sorted[i]] = -1;
      int ext = 0; for (int s_ = 0; s_ < WIN_NLOC_MAX; s_++) if (row[s_] >= 0) ext = s_ + 1;
      out.g0.push_back(cur_g0); out.nslot.push_back(ext);
      out.cv.insert(out.cv.end(), row.begin(), row.end());
      // batches of the chunk: runs of window-path landmarks (other groups end a run), bounded in landmarks and slots
      out.b0.push_back((int32_t)out.bat.size());
      int rg0 = -1, rslots = 0;
      auto close_batch = [&](int ge) { if (rg0 >= 0) out.bat.push_back(make_int4(rg0, ge, gp[rg0], gp[ge])); rg0 = -1; rslots = 0; };
      for (int g = cur_g0; g < g_end; g++) {
        if (gwin[g] != 1) { close_batch(g); continue; }
        const int ns_ = (gp[g+1] - gp[g])*NPs;
        if (rg0 >= 0 && (rslots + ns_ > WIN_BATCH_SLOTS || g - rg0 >= WIN_BATCH_LMK)) close_batch(g);
        if (rg0 < 0) rg0 = g;
        rslots += ns_;
      }
      close_batch(g_end);
      chunk_id++; cur.clear(); cur_g0 = g_end;
    };
    for (int g = ga; g < gb_; g++) {
      if (gl[g] < 0) continue;
      const int T = gp[g+1] - gp[g];
      bool dup = false; int fresh = 0;
      if (T > WIN_TMAX) { gwin[g] = 2; continue; }
      for (int s_ = gp[g]; s_ < gp[g+1] && !dup; s_++) for (int k = 0; k < NPs; k++) {
        const int p_ = prow[k][s_];
        if (gstamp[p_] == g) { dup = true; break; }
        gstamp[p_] = g;
        if (inchunk[p_] != chunk_id) fresh++;
      }
      if (dup) { gwin[g] = 2; continue; }
      if (!cur.empty() && (int)cur.size() + fresh > cap) {      // a landmark wider than cap gets a chunk of its own
        close_chunk(g);
      }
      for (int s_ = gp[g]; s_ < gp[g+1]; s_++) for (int k = 0; k < NPs; k++) {
        const int p_ = prow[k][s_];
        if (inchunk[p_] != chunk_id) { inchunk[p_] = chunk_id; cur.push_back(p_); }
      }
      gwin[g] = 1;
    }
    close_chunk(gb_);
    out.b0.push_back((int32_t)out.bat.size());
  }
  // runs: a segment's chunks that have batches, run_len at a time (never across a segment: the slots restart there)
  auto has_batches = [&](const SegOut& o, size_t c) { return o.b0[c + 1] > o.b0[c]; };
  size_t nch = 0; for (int t = 0; t < nseg; t++) for (size_t c = 0; c + 1 < seg[t].b0.size(); c++) nch += has_batches(seg[t], c);
  const int run_len = slide ? std::max<int>(WIN_RUN_MIN_CHUNKS, (int)((nch + WIN_RUNS - 1)/WIN_RUNS)) : 1;
  // census: the blocks the accumulate kernel flushes per solve, by its rule (a slot pair that a landmark's clique
  // touched, when either slot changes variable and at the run's end)
#pragma omp parallel for schedule(static, 1)
  for (int t = 0; t < nseg; t++) {
    SegOut& o = seg[t];
    uint64_t tch[WIN_NLOC_MAX] = {};      // tch[a] bit b: slot pair (a, b) touched since its last flush
    auto flush = [&](uint64_t E) {        // E: slots that change variable
      for (int a_ = 0; a_ < WIN_NLOC_MAX; a_++) {
        const uint64_t low = tch[a_] & ((2ull << a_) - 1);
        o.flushed += __builtin_popcountll((E >> a_) & 1 ? low : low & E);
      }
      for (int a_ = 0; a_ < WIN_NLOC_MAX; a_++) tch[a_] = (E >> a_) & 1 ? 0 : tch[a_] & ~E;
    };
    int in_run = 0; int prev = -1;
    for (size_t c = 0; c + 1 < o.b0.size(); c++) {
      if (!has_batches(o, c)) continue;
      uint64_t E = 0;
      if (in_run == run_len) { E = ~0ull; in_run = 0; }
      else if (prev >= 0) for (int s_ = 0; s_ < WIN_NLOC_MAX; s_++) if (o.cv[(size_t)prev*WIN_NLOC_MAX + s_] != o.cv[c*WIN_NLOC_MAX + s_]) E |= 1ull << s_;
      flush(E);
      in_run++; prev = (int)c;
      const int ge = c + 1 < o.g0.size() ? o.g0[c + 1] : (int)((int64_t)ng*(t + 1)/nseg);
      for (int g = o.g0[c]; g < ge; g++) if (gwin[g] == 1) {
        uint64_t m = 0;
        for (int s_ = gp[g]; s_ < gp[g+1]; s_++) for (int k = 0; k < NPs; k++) m |= 1ull << lvar[(size_t)k*stride + s_];
        for (uint64_t r_ = m; r_; r_ &= r_ - 1) tch[__builtin_ctzll(r_)] |= m;
      }
    }
    flush(~0ull);
  }
  for (int t = 0; t < nseg; t++) {
    const SegOut& o = seg[t];
    w.win_flushed += o.flushed;
    int r0 = -1, in_run = 0, ext = 0;
    auto close_run = [&]() {
      if (r0 < 0) return;
      const int nst = (win_ntiles(ext) + WIN_ACC_WARPS - 1)/WIN_ACC_WARPS;
      for (int st = 0; st < nst; st++) w.jobs.push_back(make_int4(r0, (int)w.chunk_batch.size(), st, ext));
      w.win_ctas += nst; r0 = -1; in_run = 0; ext = 0;
    };
    for (size_t c = 0; c + 1 < o.b0.size(); c++) {
      if (!has_batches(o, c)) continue;
      if (in_run == run_len) close_run();
      if (r0 < 0) r0 = (int)w.chunk_batch.size();
      w.chunk_batch.push_back((int32_t)w.batches.size());
      w.batches.insert(w.batches.end(), o.bat.begin() + o.b0[c], o.bat.begin() + o.b0[c + 1]);
      w.cvars.insert(w.cvars.end(), o.cv.begin() + c*WIN_NLOC_MAX, o.cv.begin() + (c + 1)*WIN_NLOC_MAX);
      ext = std::max(ext, o.nslot[c]); in_run++;
    }
    close_run();
  }
  w.chunk_batch.push_back((int32_t)w.batches.size());
  { size_t nw = 0; for (int g = 0; g < ng; g++) nw += gwin[g] == 1 || gl[g] < 0; w.all_window = nw == (size_t)ng; }
  return w;
}

}  // namespace dynoba
