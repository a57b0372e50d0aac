// kernels_window.cu -- K4: landmark Schur scatter WITHOUT atomics in the inner loop, as a two-kernel pipeline.
//
//   K4a schur_stage_kernel   one warp (or half-warp) per landmark: V = sum B^T B + lambda I, M = chol(V)^-1, and for every clique
//                            variable of every factor one 336-byte SLOT
//                                Wt = (A^T B M^T)^T (3x6),  A (3x6, whitened Jacobian tile),  rb = b - B V^-1 g_l,  meta
//                            written once to an HBM scratch array that is laid out in factor order, so the slots of a
//                            run of landmarks are ONE contiguous byte range.
//   K4b schur_accum_kernel   the landmarks of a factor block are cut (on the host, DevWindows) into chunks whose cliques
//                            live in a window of at most NLOC pose-like variables, and the chunks into RUNS of
//                            consecutive chunks.  A CTA of 512 threads owns (a stripe of) the lower-triangular 6x6 blocks
//                            of the window's slot pairs, ONE BLOCK PER THREAD (a warp = an 8x4 tile of blocks), in
//                            registers (output-stationary), and streams the run's slots, chunk after chunk, through shared
//                            memory with bulk asynchronous copies (cp.async.bulk + mbarrier, double-buffered); every thread adds
//                                S_ab += [same factor] A_a^T A_b - What_a What_b^T
//                            for the landmarks whose clique contains both of its variables (What_a What_b^T =
//                            W_a V^-1 W_b^T).  g_S is accumulated by the diagonal threads in shared memory.  A variable
//                            keeps its window slot while consecutive chunks contain it (NP = 2: a dynamic landmark's
//                            chunk is ~28 landmarks of one object born at one frame, the next chunk is the same object a
//                            frame later), so a block is flushed into the tiled band storage only when one of its two
//                            slots changes variable, and at the run's end.
// Arithmetic is the same as kernels_schur.cu (GTSAM's landmark elimination, SURVEY.md 8a a11).
#include "internal.cuh"

namespace dynoba {

// acc[e] with a run-time index (rare slow path of the flush): a select chain keeps the accumulators in registers
__device__ __forceinline__ double acc_at(const double (&acc)[36], int e) {
  double v = 0.0;
#pragma unroll
  for (int k = 0; k < 36; k++) if (k == e) v = acc[k];
  return v;
}

constexpr int STG_WARPS = 2;          // K4a: warps per CTA (NP = 2: 43 KB of slot images, five CTAs per SM)
constexpr int ACC_THREADS = WIN_ACC_WARPS*32;
constexpr int WSLOT = WIN_SLOT_DOUBLES;   // 42 doubles = 21 x 16 B: odd stride => conflict-free LDS.128 across slots
// K4a: a lane's NP slots in the shared-memory image, in 16-byte units, padded to an odd count so that the lanes' STS.128
// are conflict-free (NP = 2: 43 instead of 42)
template <int NP> constexpr int STG_LANE16 = NP*(WSLOT/2) | 1;

// slot meta word: bits 0-7 local variable (255 = not on the window path), 8-15 factor within the landmark, 16-47 group
__device__ __forceinline__ double pack_meta(unsigned lvar, unsigned fac, unsigned g) {
  return __longlong_as_double((long long)(((unsigned long long)g << 16) | ((unsigned long long)fac << 8) | lvar));
}

// One landmark staged by a group of W = 32 or 16 lanes (`hl` = lane within the group, `mask` = the group's lanes): lane
// `hl` owns factor `hl` of the landmark.  The lanes build the landmark's slots in `img` (W lanes of STG_LANE16<NP>
// 16-byte units), and the group then writes them as one contiguous range, 16 bytes per lane and store: a lane storing
// its own 336-byte slot would touch 32 half-filled sectors per warp store.
template <int NP, int PCOL0, int LCOL, int W>
__device__ __forceinline__ void stage_landmark(const DevBlock& blk, const DevWindows& Wn, double lambda, int* __restrict__ fail,
                                               int g, int hl, unsigned mask, double* __restrict__ img) {
  constexpr int JC = NP*6 + 3;
  auto gsum = [&](double x) {
#pragma unroll
    for (int o = W/2; o > 0; o >>= 1) x += __shfl_xor_sync(mask, x, o);
    return x;
  };
  const int f0 = blk.grp_ptr[g], T = blk.grp_ptr[g + 1] - f0;
  double* slots = Wn.slots;
  if (Wn.grp_win[g] != 1) {       // not ours: leave the slots marked invalid (they sit inside contiguous copy ranges)
    for (int i = hl; i < T*NP; i += W) slots[((size_t)f0*NP + i)*WSLOT + 39] = pack_meta(255u, 0u, (unsigned)g);
    return;
  }
  double V[9], gl[3], Bm[9], bb[3];
#pragma unroll
  for (int k = 0; k < 9; k++) V[k] = 0.0;
  gl[0] = gl[1] = gl[2] = 0.0;
  const bool have = hl < T;            // T <= W: guaranteed by the caller (T <= WIN_TMAX <= 32 by the host)
  const int f = f0 + hl;
  double Aall[NP*18];                  // every load is issued up front: one memory latency per landmark
  if (have) {
#pragma unroll
    for (int r = 0; r < 3; r++) {
      bb[r] = blk.b[(size_t)r*blk.stride + f];
#pragma unroll
      for (int c = 0; c < 3; c++) Bm[r*3 + c] = blk.J[(size_t)(r*JC + LCOL + c)*blk.stride + f];
    }
#pragma unroll
    for (int s = 0; s < NP; s++)
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 6; c++) Aall[s*18 + r*6 + c] = blk.J[(size_t)(r*JC + PCOL0 + 6*s + c)*blk.stride + f];
#pragma unroll
    for (int c1 = 0; c1 < 3; c1++) {
#pragma unroll
      for (int r = 0; r < 3; r++) gl[c1] += Bm[r*3 + c1]*bb[r];
#pragma unroll
      for (int c2 = 0; c2 <= c1; c2++)
#pragma unroll
        for (int r = 0; r < 3; r++) V[c1*3 + c2] += Bm[r*3 + c1]*Bm[r*3 + c2];
    }
  }
#pragma unroll
  for (int c1 = 0; c1 < 3; c1++) {
    gl[c1] = gsum(gl[c1]);
#pragma unroll
    for (int c2 = 0; c2 <= c1; c2++) V[c1*3 + c2] = gsum(V[c1*3 + c2]);
    V[c1*3 + c1] += lambda;
  }
  // M = chol(V)^-1 (lower)
  bool ok = V[0] > 0;
  const double l00 = sqrt(V[0]), l10 = V[3]/l00, l20 = V[6]/l00;
  const double d1 = V[4] - l10*l10; ok = ok && d1 > 0;
  const double l11 = sqrt(d1), l21 = (V[7] - l20*l10)/l11;
  const double d2 = V[8] - l20*l20 - l21*l21; ok = ok && d2 > 0;
  const double l22 = sqrt(d2);
  if (!ok) {                           // landmark skipped: the trial step is rejected anyway
    if (hl == 0) atomicOr(fail, 1);
    for (int i = hl; i < T*NP; i += W) slots[((size_t)f0*NP + i)*WSLOT + 39] = pack_meta(255u, 0u, (unsigned)g);
    return;
  }
  if (have) {
    const double m00 = 1.0/l00, m11 = 1.0/l11, m22 = 1.0/l22;
    const double m10 = -l10*m00*m11, m21 = -l21*m11*m22, m20 = -(l20*m00 + l21*m10)*m22;
    const double y0 = m00*gl[0], y1 = m10*gl[0] + m11*gl[1], y2 = m20*gl[0] + m21*gl[1] + m22*gl[2];   // y = M g_l
    double Bh[9];                      // Bh = B M^T
#pragma unroll
    for (int r = 0; r < 3; r++) {
      Bh[r*3 + 0] = Bm[r*3]*m00;
      Bh[r*3 + 1] = Bm[r*3]*m10 + Bm[r*3 + 1]*m11;
      Bh[r*3 + 2] = Bm[r*3]*m20 + Bm[r*3 + 1]*m21 + Bm[r*3 + 2]*m22;
    }
    double rb[3];                      // rb = b - Bh y
#pragma unroll
    for (int r = 0; r < 3; r++) rb[r] = bb[r] - (Bh[r*3]*y0 + Bh[r*3 + 1]*y1 + Bh[r*3 + 2]*y2);
#pragma unroll
    for (int s = 0; s < NP; s++) {
      double2* o = reinterpret_cast<double2*>(img) + hl*STG_LANE16<NP> + s*(WSLOT/2);
      const double* A = Aall + s*18;
      double w[18];                    // w[k*6 + c] = What[c][k] = sum_r A[r][c] Bh[r][k]
#pragma unroll
      for (int k = 0; k < 3; k++)
#pragma unroll
        for (int c = 0; c < 6; c++) w[k*6 + c] = A[c]*Bh[k] + A[6 + c]*Bh[3 + k] + A[12 + c]*Bh[6 + k];
#pragma unroll
      for (int i = 0; i < 9; i++) o[i] = make_double2(w[2*i], w[2*i + 1]);
#pragma unroll
      for (int i = 0; i < 9; i++) o[9 + i] = make_double2(A[2*i], A[2*i + 1]);
      o[18] = make_double2(rb[0], rb[1]);
      o[19] = make_double2(rb[2], pack_meta((unsigned)Wn.lvar[(size_t)s*blk.stride + f], (unsigned)hl, (unsigned)g));
      o[20] = make_double2(0.0, 0.0);  // the pad too: every sector of the range is written whole
    }
  }
  __syncwarp(mask);
  const double2* src = reinterpret_cast<const double2*>(img);
  double2* dst = reinterpret_cast<double2*>(slots + (size_t)f0*NP*WSLOT);
  constexpr int PAD = STG_LANE16<NP> - NP*(WSLOT/2);   // 16-byte units after each lane's slots in the image
  for (int i = hl; i < T*NP*(WSLOT/2); i += W) dst[i] = src[i + PAD*(i/(NP*(WSLOT/2)))];
  __syncwarp(mask);                    // the image is read before the group's next landmark overwrites it
}

// A warp takes two consecutive landmarks: side by side on its two half-warps when both have at most 16 factors (the
// common case: tracks average 8.5 / 11.4 observations), one after the other on all 32 lanes otherwise.
template <int NP, int PCOL0, int LCOL>
__global__ void __launch_bounds__(STG_WARPS*32, NP == 2 ? 5 : 6)   // the CTAs per SM the slot images / registers allow
schur_stage_kernel(DevBlock blk, DevWindows Wn, double lambda, int* __restrict__ fail) {
  __shared__ __align__(16) double img[STG_WARPS][32*2*STG_LANE16<NP>];   // a warp's slot images: 32 lanes' slots
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g0 = 2*(blockIdx.x*STG_WARPS + warp);
  if (g0 >= blk.n_groups) return;
  const bool two = g0 + 1 < blk.n_groups;
  const int T0 = blk.grp_ptr[g0 + 1] - blk.grp_ptr[g0], T1 = two ? blk.grp_ptr[g0 + 2] - blk.grp_ptr[g0 + 1] : 0;
  if (two && T0 <= 16 && T1 <= 16) {
    const int half = lane >> 4;
    stage_landmark<NP, PCOL0, LCOL, 16>(blk, Wn, lambda, fail, g0 + half, lane & 15, half ? 0xffff0000u : 0x0000ffffu,
                                        img[warp] + half*16*2*STG_LANE16<NP>);
  } else {
#pragma unroll 1
    for (int k = 0; k < (two ? 2 : 1); k++)
      stage_landmark<NP, PCOL0, LCOL, 32>(blk, Wn, lambda, fail, g0 + k, lane, 0xffffffffu, img[warp]);
  }
}

// ---- mbarrier / bulk-copy helpers (sm_90+ PTX)
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}

template <int NP>
__global__ void __launch_bounds__(ACC_THREADS, 1)
schur_accum_kernel(DevWindows Wn, DevBand B) {
  extern __shared__ __align__(128) unsigned char asm_[];
  double* buf = reinterpret_cast<double*>(asm_);                                        // [2][WIN_BATCH_SLOTS*WSLOT]
  double* gs = buf + 2*WIN_BATCH_SLOTS*WSLOT;                                            // [WIN_NLOC_MAX*6]
  short* map = reinterpret_cast<short*>(gs + WIN_NLOC_MAX*6);                            // [2][WIN_BATCH_LMK][WIN_NLOC_MAX]
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(map + 2*WIN_BATCH_LMK*WIN_NLOC_MAX);   // [2]
  const int tid = threadIdx.x;
  const int4 job = Wn.jobs[blockIdx.x];                 // (first chunk, end chunk, stripe, window slots)
  const int nslot = job.w;
  // my block (slots a >= b): warp <-> 8x4 tile of the window's lower triangle, the stripes of a run split the tiles evenly
  const int ntile = win_ntiles(nslot);
  const int nst = (ntile + WIN_ACC_WARPS - 1)/WIN_ACC_WARPS;
  const int per = (ntile + nst - 1)/nst;
  int a = 0, b = 0; bool active = false;
  {
    const int warp = tid >> 5, lane = tid & 31;
    int t = job.z*per + warp;
    if (warp < per && t < ntile) {
      int tr = 0;
      for (;; tr++) { const int rmax = (8*tr + 7 < nslot - 1) ? 8*tr + 7 : nslot - 1; const int n = rmax/4 + 1; if (t < n) break; t -= n; }
      a = 8*tr + (lane >> 2); b = 4*t + (lane & 3);
      active = a < nslot && b <= a;
    }
  }
  const bool diag = active && a == b;
  double acc[36];
#pragma unroll
  for (int i = 0; i < 36; i++) acc[i] = 0.0;
  bool touched = false;
  for (int i = tid; i < WIN_NLOC_MAX*6; i += ACC_THREADS) gs[i] = 0.0;
  if (tid == 0) {
    mbar_init(bar, 1); mbar_init(bar + 1, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int4* batches = Wn.batches;       // (first group, end group, first factor, end factor)
  const int b0 = Wn.chunk_batch[job.x], b1 = Wn.chunk_batch[job.y];   // the run's batches, chunk after chunk
  if (tid == 0) {
    const int4 bt = batches[b0];
    const unsigned bytes = (unsigned)((bt.w - bt.z)*NP*WSLOT*8);
    mbar_expect_tx(bar, bytes);
    bulk_g2s(buf, Wn.slots + (size_t)bt.z*NP*WSLOT, bytes, bar);
  }
  int4 bt = batches[b0];
  int chunk = job.x - 1, cend = b0;       // batches of `chunk` end at cend
  int pa = -1, pb = -1;                   // solver positions of the variables in slots a, b during `chunk`
  for (int bi = b0;; bi++) {
    if (bi == cend) {
      // chunk boundary (and the run's end): a block whose slot changes variable goes to S, and its slot pair starts over
      int na = -1, nb = -1;
      if (bi < b1) {
        chunk++; cend = Wn.chunk_batch[chunk + 1];
        if (active) { na = Wn.cvars[(size_t)chunk*WIN_NLOC_MAX + a]; nb = Wn.cvars[(size_t)chunk*WIN_NLOC_MAX + b]; }
      }
      if (touched && (na != pa || nb != pb)) {
        // block (pa, pb) of S, lower triangle: slots are not in position order, so a block with pa < pb goes in transposed
        const bool tr = pa < pb;
        const int pi = tr ? pb : pa, pj = tr ? pa : pb;
        const BandBlockRef cref = band_block_ref(B, pi*6, pj*6);   // the block's storage, resolved once for its 36 entries
        if (cref.fast) {
          // inside one band chain: tile coordinates of the block's corner, then 36 additions with compile-time offsets (a
          // block spans at most two tile rows and two tile columns)
          const int li0 = cref.rev ? cref.oi - (pj*6 + 5) : pi*6 - cref.oi, lj0 = cref.rev ? cref.oi - (pi*6 + 5) : pj*6 - cref.oj;
#pragma unroll
          for (int r = 0; r < 6; r++)
#pragma unroll
            for (int c = 0; c < 6; c++) {
              if (a == b && c > r) continue;
              // natural: (li, lj) = (li0 + r, lj0 + c); reversed chain: row and column swap and run backwards
              const int li = cref.rev ? li0 + (5 - c) : li0 + r, lj = cref.rev ? lj0 + (5 - r) : lj0 + c;
              red_add(cref.base + tile_elem(cref.tpc, lj >> 5, (li >> 5) - (lj >> 5), li & 31, lj & 31), tr ? acc[c*6 + r] : acc[r*6 + c]);
            }
        } else {
#pragma unroll 1
          for (int e = 0; e < 36; e++) {
            const int r = e/6, c = e - 6*r;
            if (a == b && c > r) continue;
            red_add(band_at_slow(B, pi*6 + r, pj*6 + c), acc_at(acc, tr ? c*6 + r : e));
          }
        }
        if (diag) {
#pragma unroll
          for (int c = 0; c < 6; c++) { red_add(rhs_at(B, pa*6 + c), gs[a*6 + c]); gs[a*6 + c] = 0.0; }
        }
#pragma unroll
        for (int i = 0; i < 36; i++) acc[i] = 0.0;
        touched = false;
      }
      pa = na; pb = nb;
      if (bi == b1) break;
    }
    const int cur = (bi - b0) & 1;
    const unsigned parity = (unsigned)(((bi - b0) >> 1) & 1);
    int4 btn = bt;
    if (bi + 1 < b1) btn = batches[bi + 1];
    const int nw = bt.y - bt.x, nslots = (bt.w - bt.z)*NP;
    short* mp = map + cur*WIN_BATCH_LMK*WIN_NLOC_MAX;
    {   // clear the rows of this batch's landmarks (two shorts per store)
      int* mp32 = reinterpret_cast<int*>(mp);
      for (int i = tid; i < nw*(WIN_NLOC_MAX/2); i += ACC_THREADS) mp32[i] = -1;
    }
    mbar_wait(bar + cur, parity);
    __syncthreads();                      // map cleared; every thread is done with the other buffer (batch bi-1)
    if (tid == 0 && bi + 1 < b1) {
      const unsigned bytes = (unsigned)((btn.w - btn.z)*NP*WSLOT*8);
      mbar_expect_tx(bar + (cur ^ 1), bytes);
      bulk_g2s(buf + (size_t)(cur ^ 1)*WIN_BATCH_SLOTS*WSLOT, Wn.slots + (size_t)btn.z*NP*WSLOT, bytes, bar + (cur ^ 1));
    }
    const double* bufc = buf + (size_t)cur*WIN_BATCH_SLOTS*WSLOT;
    for (int s = tid; s < nslots; s += ACC_THREADS) {
      const unsigned long long m = (unsigned long long)__double_as_longlong(bufc[s*WSLOT + 39]);
      const unsigned lv = (unsigned)(m & 0xffu);
      if (lv != 255u) mp[((int)(m >> 16) - bt.x)*WIN_NLOC_MAX + lv] = (short)s;
    }
    __syncthreads();
    if (active) {
#pragma unroll 1
      for (int w = 0; w < nw; w++) {
        const int sa = mp[w*WIN_NLOC_MAX + a], sb = mp[w*WIN_NLOC_MAX + b];
        if ((sa | sb) < 0) continue;
        touched = true;
        const double2* pa = reinterpret_cast<const double2*>(bufc + sa*WSLOT);
        const double2* pb = reinterpret_cast<const double2*>(bufc + sb*WSLOT);
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const double2 a0 = pa[3*k], a1 = pa[3*k + 1], a2 = pa[3*k + 2];
          const double2 c0 = pb[3*k], c1 = pb[3*k + 1], c2 = pb[3*k + 2];
          const double av[6] = {a0.x, a0.y, a1.x, a1.y, a2.x, a2.y};
          const double cv[6] = {c0.x, c0.y, c1.x, c1.y, c2.x, c2.y};
#pragma unroll
          for (int r = 0; r < 6; r++)
#pragma unroll
            for (int c = 0; c < 6; c++) acc[r*6 + c] -= av[r]*cv[c];
        }
        const unsigned long long ma = (unsigned long long)__double_as_longlong(bufc[sa*WSLOT + 39]);
        const unsigned long long mb = (unsigned long long)__double_as_longlong(bufc[sb*WSLOT + 39]);
        if (((ma ^ mb) & 0xff00ull) == 0) {      // same factor: the J^T J term
#pragma unroll
          for (int k = 0; k < 3; k++) {
            const double2 a0 = pa[9 + 3*k], a1 = pa[9 + 3*k + 1], a2 = pa[9 + 3*k + 2];
            const double2 c0 = pb[9 + 3*k], c1 = pb[9 + 3*k + 1], c2 = pb[9 + 3*k + 2];
            const double av[6] = {a0.x, a0.y, a1.x, a1.y, a2.x, a2.y};
            const double cv[6] = {c0.x, c0.y, c1.x, c1.y, c2.x, c2.y};
#pragma unroll
            for (int r = 0; r < 6; r++)
#pragma unroll
              for (int c = 0; c < 6; c++) acc[r*6 + c] += av[r]*cv[c];
          }
          if (diag) {                            // g_S: the diagonal thread is the only owner of its variable's rhs
            const double r0 = bufc[sa*WSLOT + 36], r1 = bufc[sa*WSLOT + 37], r2 = bufc[sa*WSLOT + 38];
            const double* A = bufc + sa*WSLOT + 18;
#pragma unroll
            for (int c = 0; c < 6; c++) gs[a*6 + c] += A[c]*r0 + A[6 + c]*r1 + A[12 + c]*r2;
          }
        }
      }
    }
    bt = btn;
  }
}

static size_t acc_smem() {
  return (size_t)2*WIN_BATCH_SLOTS*WSLOT*8 + (size_t)WIN_NLOC_MAX*6*8 + (size_t)2*WIN_BATCH_LMK*WIN_NLOC_MAX*2 + 16;
}

int launch_schur_window(const DevBlock& blk, const DevWindows& Wn, const DevBand& B, double lambda, int* fail, cudaStream_t s) {
  if (Wn.n_jobs == 0) return 0;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(schur_accum_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)acc_smem());
    cudaFuncSetAttribute(schur_accum_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)acc_smem());
    // the stage kernels' occupancy is set by their slot images: ask for the whole unified L1 as shared memory
    cudaFuncSetAttribute(schur_stage_kernel<1, 0, 6>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(schur_stage_kernel<2, 0, 12>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    attr = true;
  }
  const int sgrid = ((blk.n_groups + 1)/2 + STG_WARPS - 1)/STG_WARPS;
  switch (blk.type) {
    case F_POSE2POINT3: case F_STEREO3:
      schur_stage_kernel<1, 0, 6><<<sgrid, STG_WARPS*32, 0, s>>>(blk, Wn, lambda, fail);
      schur_accum_kernel<1><<<Wn.n_jobs, ACC_THREADS, acc_smem(), s>>>(Wn, B); return 2;
    case F_HYBRID3: case F_HYBRID_STEREO3:
      schur_stage_kernel<2, 0, 12><<<sgrid, STG_WARPS*32, 0, s>>>(blk, Wn, lambda, fail);
      schur_accum_kernel<2><<<Wn.n_jobs, ACC_THREADS, acc_smem(), s>>>(Wn, B); return 2;
    default: return 0;
  }
}

}  // namespace dynoba
