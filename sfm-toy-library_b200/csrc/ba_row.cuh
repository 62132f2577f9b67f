// ba_row.cuh -- K3c: the off-diagonal blocks of the reduced camera system in gather mode (default), the fixed-order combine
// kernel and the stable camera-major sort.  Included by ba.cu inside its anonymous namespace (uses BAView, LMX, blk_index,
// dmma_m8n8k4).
//
// Formulation.  Inside a point the observations are stored in ascending camera order (std::map order, reference
// SfMBundleAdjustmentUtils.cpp:146), so every pair of observations (i, j) of a point with cameras ci < cj contributes
// -Z_i Z_j^T to block S[ci, cj].  The (i, j) index pairs are listed once per problem, per (camera pair, point segment) and
// sorted by point (pair_fill_sorted_kernel, no arrival-order atomics); ba_pair_kernel walks them with one
// mma.sync.m8n8k4.f64 per entry and writes one partial block per (pair, segment, split).  Point segments are sized so that
// the slice of Zbuf they read stays L2-resident (pair_segments in ba.cu).
//   * The diagonal blocks, camera-focal column, rhs, gradient and J^T J diagonal come from ba_camera_kernel<DET> (ba.cu): one
//     partial record per (slice, camera).
//   * ba_combine_kernel sums the partial blocks and records in a fixed order.  No floating-point atomics anywhere: two runs
//     give bitwise identical results.
#pragma once

constexpr int ROW_HDR = 64;                               // doubles of a camera partial record (= CAM_REC of ba_camera_kernel)
struct RowArgs {
    int diag_per_cta;             // camera-major entries per CTA slice of the diagonal kernel
    double* diag_part;            // [(diag grid + nc)][ROW_HDR]   record of (slice s, camera c) = s + c
    const int32_t* pair_off;      // [nblk * nseg + 1] entry-list offsets of (camera pair, point segment)
    const double* pair_part;      // [nblk * nseg * splits][36] partial blocks written by ba_pair_kernel
    const int32_t* pair_blk;      // [n_nonempty] camera pairs that have entries
    int nseg, splits, n_nonempty;
};

// ---------------------------------------------------------------------------------------------------------------
// K3c: off-diagonal blocks without atomics.  For every camera pair (ci < cj) the list of (obs_i, obs_j)
// index pairs of the points both cameras see is built once per problem (the structure is fixed across LM iterations).
// One warp per (pair, split): lanes stride over the list, each accumulating a full 6x6 block  sum Z_i Z_j^T  in 36
// registers from two 144-byte reads, then a warp shuffle reduction and 36 REDs per warp (instead of 36 per entry).
// ---------------------------------------------------------------------------------------------------------------
constexpr int PAIR_WARPS = 4;
// pair_off is indexed by key = blk * nseg + seg (seg = point-range segment): the grid walks the segments in the slow
// (y) dimension, LAST segment first, so that all resident warps read the same L2-sized slice of Zbuf -- which then lives
// in L2 (the tail of Zbuf is still L2-resident from the point kernel that just wrote it).
// The accumulation  S[ci,cj] -= sum_e Z_i(e) Z_j(e)^T  is a (6 x 3E)(3E x 6) product in fp64: it runs on the FP64
// tensor pipe as one  mma.sync.m8n8k4.f64  per entry (6x6x3 padded to 8x8x4).  The operand fragments want lane l to hold
// element (l>>2, l&3) of the 8x4 tile, i.e. double number (l>>2)*3 + (l&3) of the 18-double Z record: one coalesced
// 8-byte load per lane per operand (18 of 32 lanes active, one 144-byte record = at most two 128-byte lines), instead
// of 18 uncoalesced 16-byte loads per lane in a lane-per-entry SIMT formulation (which was L1-wavefront bound).
constexpr int PAIR_UNROLL = 8;
// Occupancy: a bound of 8 CTAs per SM capped the kernel at 64 registers, and ptxas spilled the batch's operands and
// accumulator fragments to local memory inside the entry loop (72 bytes of spill stores).  With 6 the kernel takes 72
// registers and no spills, and 7 CTAs (28 warps) still fit in the register file.
// Measured: 0.365 -> 0.307 ms per cfg 3 iteration (H100 80GB HBM3 at 400 W, L2 flushed).
constexpr int PAIR_MIN_CTAS_PER_SM = 6;
__global__ void __launch_bounds__(PAIR_WARPS * 32, PAIR_MIN_CTAS_PER_SM) ba_pair_kernel(const double* __restrict__ Zbuf, const int32_t* __restrict__ pair_off,
                                                                   const uint2* __restrict__ pair_ent, int n_nonempty, int nseg, int splits,
                                                                   const int32_t* __restrict__ pair_blk, double* __restrict__ pair_part, const LMState* __restrict__ st) {
    if (st && st->status != LM_RUNNING) return;
    const int lane = threadIdx.x & 31;
    const int q = blockIdx.x * PAIR_WARPS + (threadIdx.x >> 5);       // index into the list of non-empty pairs
    if (q >= n_nonempty) return;
    const int seg = nseg - 1 - (int)(blockIdx.y / splits), sp = blockIdx.y % splits;
    const int blk = pair_blk[q];
    const int start = pair_off[(size_t)blk * nseg + seg], len = pair_off[(size_t)blk * nseg + seg + 1] - start;
    // split sp of the list: [start + floor(len*sp/splits), start + floor(len*(sp+1)/splits)), in 32-bit arithmetic
    const int lq = len / splits, lr = len - lq * splits;
    const int b0 = start + lq * sp + lr * sp / splits, b1 = start + lq * (sp + 1) + lr * (sp + 1) / splits;
    if (b1 <= b0) return;
    const int fr = lane >> 2, fc = lane & 3;
    const bool valid = fr < 6 && fc < 3;
    const int fidx = valid ? fr * 3 + fc : 0;
    double c0[4], c1[4];               // 4 independent accumulator fragments
#pragma unroll
    for (int u = 0; u < 4; ++u) { c0[u] = 0.0; c1[u] = 0.0; }
    // Entries arrive in batches of PAIR_UNROLL: lanes 0..7 fetch the batch's index pairs with ONE coalesced 64-byte load (a
    // broadcast load per entry cost a wavefront each) and hand them round with shuffles; the NEXT batch's indices are
    // requested before this batch's operands are consumed, so that the index round trip and the operand round trip of
    // consecutive batches overlap (the kernel is latency bound: 83% long-scoreboard stalls).
    uint2 cur = make_uint2(0u, 0u);
    if (lane < PAIR_UNROLL && b0 + lane < b1) cur = __ldg(pair_ent + b0 + lane);
    for (int e = b0; e < b1; e += PAIR_UNROLL) {
        uint2 nxt = make_uint2(0u, 0u);
        const int en = e + PAIR_UNROLL;
        if (lane < PAIR_UNROLL && en + lane < b1) nxt = __ldg(pair_ent + en + lane);
        double a[PAIR_UNROLL], b[PAIR_UNROLL];
#pragma unroll
        for (int u = 0; u < PAIR_UNROLL; ++u) {
            const unsigned ox = __shfl_sync(0xffffffffu, cur.x, u), oy = __shfl_sync(0xffffffffu, cur.y, u);
            const bool live = valid && e + u < b1;                     // past the end: indices are 0, operands forced to 0
            const double va = __ldg(Zbuf + (size_t)ox * 18 + fidx), vb = __ldg(Zbuf + (size_t)oy * 18 + fidx);
            a[u] = live ? va : 0.0; b[u] = live ? vb : 0.0;
        }
#pragma unroll
        for (int u = 0; u < PAIR_UNROLL; ++u) dmma_m8n8k4(c0[u & 3], c1[u & 3], a[u], b[u]);
        cur = nxt;
    }
    double s0 = 0.0, s1 = 0.0;
#pragma unroll
    for (int u = 0; u < 4; ++u) { s0 += c0[u]; s1 += c1[u]; }
    // accumulator fragment: row = lane>>2, columns 2*(lane&3) and 2*(lane&3)+1.  One partial block per (pair, segment, split):
    // ba_combine_kernel adds them up in a fixed order (no atomics: bitwise reproducible)
    const int cc = 2 * fc;
    if (fr < 6 && cc < 6)
        *reinterpret_cast<double2*>(pair_part + (((size_t)blk * nseg + seg) * splits + sp) * 36 + fr * 6 + cc) = make_double2(s0, s1);
}

// pair-list construction (once per problem): thread per point; key = blk * nseg + seg(point)
__device__ __forceinline__ int point_segment(int p, int np, int nseg) { return (int)((long long)p * nseg / np); }
__global__ void __launch_bounds__(256) pair_count_kernel(const int32_t* __restrict__ pt_off, const int32_t* __restrict__ obs_cam, int np, int nb,
                                                         int nseg, int* __restrict__ cnt) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= np) return;
    const int o0 = pt_off[p], o1 = pt_off[p + 1], seg = point_segment(p, np, nseg);
    for (int i = o0; i < o1; ++i)
        for (int j = i + 1; j < o1; ++j) atomicAdd(cnt + (size_t)blk_index(obs_cam[i], obs_cam[j], nb) * nseg + seg, 1);
}
// exclusive scan of cnt[nkeys] -> pair_off[nkeys+1] and cursor[nkeys]; single CTA, chained over 1024-element chunks
__global__ void __launch_bounds__(1024) pair_scan_kernel(const int* __restrict__ cnt, int nkeys, int32_t* __restrict__ pair_off, int* __restrict__ cursor) {
    __shared__ int wsum[32], carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int base = 0; base < nkeys; base += 1024) {
        const int i = base + threadIdx.x;
        const int c = i < nkeys ? cnt[i] : 0;
        int s = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int a = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += a; }
        if (lane == 31) wsum[w] = s;
        __syncthreads();
        if (w == 0) {
            int a = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, a, o); if (lane >= o) a += x; }
            wsum[lane] = a;
        }
        __syncthreads();
        const int ex = carry_s + (w ? wsum[w - 1] : 0) + s - c;
        if (i < nkeys) { cursor[i] = ex; pair_off[i] = ex; }
        __syncthreads();
        if (threadIdx.x == 0) carry_s += wsum[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) pair_off[nkeys] = carry_s;
}
// list of camera pairs that have at least one entry; single CTA (nblk = nc(nc+1)/2 is small)
__global__ void __launch_bounds__(1024) pair_compact_kernel(const int32_t* __restrict__ pair_off, int nblk, int nseg, int32_t* __restrict__ pair_blk,
                                                            int* __restrict__ n_nonempty) {
    __shared__ int wcnt[32], carry_q;
    if (threadIdx.x == 0) carry_q = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int base = 0; base < nblk; base += 1024) {
        const int i = base + threadIdx.x;
        const int f = i < nblk ? (pair_off[(size_t)(i + 1) * nseg] > pair_off[(size_t)i * nseg]) : 0;
        int q = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int b = __shfl_up_sync(0xffffffffu, q, o); if (lane >= o) q += b; }
        if (lane == 31) wcnt[w] = q;
        __syncthreads();
        if (w == 0) {
            int b = wcnt[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, b, o); if (lane >= o) b += y; }
            wcnt[lane] = b;
        }
        __syncthreads();
        if (f) pair_blk[carry_q + (w ? wcnt[w - 1] : 0) + q - 1] = i;
        __syncthreads();
        if (threadIdx.x == 0) carry_q += wcnt[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) *n_nonempty = carry_q;
}
// Deterministic fill of the entry lists (once per problem): one CTA per camera ci walks ci's STABLE camera-major list (ascending
// point) in chunks; the observations of the same point by cameras cj > ci are the records that follow it in the point-major
// order (cm_np of them).  The position of entry (ci, cj, point) in list (ci,cj) is the number of earlier points seen by both,
// computed without arrival-order atomics: per chunk a 32-bit lane mask per (warp, cj) (atomicOr: order-independent), a prefix
// over the warps, a running count per cj.  The lists of (ci,cj) for all point segments are contiguous and ascending in point,
// so the segment boundaries (pair_off, from the counting kernel) fall out by themselves.
constexpr int PFILL_THREADS = 256;
constexpr int PFILL_WARPS = PFILL_THREADS / 32;
__global__ void __launch_bounds__(PFILL_THREADS) pair_fill_sorted_kernel(const int32_t* __restrict__ cm_off, const int32_t* __restrict__ cm_obs, const uint8_t* __restrict__ cm_np,
                                                                        const int32_t* __restrict__ obs_cam, int nb, int nseg, const int32_t* __restrict__ pair_off,
                                                                        uint2* __restrict__ ent) {
    extern __shared__ unsigned pf_smem[];
    unsigned* mask = pf_smem;                       // [PFILL_WARPS][nb]
    int* running = reinterpret_cast<int*>(mask + (size_t)PFILL_WARPS * nb);   // [nb]: entries of list (ci, cj) placed so far
    int* wbase = running + nb;                      // [PFILL_WARPS][nb]
    const int ci = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int begin = cm_off[ci], end = cm_off[ci + 1];
    for (int k = threadIdx.x; k < nb; k += PFILL_THREADS) running[k] = 0;
    for (int b0 = begin; b0 < end; b0 += PFILL_THREADS) {
        for (int k = threadIdx.x; k < PFILL_WARPS * nb; k += PFILL_THREADS) mask[k] = 0u;
        __syncthreads();
        const int i = b0 + threadIdx.x;
        const int o = i < end ? cm_obs[i] : 0, ne = i < end ? (int)cm_np[i] : 0;
        for (int q = 0; q < ne; ++q) atomicOr(mask + (size_t)warp * nb + obs_cam[o + 1 + q], 1u << lane);
        __syncthreads();
        for (int k = threadIdx.x; k < nb; k += PFILL_THREADS) {
            int run = running[k];
#pragma unroll
            for (int w = 0; w < PFILL_WARPS; ++w) { wbase[w * nb + k] = run; run += __popc(mask[(size_t)w * nb + k]); }
            running[k] = run;
        }
        __syncthreads();
        for (int q = 0; q < ne; ++q) {
            const int cj = obs_cam[o + 1 + q];
            const int pos = pair_off[(size_t)blk_index(ci, cj, nb) * nseg] + wbase[warp * nb + cj] + __popc(mask[(size_t)warp * nb + cj] & ((1u << lane) - 1u));
            ent[pos] = make_uint2((unsigned)o, (unsigned)(o + 1 + q));
        }
        __syncthreads();
    }
}

// Fixed-order sums of the partial results -> the reduced system in the layout the rest of the solver (rank exchange,
// ba_assemble_kernel, ba_cam_update_kernel) reads: Sblk | Scf | Sff | rhs | gcf | dcf.
//   CTAs [0, nc): camera c -- the partial records of ba_camera_kernel<DET> in slice order (diagonal block, camera-focal column,
//     rhs, gradient, J^T J diagonal).  The focal terms need a sum over cameras: the last of these CTAs to finish adds them up in
//     camera order (fixed order whoever is last).
//   CTAs [nc, ..): one warp per non-empty camera pair -- the partial blocks of ba_pair_kernel in (segment, split) order (a warp
//     whose range of the list is empty wrote nothing: same arithmetic as in the kernel).  Empty pairs stay zero (never written).
// norm_only: only the squared column norms of the unscaled Jacobian (Jacobi scaling at x0) -> colnorm [6 nc + 1].
constexpr int COMBINE_THREADS = 256;
__global__ void __launch_bounds__(COMBINE_THREADS) ba_combine_kernel(BAView v, RowArgs ra, int norm_only, double* __restrict__ colnorm,
                                                                     double* __restrict__ fpart /* [nc][2] */, unsigned* __restrict__ counter) {
    if (v.st && v.st->status != LM_RUNNING) return;
    const int nc = v.nc;
    if ((int)blockIdx.x >= nc) {
        const int q = ((int)blockIdx.x - nc) * (COMBINE_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
        if (q >= ra.n_nonempty) return;
        const size_t blk = ra.pair_blk[q];
        double s0 = 0.0, s1 = 0.0;                                          // elements lane and lane + 32 (< 36) of the block
        for (int seg = 0; seg < ra.nseg; ++seg) {
            const int start = ra.pair_off[blk * ra.nseg + seg], len = ra.pair_off[blk * ra.nseg + seg + 1] - start;
            if (len <= 0) continue;
            const int lq = len / ra.splits, lr = len - lq * ra.splits;
            const double* pb = ra.pair_part + (blk * ra.nseg + seg) * ra.splits * 36;
            for (int sp = 0; sp < ra.splits; ++sp, pb += 36) {
                if (lq == 0 && lr * sp / ra.splits == lr * (sp + 1) / ra.splits) continue;     // this split's range is empty: nothing was written
                s0 += pb[lane];
                if (lane < 4) s1 += pb[32 + lane];
            }
        }
        v.Sblk[blk * 36 + lane] = -s0;
        if (lane < 4) v.Sblk[blk * 36 + 32 + lane] = -s1;
        return;
    }
    const int c = blockIdx.x;
    int dfirst = 0, dlast = -1;
    if (v.cm_off[c + 1] > v.cm_off[c]) { dfirst = v.cm_off[c] / ra.diag_per_cta; dlast = (v.cm_off[c + 1] - 1) / ra.diag_per_cta; }
    auto sum = [&](int idx) {
        double s = 0.0;
        for (int sl = dfirst; sl <= dlast; ++sl) s += ra.diag_part[(size_t)(sl + c) * ROW_HDR + idx];
        return s;
    };
    if (norm_only) {
        if (threadIdx.x < 6) colnorm[6 * c + threadIdx.x] = sum(54 + threadIdx.x);
        if (threadIdx.x == 6) fpart[2 * c] = sum(60);
    } else if (threadIdx.x < 62) {
        const int t = threadIdx.x;
        const double s = sum(t);
        if (t < 36) v.Sblk[blk_index(c, c, nc) * 36 + t] = s;
        else if (t < 42) v.Scf[6 * c + (t - 36)] = s;
        else if (t < 48) v.rhs[6 * c + (t - 42)] = s;
        else if (t < 54) v.gcf[6 * c + (t - 48)] = s;
        else if (t < 60) v.dcf[6 * c + (t - 54)] = s;
        else fpart[2 * c + (t - 60)] = s;
    }
    __shared__ bool is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicInc(counter, nc - 1) == (unsigned)(nc - 1);      // wraps to 0: ready for the next launch
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    if (threadIdx.x == 0) {
        double ff = 0.0, gf = 0.0;
        for (int k = 0; k < nc; ++k) { ff += __ldcg(fpart + 2 * k); gf += __ldcg(fpart + 2 * k + 1); }
        const int fidx = 6 * nc;
        if (norm_only) colnorm[fidx] = ff;
        else {
            // the point kernel's last CTA stored the point part of S_ff and rhs_f there (stream order: it ran before)
            *v.Sff += ff; v.dcf[fidx] = ff; v.rhs[fidx] += gf; v.gcf[fidx] = gf;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Stable camera-major copy of the observation list (structure fixed across LM iterations, built once per problem): a counting
// sort by camera in which the rank of an observation among those of its camera is computed WITHOUT arrival-order atomics
// (__match_any_sync inside a warp, a prefix over the warps of a CTA, a scan over the CTAs) -- so each camera's list is in
// ascending point order, the same on every run.  SCATTER = false: per-CTA histograms only.
// ---------------------------------------------------------------------------------------------------------------
constexpr int CMS_THREADS = 256;
constexpr int CMS_WARPS = CMS_THREADS / 32;
template <bool SCATTER>
__global__ void __launch_bounds__(CMS_THREADS) cm_sort_kernel(const int32_t* __restrict__ obs_cam, const float2* __restrict__ obs_xy,
                                                              const int32_t* __restrict__ obs_pt, const int32_t* __restrict__ pt_off, int nobs, int nc,
                                                              int* __restrict__ hist /* [ncta][nc]: counts (in), exclusive prefix over CTAs (SCATTER) */,
                                                              const int32_t* __restrict__ cm_off, float2* __restrict__ cm_xy, int32_t* __restrict__ cm_pt,
                                                              int32_t* __restrict__ cm_obs, uint8_t* __restrict__ cm_np) {
    extern __shared__ int wcnt[];                                           // [CMS_WARPS][nc]
    const int o = blockIdx.x * CMS_THREADS + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < CMS_WARPS * nc; i += CMS_THREADS) wcnt[i] = 0;
    __syncthreads();
    const bool valid = o < nobs;
    const int c = valid ? obs_cam[o] : -1 - lane;                           // invalid lanes get distinct keys
    const unsigned m = __match_any_sync(0xffffffffu, c);
    const int rank = __popc(m & ((1u << lane) - 1u));
    if (valid && rank == 0) wcnt[warp * nc + c] = __popc(m);
    __syncthreads();
    for (int k = threadIdx.x; k < nc; k += CMS_THREADS) {
        int run = 0;
#pragma unroll
        for (int w = 0; w < CMS_WARPS; ++w) { const int t = wcnt[w * nc + k]; wcnt[w * nc + k] = run; run += t; }
        if (!SCATTER) hist[(size_t)blockIdx.x * nc + k] = run;
    }
    if (!SCATTER) return;
    __syncthreads();
    if (valid) {
        const int pos = cm_off[c] + hist[(size_t)blockIdx.x * nc + c] + wcnt[warp * nc + c] + rank;
        const int p = obs_pt[o];
        cm_xy[pos] = obs_xy[o]; cm_pt[pos] = p; cm_obs[pos] = o; cm_np[pos] = (uint8_t)(pt_off[p + 1] - o - 1);
    }
}
// per camera: exclusive scan of hist[.][c] over the CTAs (in place) and the camera's total.  One CTA per camera.
__global__ void __launch_bounds__(1024) cm_scan_ctas_kernel(int* __restrict__ hist, int ncta, int nc, int* __restrict__ total) {
    __shared__ int wsum[32], carry_s;
    const int c = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < ncta; base += 1024) {
        const int i = base + threadIdx.x;
        const int val = i < ncta ? hist[(size_t)i * nc + c] : 0;
        int s = val;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int a = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += a; }
        if (lane == 31) wsum[w] = s;
        __syncthreads();
        if (w == 0) {
            int a = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, a, o); if (lane >= o) a += y; }
            wsum[lane] = a;
        }
        __syncthreads();
        if (i < ncta) hist[(size_t)i * nc + c] = carry_s + (w ? wsum[w - 1] : 0) + s - val;
        __syncthreads();
        if (threadIdx.x == 0) carry_s += wsum[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) total[c] = carry_s;
}
