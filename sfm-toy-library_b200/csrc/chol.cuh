// chol.cuh -- K4: dense Cholesky of the reduced camera system (fp64, lower triangle, 32x32 tiles) and the triangular
// solves.  Replaces the dense factorisation inside Ceres' DENSE_SCHUR linear solver that adjustBundle selects
// (reference SfMToyLib/SfMBundleAdjustmentUtils.cpp:171-173).  Shared by ba.cu and tools/chol_microbench.cu.
//
// Matrix layout: A is (npad x npad) row-major, npad a multiple of NB, only the lower triangle is read or written; row n
// carries the right-hand side (forward substitution for free), the remaining pad rows are identity.
#pragma once
#include <cuda_runtime.h>

namespace {

constexpr int NB = 32;                 // Cholesky tile

// A tile is factored by PANEL_WARPS warps (lane = row, the columns dealt to the warps in groups of four).  A single warp
// working through the tile is issue-latency bound (measured: ~5 k dependent instructions at IPC 0.09 = 26 us), so every
// pivot round is split between an owning warp that produces the columns and one barrier after which every warp applies them
// to its own columns.  Pivots with global index >= n are forced to 1 with a zero column (augmented rhs row / padding rows).
constexpr int PANEL_WARPS = 4;

// Barrier among the PANEL_WARPS*32 threads that factor a tile.  The dataflow kernel's CTA has a fifth warp, so this is not
// barrier 0.
__device__ __forceinline__ void chol_factor_barrier() {
    asm volatile("bar.sync 1, %0;" :: "n"(PANEL_WARPS * 32) : "memory");
}

// Factorisation of a 32x32 tile in quad-pivot rounds.  Measured per 32-column tile: one barrier per pivot 6.2 us, pair
// pivots 4.1 us.  A cycle-stamped trace (tools/chol_microbench.cu built with -DCHOL_FINE_TRACE) showed that the cost of a
// round is the NUMBER of instructions the owning warp executes between two barriers (a single warp of mostly dependent fp64
// code runs at ~5 cycles per instruction), not the depth of the pivot recurrence, so the round is built to be short:
//   * warp w owns the column QUADS 16q+4w .. 16q+4w+3 (col[q][h], lane = row): one barrier and one shared-memory round trip
//     serve FOUR pivots;
//   * the owner fetches the 10 entries of the quad's 4x4 diagonal block with shuffles issued together and every lane
//     factors that block redundantly; two pivots share one reciprocal-square-root latency: with D2 = a00 a11 - a10^2 (the
//     leading 2x2 minor, the same cancellation as a11 - a10^2/a00), 1/L11 = rsqrt(D2) sqrt(a00), so both MUFU seeds are in
//     flight together;
//   * no validity or padding selects on the chain: a non-positive pivot only raises `bad` (off the chain) and lets NaNs run
//     through a factor that is thrown away; the padded last tile (pivots >= n forced to 1, zero column) takes the
//     select-carrying TAIL instantiation;
//   * the column vectors are computed for all lanes alike: rows inside the 4x4 block come out right by themselves (the tile
//     is kept fully symmetric), rows above it hold round-off that nothing reads -- whoever stores the factor masks them;
//   * the factor is published TRANSPOSED (LT[j][row], conflict-free, one store per column): the same array serves the
//     update (broadcast LDS of LT[j][c]), the streaming warp and the inverse for the back substitution; nothing is
//     overwritten, so no ping-pong.
__device__ __forceinline__ double chol_rsqrt_fast(double d) {
    double y; asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
    const double t = y * y, e = fma(-d, t, 1.0), p2 = fma(e, 0.375, 0.5), q = y * e;
    return fma(p2, q, y);
}
// Two consecutive pivots of a 2x2 block [a00 .; a10 a11] from two INDEPENDENT reciprocal square roots.
// A pivot a00 or minor D2 is accepted when it is a NORMAL positive double below DBL_MAX: rsqrt.approx.ftz flushes a subnormal to
// zero and returns +inf, which would hand a non-finite factor back with no failure raised (seen at the last pivot of a matrix,
// where no later pivot turns NaN).  So fail == 0 means every pivot and every paired minor was in [DBL_MIN, DBL_MAX).  An SPD
// matrix is factored when its pivots lie within about [1e-150, 1e150] (D2 ~ a00 a11 must neither overflow nor go subnormal),
// as a Jacobi-scaled BA system does; outside that range the solve reports a failure rather than a wrong answer.
template <bool TAIL>
__device__ __forceinline__ void chol_pivot_pair(double a00, double a10, double a11, bool pad0, bool pad1, double& inv0, double& inv1, bool& bad) {
    const double D2 = fma(a00, a11, -(a10 * a10));
    const double s1 = chol_rsqrt_fast(a00), s2 = chol_rsqrt_fast(D2);
    const double sq0 = a00 * s1;                               // sqrt(a00)
    const bool good0 = a00 >= 2.2250738585072014e-308 && a00 < 1.7976931348623157e308, good1 = D2 >= 2.2250738585072014e-308 && D2 < 1.7976931348623157e308;
    if (!TAIL) {
        inv0 = s1; inv1 = s2 * sq0;
        bad = bad || !good0 || !good1;
    } else {
        inv0 = pad0 ? 0.0 : (good0 ? s1 : 1.0);
        inv1 = pad1 ? 0.0 : (good0 && good1 ? s2 * sq0 : 1.0);
        bad = bad || (!pad0 && !good0) || (!pad1 && !good1);
    }
}
#ifdef CHOL_FINE_TRACE
__device__ unsigned long long g_chol_fine[64], g_chol_fine2[64];
#define CHOL_FINE(k) do { if (gbase == 10 * NB && lane == 0) g_chol_fine[k] = (unsigned long long)clock64(); } while (0)
#define CHOL_FINE2(k) do { if (gbase == 10 * NB && lane == 0) g_chol_fine2[(j0 / 4) * 8 + (k)] = (unsigned long long)clock64(); } while (0)
#else
#define CHOL_FINE(k) do { } while (0)
#define CHOL_FINE2(k) do { } while (0)
#endif
// The owner's part of a round: factor the quad j0..j0+3 held in a[0..3] (lane = row), publish LT[j0+k][lane] and invd[j0+k].
template <bool TAIL>
__device__ __forceinline__ void chol_quad_owner(const double (&a)[4], double (*LT)[NB], double* invd, int lane, int j0, int gbase, int n, bool& bad) {
    const double a00 = __shfl_sync(0xffffffffu, a[0], j0), a10 = __shfl_sync(0xffffffffu, a[0], j0 + 1),
                 a20 = __shfl_sync(0xffffffffu, a[0], j0 + 2), a30 = __shfl_sync(0xffffffffu, a[0], j0 + 3),
                 a11 = __shfl_sync(0xffffffffu, a[1], j0 + 1), a21 = __shfl_sync(0xffffffffu, a[1], j0 + 2),
                 a31 = __shfl_sync(0xffffffffu, a[1], j0 + 3), a22 = __shfl_sync(0xffffffffu, a[2], j0 + 2),
                 a32 = __shfl_sync(0xffffffffu, a[2], j0 + 3), a33 = __shfl_sync(0xffffffffu, a[3], j0 + 3);
    CHOL_FINE2(0);
    const int g0 = gbase + j0;
    double i0, i1, i2, i3;
    chol_pivot_pair<TAIL>(a00, a10, a11, g0 >= n, g0 + 1 >= n, i0, i1, bad);
    const double l10 = a10 * i0, l20 = a20 * i0, l30 = a30 * i0;
    const double l21 = fma(-l20, l10, a21) * i1, l31 = fma(-l30, l10, a31) * i1;
    const double b22 = fma(-l21, l21, fma(-l20, l20, a22)), b32 = fma(-l31, l21, fma(-l30, l20, a32)), b33 = fma(-l31, l31, fma(-l30, l30, a33));
    chol_pivot_pair<TAIL>(b22, b32, b33, g0 + 2 >= n, g0 + 3 >= n, i2, i3, bad);
    const double l32 = b32 * i2;
    CHOL_FINE2(1);
    // the four columns for this lane's row
    double v0 = a[0] * i0;
    double v1 = fma(-v0, l10, a[1]) * i1;
    double v2 = fma(-v1, l21, fma(-v0, l20, a[2])) * i2;
    double v3 = fma(-v2, l32, fma(-v1, l31, fma(-v0, l30, a[3]))) * i3;
    if (TAIL) {                                                       // forced pivots: 1 on the diagonal, zero column
        if (g0 >= n) v0 = lane == j0 ? 1.0 : 0.0;
        if (g0 + 1 >= n) v1 = lane == j0 + 1 ? 1.0 : 0.0;
        if (g0 + 2 >= n) v2 = lane == j0 + 2 ? 1.0 : 0.0;
        if (g0 + 3 >= n) v3 = lane == j0 + 3 ? 1.0 : 0.0;
    }
    CHOL_FINE2(2);
    LT[j0][lane] = v0; LT[j0 + 1][lane] = v1; LT[j0 + 2][lane] = v2; LT[j0 + 3][lane] = v3;
    if (lane == 0) { *reinterpret_cast<double2*>(invd + j0) = make_double2(i0, i1); *reinterpret_cast<double2*>(invd + j0 + 2) = make_double2(i2, i3); }
    CHOL_FINE2(3);
}
// col[q][h] = element (row `lane`, column 16q + 4w + h) of the (fully symmetric) tile.  Leaves the factor transposed in LT
// (LT[j][r] = L(r,j) for r >= j; r < j: round-off, to be masked by the reader) and the reciprocal pivots in invd; ends with a
// barrier.  Warp 0 hands every finished quad to the streaming warp through the quad's named barrier (ids 2..9, 32 + 32
// threads; warp 0 only arrives) -- a hand-over compute-sanitizer's racecheck can see.
__device__ __forceinline__ bool chol_tile_factor4(double (&col)[NB / (4 * PANEL_WARPS)][4], double (*LT)[NB], double* invd,
                                                  int lane, int w, int gbase, int n, int* bad_flag) {
    bool bad = false;
    const bool tail = gbase + NB > n;
    if (w == 0) CHOL_FINE(0);
#pragma unroll 1
    for (int jb = 0; jb < NB; jb += 4 * PANEL_WARPS) {
#pragma unroll
        for (int ow = 0; ow < PANEL_WARPS; ++ow) {                    // pivots j0..j0+3 are columns col[0][0..3] of warp ow
            const int j0 = jb + 4 * ow;
            if (w == ow) {
                CHOL_FINE(1 + (j0 / 4) * 4);
                if (tail) chol_quad_owner<true>(col[0], LT, invd, lane, j0, gbase, n, bad);
                else chol_quad_owner<false>(col[0], LT, invd, lane, j0, gbase, n, bad);
                CHOL_FINE(2 + (j0 / 4) * 4);
            }
            chol_factor_barrier();
            if (w == 0) CHOL_FINE(3 + (j0 / 4) * 4);
            if (w == 0) { __threadfence_block(); asm volatile("bar.arrive %0, 64;" ::"r"(2 + j0 / 4) : "memory"); }
            const double m0 = LT[j0][lane], m1 = LT[j0 + 1][lane], m2 = LT[j0 + 2][lane], m3 = LT[j0 + 3][lane];
#pragma unroll
            for (int q = 0; q < NB / (4 * PANEL_WARPS); ++q) {
                const int c0 = jb + 4 * PANEL_WARPS * q + 4 * w;      // columns held in col[q][0..3]; >= NB means wrapped (finished)
                if (c0 > j0 && c0 < NB) {
#pragma unroll
                    for (int hh = 0; hh < 4; hh += 2) {
                        const double2 u0 = *reinterpret_cast<const double2*>(&LT[j0][c0 + hh]), u1 = *reinterpret_cast<const double2*>(&LT[j0 + 1][c0 + hh]),
                                      u2 = *reinterpret_cast<const double2*>(&LT[j0 + 2][c0 + hh]), u3 = *reinterpret_cast<const double2*>(&LT[j0 + 3][c0 + hh]);
                        col[q][hh] = fma(-m3, u3.x, fma(-m2, u2.x, fma(-m1, u1.x, fma(-m0, u0.x, col[q][hh]))));
                        col[q][hh + 1] = fma(-m3, u3.y, fma(-m2, u2.y, fma(-m1, u1.y, fma(-m0, u0.y, col[q][hh + 1]))));
                    }
                }
            }
        }
        if (w == 0) CHOL_FINE(4 + (jb / 4 + 3) * 4);
        // rotate the register set by one quad
#pragma unroll
        for (int q = 0; q < NB / (4 * PANEL_WARPS) - 1; ++q)
#pragma unroll
            for (int h = 0; h < 4; ++h) col[q][h] = col[q + 1][h];
    }
    if (bad) *bad_flag = 1;                        // a pivot is seen by its owning warp only
    chol_factor_barrier();
    return *bad_flag != 0;
}

// One warp solves X L^T = B for row `lane` of B, with the factor stored transposed (LT[j][c] = L(c,j)) as chol_tile_factor4
// leaves it and the reciprocal pivots in invd.  b[] is rotated by PANEL_WARPS per group of pivots, so that the loop over the
// groups stays rolled with static register indices (b[0] is always the current pivot's column); L(c,j) arrives as a
// broadcast LDS.  On return b[] is back in natural order.
__device__ __forceinline__ void chol_tile_trsm_t(double (&b)[NB], const double (*LT)[NB], const double* invd) {
#pragma unroll 1
    for (int jb = 0; jb < NB; jb += PANEL_WARPS) {
#pragma unroll
        for (int u = 0; u < PANEL_WARPS; ++u) {
            const int j = jb + u;
            const double xj = b[u] * invd[j];
            b[u] = xj;
#pragma unroll
            for (int p2 = u + 1; p2 < NB; ++p2)
                if (jb + p2 < NB) b[p2] = fma(-xj, LT[j][jb + p2], b[p2]);
        }
        double t[PANEL_WARPS];
#pragma unroll
        for (int u = 0; u < PANEL_WARPS; ++u) t[u] = b[u];
#pragma unroll
        for (int p2 = 0; p2 < NB - PANEL_WARPS; ++p2) b[p2] = b[p2 + PANEL_WARPS];
#pragma unroll
        for (int u = 0; u < PANEL_WARPS; ++u) b[NB - PANEL_WARPS + u] = t[u];
    }
}

// ---------------------------------------------------------------------------------------------------------------
// K4: the whole factorisation as ONE persistent dataflow kernel (left-looking tile Cholesky).  A panel kernel and an update
// kernel per 32 columns would pay a kernel boundary and a cold L2 round trip twice per 32 columns (19 + 18 launches at 100
// cameras, ~390 us measured) although the arithmetic is 72 MFLOP.  Here every lower-triangle tile (i, c) has one owner CTA
// that keeps it in registers for its whole life:
//     for k < c:  wait ready(i,k), ready(c,k);  tile -= L(i,k) L(c,k)^T            (operands through shared memory)
//     i == c:     factor the tile (chol_tile_factor4), store L(c,c) + reciprocal pivots, publish it
//     i >  c:     wait for L(c,c);  solve X L(c,c)^T = tile, store L(i,c), publish ready(i,c)
// The critical path runs down the diagonal, factor(c) -> solve(c+1,c) -> update -> factor(c+1); with separate owners that is
// two global-memory hand-overs per 32 columns.  So the first sub-diagonal tile (c+1,c) and the diagonal tile (c+1,c+1) share
// one owner (the "merged" task): it carries both tiles through the updates, solves (c+1,c), applies it to the diagonal tile
// straight from shared memory and factors -- one hand-over per 32 columns.
// Publishing a tile = all stores, barrier, __threadfence + a store of the solve's epoch number into ready[] (no reset between
// solves); consuming = every thread polls (relaxed), fences, then reads the tile with ld.global.cg (L1 may hold the
// pre-factor values of a tile another CTA of this SM owned).
// Deadlock freedom: tasks are numbered column-major (the merged task sits in column c) and dealt round-robin, each CTA works
// through its tasks in ascending order, and the grid never exceeds the number of co-resident CTAs; the lowest unfinished task
// then depends only on finished tasks and its owner is resident and has nothing else to do.  Waits are bounded all the same
// (fail += 1000 on timeout).
// ---------------------------------------------------------------------------------------------------------------
constexpr long long CF_TIMEOUT_CYCLES = 2000000000LL;       // ~1 s

__device__ __forceinline__ unsigned ld_relaxed_gpu_u32(const unsigned* p) {
    unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ unsigned ld_acquire_gpu_u32(const unsigned* p) {
    unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_relaxed_gpu_u32(unsigned* p, unsigned v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long chol_globaltimer() {
    unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t;
}
__device__ __forceinline__ bool tile_wait(const unsigned* flag, unsigned epoch) {
    bool ok = ld_relaxed_gpu_u32(flag) == epoch;
    if (!ok) {
        const long long t0 = clock64();
        for (;;) {
            if (ld_relaxed_gpu_u32(flag) == epoch) { ok = true; break; }
            if (clock64() - t0 > CF_TIMEOUT_CYCLES) break;
        }
    }
    (void)ld_acquire_gpu_u32(flag);     // acquire side: the tile loads below are ordered after the flag
    return ok;
}
// after a barrier that follows the tile's stores
__device__ __forceinline__ void tile_publish(unsigned* flag, unsigned epoch) {
    __threadfence();
    st_relaxed_gpu_u32(flag, epoch);
}
// number of tasks of the dataflow kernel for nbk tile rows: column 0 holds nbk tiles, every later column c one tile fewer
// than its length because its diagonal tile rides with the merged task of column c-1
__host__ __device__ inline int chol_stream_tasks(int nbk) { return nbk + (nbk - 1) * (nbk - 2) / 2; }

// The shape of the kernel follows a timeline of the chain (tools/chol_microbench.cu).  With four warps that factor, then
// solve, then update with SIMT FMAs, each 32 columns spent 5.4 us in the factorisation, 4.6 us in the solve that FOLLOWED
// it, 1.5 us in the rank-32 update and only 0.75 us in the hand-over.  So:
//   * the factor of a diagonal tile is streamed out in groups of 4 columns while it is being computed: a fifth warp of the
//     owner CTA copies the finished columns from shared memory to A and to the LL lines below; every solve of that tile
//     column consumes the groups as they arrive and finishes a fraction of a microsecond after the factorisation instead
//     of 4.6 us later.  A per-group trace later showed the solving task seeing the groups 0.55 us apart while they were
//     written 0.35 us apart: its loader warp polled one group at a time, one L2 round trip each.  With the loads of three
//     groups in flight the step per 32 columns went from ~7.0 to ~4.8 us (H100 80GB HBM3, 700 W);
//   * the rank-32 updates run on the FP64 tensor pipe (mma.sync.m8n8k4.f64, accumulators in fragment layout for the whole
//     life of the tile, operands from shared memory with a conflict-free 36-double row stride): 40 LDS + 32 DMMA per warp
//     instead of 288 LDS + 256 DFMA;
//   * the fifth warp also hands the streamed groups to the solve of its own CTA, and after a factorisation produces
//     L(c,c)^-1 for the back substitution.
// ---------------------------------------------------------------------------------------------------------------
constexpr int CS_THREADS = PANEL_WARPS * 32 + 32;
constexpr int TS = NB + 4;              // row stride of the DMMA operand tiles

__device__ __forceinline__ void chol_dmma(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
// fragment-layout accumulator of warp w: acc[cb][h] = C[8w + lane/4][8cb + 2(lane%4) + h]
// acc -= P Q^T for the column blocks cb < ncb  (P, Q: [NB][TS] in shared memory)
__device__ __forceinline__ void tile_dmma_update(double (&acc)[4][2], const double (*P)[TS], const double (*Q)[TS], int lane, int w, int ncb) {
    const int fr = lane >> 2, fc = lane & 3;
#pragma unroll
    for (int ks = 0; ks < NB / 4; ++ks) {
        const double a = -P[8 * w + fr][4 * ks + fc];
#pragma unroll
        for (int cb = 0; cb < 4; ++cb)
            if (cb < ncb) chol_dmma(acc[cb][0], acc[cb][1], a, Q[8 * cb + fr][4 * ks + fc]);
    }
}
// one k-step (columns 4ks..4ks+3 of P and Q) of the update above
__device__ __forceinline__ void tile_dmma_update_k(double (&acc)[4][2], const double (*P)[TS], const double (*Q)[TS], int lane, int w, int ncb, int ks) {
    const int fr = lane >> 2, fc = lane & 3;
    const double a = -P[8 * w + fr][4 * ks + fc];
#pragma unroll
    for (int cb = 0; cb < 4; ++cb)
        if (cb < ncb) chol_dmma(acc[cb][0], acc[cb][1], a, Q[8 * cb + fr][4 * ks + fc]);
}
__device__ __forceinline__ void tile_to_smem_ts(double (*T)[TS], const double* __restrict__ A, int npad, int row0, int col0) {
    if (threadIdx.x < PANEL_WARPS * 32) {
        double2 v[NB * NB / (2 * PANEL_WARPS * 32)];
#pragma unroll
        for (int u = 0; u < NB * NB / (2 * PANEL_WARPS * 32); ++u) {
            const int e = threadIdx.x + u * PANEL_WARPS * 32, r = e >> 4, c = (e & 15) * 2;
            v[u] = __ldcg(reinterpret_cast<const double2*>(A + (size_t)(row0 + r) * npad + col0 + c));
        }
#pragma unroll
        for (int u = 0; u < NB * NB / (2 * PANEL_WARPS * 32); ++u) {
            const int e = threadIdx.x + u * PANEL_WARPS * 32, r = e >> 4, c = (e & 15) * 2;
            *reinterpret_cast<double2*>(&T[r][c]) = v[u];
        }
    }
}
// Hand-over of a finished 4-column group between CTAs, flag-in-data ("LL" lines as in NCCL's low-latency protocol): a double
// travels as one 16-byte line {lo, tag, hi, tag}; the reader polls the line itself and takes the value when both tags carry
// the number of the current solve.  Against "store, __threadfence, flag / poll flag, then load" this takes the fence (the
// streaming warp could publish one group per ~0.75 us, slower than the factorisation produces them) and one of the two L2
// round trips out of the chain.  Only 8-byte atomicity of the store is assumed.  Lines of a group: [4 columns][32 rows], then
// 4 reciprocal pivots; CHOL_LL_GROUP lines per group, 8 groups per tile.  Tags never repeat (solve numbers), so no reset.
constexpr int CHOL_LL_GROUP = 4 * NB + 32;
__host__ __device__ inline size_t chol_ll_bytes(int nbk) { return (size_t)nbk * (NB / PANEL_WARPS) * CHOL_LL_GROUP * 16; }
__device__ __forceinline__ void ll_store(uint4* line, double v, unsigned tag) {
    const unsigned lo = (unsigned)__double2loint(v), hi = (unsigned)__double2hiint(v);
    asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" :: "l"(line), "r"(lo), "r"(tag), "r"(hi), "r"(tag) : "memory");
}
// A poll is split into the load (ll_group_issue: this lane's lines of a group -- row `lane` of its 4 columns where that row
// exists, rows >= 4g, and lanes 0..3 a reciprocal pivot) and the test of the tags (ll_group_ready), so that the loads of several
// groups can be in flight at once.
constexpr int LL_AHEAD = 3;
__device__ __forceinline__ void ll_load(uint4& d, const uint4* line) {
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(d.x), "=r"(d.y), "=r"(d.z), "=r"(d.w) : "l"(line) : "memory");
}
__device__ __forceinline__ double ll_value(const uint4& d) { return __hiloint2double((int)d.z, (int)d.x); }
__device__ __forceinline__ bool ll_tagged(const uint4& d, unsigned tag) { return d.y == tag && d.w == tag; }
__device__ __forceinline__ void ll_group_issue(uint4 (&d)[5], const uint4* ll, int c, int g, int lane) {
    const uint4* grp = ll + ((size_t)c * (NB / PANEL_WARPS) + g) * CHOL_LL_GROUP;
    if (lane >= PANEL_WARPS * g) { ll_load(d[0], grp + lane); ll_load(d[1], grp + NB + lane); ll_load(d[2], grp + 2 * NB + lane); ll_load(d[3], grp + 3 * NB + lane); }
    if (lane < PANEL_WARPS) ll_load(d[4], grp + 4 * NB + lane);
}
__device__ __forceinline__ bool ll_group_ready(const uint4 (&d)[5], int g, int lane, unsigned tag) {
    bool r = true;
    if (lane >= PANEL_WARPS * g) r = ll_tagged(d[0], tag) && ll_tagged(d[1], tag) && ll_tagged(d[2], tag) && ll_tagged(d[3], tag);
    if (lane < PANEL_WARPS) r = r && ll_tagged(d[4], tag);
    return r;
}

// `skip` (every kernel of this file, optional): when it points at a non-zero word the launch is a no-op -- the device-resident
// LM loop enqueues whole chunks of iterations and the solve may terminate inside one.
// trace (optional, tools/chol_microbench.cu): 8 x u64 %globaltimer stamps per task: 0 start, 1 updates done, 2 first group of
// L(c,c) seen, 3 solve done, 4 (i,c) published, 5 factor done, 6 factor streamed out, 7 factor start
__global__ void __launch_bounds__(CS_THREADS) chol_stream_kernel(double* __restrict__ A, int npad, int n, int nbk, int ntasks,
                                                                 double* __restrict__ dinv, int* __restrict__ fail,
                                                                 unsigned* __restrict__ ready, uint4* __restrict__ ll, unsigned epoch,
                                                                 double* __restrict__ Linv, unsigned long long* __restrict__ trace,
                                                                 const int* __restrict__ skip = nullptr, const unsigned* __restrict__ epoch_dev = nullptr) {
    if (skip && *skip) return;
    if (epoch_dev) epoch = *epoch_dev;       // CUDA-graph replays: the solve number lives on the device (kernel arguments are frozen)
    __shared__ __align__(16) double Pt[NB][TS], Qt[NB][TS], Xs[NB][TS];
    __shared__ double Ls[NB][NB + 1];
    __shared__ __align__(16) double LT[NB][NB];        // factor of the diagonal tile, transposed (chol_tile_factor4)
    __shared__ __align__(16) double invd[NB];
    __shared__ int bad_flag, abort_flag;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, fr = lane >> 2, fc = lane & 3;
    const bool tile_warp = w < PANEL_WARPS;
    if (threadIdx.x == 0) { bad_flag = 0; abort_flag = 0; }
    __syncthreads();
#define CHOL_TRACE(slot) do { if (trace && threadIdx.x == 0) trace[(size_t)t * 8 + (slot)] = chol_globaltimer(); } while (0)
#define CHOL_TRACE_W4(slot) do { if (trace && threadIdx.x == PANEL_WARPS * 32) trace[(size_t)t * 8 + (slot)] = chol_globaltimer(); } while (0)
    for (int t = blockIdx.x; t < ntasks; t += gridDim.x) {
        int i, c; bool merged = false;
        if (t == 0) { i = c = 0; }
        else {
            int rem = t - 1, cnt = nbk - 1; c = 0;
            while (rem >= cnt) { rem -= cnt; ++c; cnt = nbk - 1 - c; }   // column c: tiles (c+1..nbk-1, c); (c+1,c) carries (c+1,c+1)
            i = c + 1 + rem; merged = rem == 0;
        }
        CHOL_TRACE(0);
        // own tile(s) -> fragment-layout accumulators
        double c1[4][2], c2[4][2];
#pragma unroll
        for (int cb = 0; cb < 4; ++cb) { c1[cb][0] = c1[cb][1] = 0.0; c2[cb][0] = c2[cb][1] = 0.0; }
        if (tile_warp) {
#pragma unroll
            for (int cb = 0; cb < 4; ++cb) {
                const double2 v = __ldcg(reinterpret_cast<const double2*>(A + (size_t)(i * NB + 8 * w + fr) * npad + c * NB + 8 * cb + 2 * fc));
                c1[cb][0] = v.x; c1[cb][1] = v.y;
                if (merged) {
                    const double2 v2 = __ldcg(reinterpret_cast<const double2*>(A + (size_t)(i * NB + 8 * w + fr) * npad + i * NB + 8 * cb + 2 * fc));
                    c2[cb][0] = v2.x; c2[cb][1] = v2.y;
                }
            }
        }
        for (int k = 0; k < c; ++k) {
            bool ok = tile_wait(ready + i * nbk + k, epoch);
            ok = tile_wait(ready + c * nbk + k, epoch) && ok;
            tile_to_smem_ts(Pt, A, npad, i * NB, k * NB);
            tile_to_smem_ts(Qt, A, npad, c * NB, k * NB);
            if (!__syncthreads_and(ok)) { if (threadIdx.x == 0) atomicAdd(fail, 1000); return; }
            if (tile_warp) {
                tile_dmma_update(c1, Pt, Qt, lane, w, 4);
                if (merged) tile_dmma_update(c2, Pt, Pt, lane, w, w + 1);      // lower triangle of the diagonal tile
            }
            __syncthreads();
        }
        CHOL_TRACE(1);
        if (i != c) {
            // (i,c) -> Xs, row layout for the solver warp
            if (tile_warp) {
#pragma unroll
                for (int cb = 0; cb < 4; ++cb) *reinterpret_cast<double2*>(&Xs[8 * w + fr][8 * cb + 2 * fc]) = make_double2(c1[cb][0], c1[cb][1]);
            }
            __syncthreads();
            if (tile_warp) {
                // X L(c,c)^T = tile, consumed group by group as the factor streams in.  A cycle-stamped trace showed a single
                // solver warp (row per lane, all 32 columns: ~500 DFMA + ~500 LDS in one instruction stream, 4.3 us) falling behind
                // a factorisation that now takes ~2.5 us, so the four tile warps share it: row per lane in EVERY warp, warp w owns
                // the columns 4g+w (b[0] = column of the current group).  Per group: every warp posts its column of the group, ONE
                // barrier (which the loader warp below joins when the group has arrived), every warp solves the 4x4 block
                // for its row redundantly (10 FMAs) and applies the rank-4 update to its own <= 7 trailing columns.  After
                // the last group only the 4x4 solve is left on the chain.
                double (*exch)[PANEL_WARPS][NB] = reinterpret_cast<double (*)[PANEL_WARPS][NB]>(&LT[0][0]);     // [2][4][32], LT is idle here
                double b[NB / PANEL_WARPS];
#pragma unroll
                for (int p2 = 0; p2 < NB / PANEL_WARPS; ++p2) b[p2] = Xs[lane][PANEL_WARPS * p2 + w];
#pragma unroll 1
                for (int g = 0; g < NB / PANEL_WARPS; ++g) {
                    const int j0 = PANEL_WARPS * g;
                    exch[g & 1][w][lane] = b[0];
                    asm volatile("bar.sync %0, %1;" ::"r"(2 + g), "n"(CS_THREADS) : "memory");      // group g in Ls / invd (fifth warp) + every warp's column posted
                    const double i0 = invd[j0], i1 = invd[j0 + 1], i2 = invd[j0 + 2], i3 = invd[j0 + 3];
                    const double x0 = exch[g & 1][0][lane] * i0;
                    const double x1 = fma(-x0, Ls[j0 + 1][j0], exch[g & 1][1][lane]) * i1;
                    const double x2 = fma(-x1, Ls[j0 + 2][j0 + 1], fma(-x0, Ls[j0 + 2][j0], exch[g & 1][2][lane])) * i2;
                    const double x3 = fma(-x2, Ls[j0 + 3][j0 + 2], fma(-x1, Ls[j0 + 3][j0 + 1], fma(-x0, Ls[j0 + 3][j0], exch[g & 1][3][lane]))) * i3;
#pragma unroll
                    for (int p2 = 1; p2 < NB / PANEL_WARPS; ++p2) {
                        if (g + p2 < NB / PANEL_WARPS) {
                            const double* lr = &Ls[j0 + PANEL_WARPS * p2 + w][j0];          // row of this warp's column, broadcast
                            b[p2] = fma(-x3, lr[3], fma(-x2, lr[2], fma(-x1, lr[1], fma(-x0, lr[0], b[p2]))));
                        }
                    }
                    if (w == (g & (PANEL_WARPS - 1))) {
                        *reinterpret_cast<double2*>(&Xs[lane][j0]) = make_double2(x0, x1);
                        *reinterpret_cast<double2*>(&Xs[lane][j0 + 2]) = make_double2(x2, x3);
                    }
#pragma unroll
                    for (int p2 = 0; p2 < NB / PANEL_WARPS - 1; ++p2) b[p2] = b[p2 + 1];
                    // lookahead tile: (c+1,c+1) -= X_G X_G^T for the PREVIOUS group (in Xs since this group's barrier), one DMMA k-step,
                    // in the slack while the next group is on its way -- same k order as a whole-tile update, so the same bits
                    if (merged && g > 0) tile_dmma_update_k(c2, Xs, Xs, lane, w, w + 1, g - 1);
                }
                CHOL_TRACE(3);
            } else {
                // the fifth warp is the loader: it polls the LL lines of the groups in order and hands group g over with the group's
                // named barrier (ids 2..9).  The loads of the next LL_AHEAD groups are in flight while a group is handed over, so
                // that groups already written arrive one L2 round trip apart in total, not one round trip each.
                bool ok = true;
                uint4 q[LL_AHEAD][5];
#pragma unroll
                for (int g = 0; g < LL_AHEAD; ++g) ll_group_issue(q[g], ll, c, g, lane);
#pragma unroll
                for (int g = 0; g < NB / PANEL_WARPS; ++g) {
                    const int j0 = PANEL_WARPS * g;
                    uint4 (&d)[5] = q[g % LL_AHEAD];
                    if (!ll_group_ready(d, g, lane, epoch)) {
                        const long long t0 = clock64();
                        for (;;) {
                            ll_group_issue(d, ll, c, g, lane);
                            if (ll_group_ready(d, g, lane, epoch)) break;
                            if (clock64() - t0 > CF_TIMEOUT_CYCLES) { ok = false; break; }
                        }
                    }
                    __syncwarp();
                    if (g == 0) CHOL_TRACE_W4(2);
                    if (lane >= j0) { Ls[lane][j0] = ll_value(d[0]); Ls[lane][j0 + 1] = ll_value(d[1]); Ls[lane][j0 + 2] = ll_value(d[2]); Ls[lane][j0 + 3] = ll_value(d[3]); }
                    if (lane < PANEL_WARPS) invd[j0 + lane] = ll_value(d[4]);
                    // no fence before the arrive: it would wait for the loads in flight; bar.arrive synchronizes with the bar.sync
                    // of the same barrier (PTX memory model), which orders the shared-memory stores above for the solving warps
                    asm volatile("bar.arrive %0, %1;" ::"r"(2 + g), "n"(CS_THREADS) : "memory");
                    if (g + LL_AHEAD < NB / PANEL_WARPS) ll_group_issue(d, ll, c, g + LL_AHEAD, lane);
                }
                if (!ok) abort_flag = 1;
            }
            __syncthreads();                                        // X in Xs
            if (abort_flag) { if (threadIdx.x == 0) atomicAdd(fail, 1000); return; }
            if (tile_warp) {
                if (merged) tile_dmma_update_k(c2, Xs, Xs, lane, w, w + 1, NB / PANEL_WARPS - 1);       // the last group's k-step
#pragma unroll
                for (int u = 0; u < NB * NB / (2 * PANEL_WARPS * 32); ++u) {          // X -> A(i,c), coalesced
                    const int e = threadIdx.x + u * PANEL_WARPS * 32, r = e >> 4, q = (e & 15) * 2;
                    *reinterpret_cast<double2*>(A + (size_t)(i * NB + r) * npad + c * NB + q) = *reinterpret_cast<const double2*>(&Xs[r][q]);
                }
                // the stores of X are issued: the fifth warp publishes the tile (its fence stalls nobody); the tile warps only arrive
                asm volatile("bar.arrive 10, %0;" ::"n"(CS_THREADS) : "memory");
            } else {
                asm volatile("bar.sync 10, %0;" ::"n"(CS_THREADS) : "memory");
                if (lane == 0) tile_publish(ready + i * nbk + c, epoch);
                CHOL_TRACE_W4(4);
            }
        }
        if (i == c || merged) {
            // diagonal tile: fragment layout -> Pt (free since the update loop; Xs may still be read) -> phase-1 layout, factor;
            // the fifth warp streams the columns out
            if (tile_warp) {
#pragma unroll
                for (int cb = 0; cb < 4; ++cb) {
                    const double v0 = merged ? c2[cb][0] : c1[cb][0], v1 = merged ? c2[cb][1] : c1[cb][1];
                    *reinterpret_cast<double2*>(&Pt[8 * w + fr][8 * cb + 2 * fc]) = make_double2(v0, v1);
                }
                chol_factor_barrier();
                CHOL_TRACE(7);
                double col[NB / (4 * PANEL_WARPS)][4];
#pragma unroll
                for (int q = 0; q < NB / (4 * PANEL_WARPS); ++q) {
                    const double2 v = *reinterpret_cast<const double2*>(&Pt[lane][4 * PANEL_WARPS * q + 4 * w]);
                    const double2 v2 = *reinterpret_cast<const double2*>(&Pt[lane][4 * PANEL_WARPS * q + 4 * w + 2]);
                    col[q][0] = v.x; col[q][1] = v.y; col[q][2] = v2.x; col[q][3] = v2.y;
                }
                const bool bad = chol_tile_factor4(col, LT, invd, lane, w, i * NB, n, &bad_flag);
                if (bad && threadIdx.x == 0) atomicAdd(fail, 1);
                CHOL_TRACE(5);
            } else {
#pragma unroll 1
                for (int g = 0; g < NB / PANEL_WARPS; ++g) {
                    asm volatile("bar.sync %0, 64;" ::"r"(2 + g) : "memory");         // group g of the factor is in Ls / invd
                    uint4* grp = ll + ((size_t)i * (NB / PANEL_WARPS) + g) * CHOL_LL_GROUP;
                    if (lane >= PANEL_WARPS * g) {
                        // rows above the diagonal inside the quad's 4x4 block hold round-off (chol_tile_factor4): store zeros
                        const int rr = lane - PANEL_WARPS * g;
                        const double v0 = LT[PANEL_WARPS * g][lane], v1 = rr >= 1 ? LT[PANEL_WARPS * g + 1][lane] : 0.0,
                                     v2 = rr >= 2 ? LT[PANEL_WARPS * g + 2][lane] : 0.0, v3 = rr >= 3 ? LT[PANEL_WARPS * g + 3][lane] : 0.0;
                        ll_store(grp + lane, v0, epoch); ll_store(grp + NB + lane, v1, epoch); ll_store(grp + 2 * NB + lane, v2, epoch); ll_store(grp + 3 * NB + lane, v3, epoch);
                        double* dst = A + (size_t)(i * NB + lane) * npad + i * NB + PANEL_WARPS * g;       // for the back substitution (after the kernel)
                        *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
                        *reinterpret_cast<double2*>(dst + 2) = make_double2(v2, v3);
                    }
                    if (lane < PANEL_WARPS) {
                        const double iv = invd[PANEL_WARPS * g + lane];
                        ll_store(grp + 4 * NB + lane, iv, epoch);
                        dinv[i * NB + PANEL_WARPS * g + lane] = iv;
                    }
                }
                CHOL_TRACE_W4(6);
                if (Linv) {             // off the critical path: L(i,i)^-1 (row-major) for the back substitution.  X L^T = I, X = L^-T
                    double b[NB];
#pragma unroll
                    for (int q = 0; q < NB; ++q) b[q] = lane == q ? 1.0 : 0.0;
                    chol_tile_trsm_t(b, LT, invd);
#pragma unroll
                    for (int q = 0; q < NB; ++q) Linv[((size_t)i * NB + q) * NB + lane] = b[q];      // Linv[q][lane] = X[lane][q]
                }
            }
        }
        __syncthreads();                                            // shared memory is reused by the next task
    }
#undef CHOL_TRACE
#undef CHOL_TRACE_W4
}

// Back substitution L^T x = y with y = row n of the factored matrix, on one CTA of 640 threads (warp 0 + 608 workers); the
// kernel for systems too large for the cluster kernel below.  Per 32-block (descending) warp 0 produces the block's unknowns
// by multiplying with L(kb,kb)^-1 (written by the dataflow factorisation, off its critical path) -- one 32-term dot product
// per lane instead of 32 dependent shuffle/FMA steps -- then worker c subtracts  sum_m L[kb*32+m][c] x_m  from y[c] for the
// columns to the left.
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"(d), "l"(gsrc) : "memory");
}
__host__ __device__ inline size_t chol_backsolve_smem(int npad) { return sizeof(double) * (size_t)npad; }

__global__ void __launch_bounds__(640) chol_backsolve_kernel(const double* __restrict__ A, const double* __restrict__ Linv,
                                                             int npad, int n, double* __restrict__ x, const int* __restrict__ skip = nullptr) {
    if (skip && *skip) return;
    extern __shared__ double sm[];
    double* y = sm;                               // [npad]
    const int tid = threadIdx.x, lane = tid & 31, nworkers = blockDim.x - 32, c0 = tid - 32;
    const bool solver = tid < 32;
    const int kb_first = (n - 1) / NB;
    for (int i = tid; i < npad; i += blockDim.x) y[i] = i < n ? A[(size_t)n * npad + i] : 0.0;
    __syncthreads();
    for (int kb = kb_first; kb >= 0; --kb) {
        const int ncols = kb * NB;                // columns to the left of the diagonal tile
        const bool has = !solver && c0 < ncols;
        // one register array, two roles: warp 0 -> column `lane` of L(kb,kb)^-1 (row-major); worker c0 -> its column of the block row
        double reg[NB];
#pragma unroll
        for (int m = 0; m < NB; ++m) reg[m] = solver ? Linv[((size_t)kb * NB + m) * NB + lane] : A[(size_t)(kb * NB + m) * npad + (has ? c0 : 0)];
        if (solver) {                             // x_r = sum_c Linv[c][r] y_c   (Linv lower triangular: exact zeros for c < r)
            double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
#pragma unroll
            for (int c = 0; c < NB; c += 4) {
                s0 = fma(reg[c], y[kb * NB + c], s0); s1 = fma(reg[c + 1], y[kb * NB + c + 1], s1);
                s2 = fma(reg[c + 2], y[kb * NB + c + 2], s2); s3 = fma(reg[c + 3], y[kb * NB + c + 3], s3);
            }
            __syncwarp();
            y[kb * NB + lane] = (s0 + s1) + (s2 + s3);
        }
        __syncthreads();
        if (has) {
            double s0 = 0, s1 = 0;
#pragma unroll
            for (int m = 0; m < NB; m += 2) { s0 = fma(reg[m], y[kb * NB + m], s0); s1 = fma(reg[m + 1], y[kb * NB + m + 1], s1); }
            y[c0] -= s0 + s1;
        }
        if (!solver) {
            for (int c = c0 + nworkers; c < ncols; c += nworkers) {       // n > 640 only
                double s = 0;
#pragma unroll 8
                for (int m = 0; m < NB; ++m) s = fma(A[(size_t)(kb * NB + m) * npad + c], y[kb * NB + m], s);
                y[c] -= s;
            }
        }
        __syncthreads();
    }
    for (int i = tid; i < n; i += blockDim.x) x[i] = y[i];
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// Back substitution on a thread-block CLUSTER, for every system whose slices fit (chol_backsolve_cluster_smem / _threads).  One
// CTA that stages every block row (32 x n doubles) in its shared memory is bound by that SM's shared-memory bandwidth, ~2 us
// per 32 unknowns.  Here BS_CLUSTER CTAs on BS_CLUSTER SMs share the columns -- CTA r owns the 32-column blocks b with
// b mod BS_CLUSTER = r: their part of y, their slice of every block row (staged with cp.async, each thread into its own
// slots, so the L2 round trip leaves the chain), and the solve of those blocks.  Per step the CTA that owns block kb turns y_kb into x_kb with the inverse tile (one 32-term dot product
// per lane) and pushes the 32 values into every CTA's shared memory with st.async, which signals that CTA's mbarrier for the step
// (complete_tx; armed locally with expect_tx = 256 bytes); every CTA waits on its own mbarrier and subtracts the block row's
// contribution from its columns (slices staged TWO steps ahead: the L2 latency of a block row exceeds a step).  No cluster-wide barrier inside the loop: one DSMEM hop (~215 cycles) per step.
// Slots (x block + mbarrier) are indexed kb mod BS_CLUSTER: a CTA solves one of any BS_CLUSTER consecutive blocks, so no CTA can
// be more than BS_CLUSTER - 1 steps ahead of another and a slot is never overwritten while somebody still reads it.
// ---------------------------------------------------------------------------------------------------------------
constexpr int BS_CLUSTER = 8;
__host__ __device__ inline int chol_backsolve_cluster_threads(int n) { const int nb = (n - 1) / NB + 1; return 32 + 32 * ((nb + BS_CLUSTER - 1) / BS_CLUSTER); }
__host__ __device__ inline size_t chol_backsolve_cluster_smem(int n) {
    const size_t nwork = (size_t)chol_backsolve_cluster_threads(n) - 32;
    return sizeof(double) * ((size_t)BS_CLUSTER * NB + (size_t)NB * NB + nwork + 2 * (size_t)NB * nwork);
}
__device__ __forceinline__ unsigned bs_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned bs_mapa(unsigned addr, unsigned rank) { unsigned r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank)); return r; }
__device__ __forceinline__ bool bs_mbar_try_wait(unsigned addr, unsigned parity) {
    unsigned ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    return ok != 0;
}
__global__ void __cluster_dims__(BS_CLUSTER, 1, 1) __launch_bounds__(512)
chol_backsolve_cluster_kernel(const double* __restrict__ A, const double* __restrict__ Linv, int npad, int n, double* __restrict__ x,
                              int* __restrict__ fail, const int* __restrict__ skip = nullptr) {
    if (skip && *skip) return;                    // the same flag for every CTA of the cluster
    extern __shared__ double sm[];
    __shared__ __align__(8) unsigned long long mbar[BS_CLUSTER];
    const int tid = threadIdx.x, lane = tid & 31, nwork = blockDim.x - 32, t = tid - 32;
    const bool solver = tid < 32;
    unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    const int kb_first = (n - 1) / NB;
    double* xb = sm;                              // [BS_CLUSTER][NB]   x blocks as they arrive
    double* dstage = xb + BS_CLUSTER * NB;        // [NB][NB]           inverse tile of the next block this CTA solves
    double* yl = dstage + NB * NB;                // [nwork]            y of the own columns
    double* stage = yl + nwork;                   // [2][NB][nwork]     own slices of the next two block rows (buffer kb & 1)
    const int blk = (int)r + (t >> 5) * BS_CLUSTER, col = blk * NB + (t & 31);      // worker t's column
    const bool own = !solver && blk <= kb_first;
    auto arm = [&](int slot) {                    // one local arrival + the 256 bytes of an x block complete a phase
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bs_smem_u32(&mbar[slot])), "r"(NB * 8) : "memory");
    };
    if (tid == 0) {
#pragma unroll
        for (int j = 0; j < BS_CLUSTER; ++j) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bs_smem_u32(&mbar[j])) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int j = 0; j < BS_CLUSTER && j <= kb_first; ++j) arm((kb_first - j) % BS_CLUSTER);      // first use of every slot
    }
    auto issue_row = [&](int kb) {                // worker: its column of block row kb -> stage buffer kb & 1
        if (own && blk < kb) {
            double* dst = stage + (size_t)(kb & 1) * NB * nwork + t;
#pragma unroll
            for (int m = 0; m < NB; ++m) cp_async8(dst + (size_t)m * nwork, A + (size_t)(kb * NB + m) * npad + col);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    auto issue_tile = [&](int kb) {               // solver warp: column `lane` of L(kb,kb)^-1 (row-major)
        if (kb >= 0) {
#pragma unroll
            for (int m = 0; m < NB; ++m) cp_async8(dstage + m * NB + lane, Linv + ((size_t)kb * NB + m) * NB + lane);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    if (solver) issue_tile(kb_first - ((kb_first - (int)r) % BS_CLUSTER + BS_CLUSTER) % BS_CLUSTER);
    else { issue_row(kb_first); issue_row(kb_first - 1); }
    if (own) yl[t] = col < n ? A[(size_t)n * npad + col] : 0.0;
    __syncthreads();
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    bool ok = true;
    for (int kb = kb_first; kb >= 0; --kb) {
        const int slot = kb % BS_CLUSTER;
        const unsigned parity = (unsigned)((kb_first - kb) / BS_CLUSTER) & 1u;
        const bool active = own && blk < kb;
        double reg[NB];
        if (!solver) {
            asm volatile("cp.async.wait_group 1;" ::: "memory");         // block row kb has landed (row kb-1 may still be in flight)
            if (active) {
                const double* src = stage + (size_t)(kb & 1) * NB * nwork + t;
#pragma unroll
                for (int m = 0; m < NB; ++m) reg[m] = src[(size_t)m * nwork];
            }
            issue_row(kb - 2);                                           // into the buffer just read (own slots only)
        } else if ((int)r == slot) {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            const double* yk = yl + ((kb - (int)r) / BS_CLUSTER) * NB;
            double s0 = 0, s1 = 0, s2 = 0, s3 = 0;      // x_r = sum_c Linv[c][r] y_c   (Linv lower triangular: exact zeros for c < r)
#pragma unroll
            for (int c = 0; c < NB; c += 4) {
                s0 = fma(dstage[c * NB + lane], yk[c], s0); s1 = fma(dstage[(c + 1) * NB + lane], yk[c + 1], s1);
                s2 = fma(dstage[(c + 2) * NB + lane], yk[c + 2], s2); s3 = fma(dstage[(c + 3) * NB + lane], yk[c + 3], s3);
            }
            const double xv = (s0 + s1) + (s2 + s3);
            const unsigned xa = bs_smem_u32(xb + slot * NB + lane), ma = bs_smem_u32(&mbar[slot]);
#pragma unroll
            for (unsigned p = 0; p < BS_CLUSTER; ++p)                    // the store itself signals the peer's mbarrier (complete_tx, 8 bytes)
                asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b64 [%0], %1, [%2];"
                             :: "r"(bs_mapa(xa, p)), "l"(__double_as_longlong(xv)), "r"(bs_mapa(ma, p)) : "memory");
            if (kb * NB + lane < n) x[kb * NB + lane] = xv;
            __syncwarp();                          // every lane is done with dstage
            issue_tile(kb - BS_CLUSTER);
        }
        {   // everybody waits for x_kb (every thread on every step: the parity of a slot is only meaningful in order)
            const unsigned ma = bs_smem_u32(&mbar[slot]);
            if (!bs_mbar_try_wait(ma, parity)) {
                const long long t0 = clock64();
                while (!bs_mbar_try_wait(ma, parity)) if (clock64() - t0 > CF_TIMEOUT_CYCLES) { ok = false; break; }
            }
            if (tid == 0 && kb - BS_CLUSTER >= 0) arm(slot);             // this phase is complete: arm the slot's next use
        }
        if (active) {
            const double* xk = xb + slot * NB;
            double s0 = 0, s1 = 0, s2 = 0, s3 = 0;
#pragma unroll
            for (int m = 0; m < NB; m += 4) {
                s0 = fma(reg[m], xk[m], s0); s1 = fma(reg[m + 1], xk[m + 1], s1); s2 = fma(reg[m + 2], xk[m + 2], s2); s3 = fma(reg[m + 3], xk[m + 3], s3);
            }
            yl[t] -= (s0 + s1) + (s2 + s3);
        }
        if (!__syncthreads_and(ok)) { if (tid == 0) atomicAdd(fail, 1000); break; }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    // nobody leaves while a peer may still push into its shared memory
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
