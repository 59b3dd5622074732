// fused2d_wpair.cuh -- TWO consecutive analysis levels of the 2-D transform in one kernel, built from
// independent warps (float32, even filter length <= 8).
//
// Replaces two turns of the reference's level loop (src/ptwt/conv_transform_2.py:142-149:
// F.pad -> conv2d(4 x [L x L], stride 2) -> split, with res_ll fed back) without writing the first
// level's approximation band to HBM: with one launch per level that band makes a round trip
// (+25 % traffic at the first level, 1.33x over the whole pyramid).
//
// Structure (no CTA-wide barrier anywhere; a CTA is ONE warp; adjacent strips form a cluster that passes a split
// cluster barrier once per group, so that they stream their rows in step):
//   * a warp owns a strip of 128 level-1 columns (lane <-> 4 adjacent columns) and a segment of rows
//     and marches down it; input rows arrive by TMA (cp.async.bulk.tensor, 8-byte elements so that
//     the 264-sample rows fit one box) in groups of 4 rows into a private 3-stage ring, completion on
//     the warp's own mbarriers; the warp that consumed a stage re-arms it;
//   * row pass: each lane slides the L taps over its 16-sample window (4 LDS.128 per row);
//   * column pass WITHOUT a shared-memory ring: every pair of input rows is scattered into the L/2
//     output rows it contributes to, held as paired (float2) accumulators in registers
//     (acc[i] += dec[2(i-k)+1] * row[2k] + dec[2(i-k)] * row[2k+1]); one output row completes per
//     pair and goes straight to HBM (three detail bands, 128-bit stores, 512 contiguous bytes/warp);
//   * the completed approximation row goes to a two-row buffer in shared memory (the only exchange
//     between lanes); level 2 reads it back with lane <-> 2 level-2 columns, runs the same row pass
//     and keeps the row-filtered lines in an 8-row ring; its column pass gathers the L ring rows of
//     one output row (no level-2 state in registers, one copy of the code) and stores the four bands;
//   * boundary extension: out-of-range input samples are patched into the staged tile from the
//     extension source (all modes but periodic; zero fill is TMA's out-of-bounds fill); the level-2
//     extension of the approximation band is served from the ring (rows) and by patching the ring
//     rows of the edge strips (columns), so level 2 sees exactly ext(cA1) like the reference.
//
// Horizontal halo: a strip computes HL1 extra approximation columns on its left (6 % redundant
// arithmetic, the re-read input columns hit L2); vertical halo: a segment restarts both levels
// (3 (L/2-1) row pairs + L-2 approximation rows).
//
// Algorithmic bytes: 4 B * (H*W read + 3*Mh1*Mw1 + 4*Mh2*Mw2 written).
#pragma once

#include "fused2d.cuh"

namespace wtb {

constexpr int WPAIR_MAXSEG = 48;

struct WPairParams {
    const float* x;            // level input [batch, H, W]
    int64_t x_bs, x_rs;
    float* d1;                 // first-level detail bands: k = 1, 2, 3 at d1 + (k-1) * d1_band
    int64_t d1_bs, d1_rs, d1_band;
    float* o2[4];              // second-level bands k = 0 (approximation), 1, 2, 3
    int64_t o2_bs[4], o2_rs[4];
    int H, W, Mh1, Mw1, Mh2, Mw2;
    int mode, batch0;
    int nseg;
    int seg_start[WPAIR_MAXSEG + 1];   // second-level row ranges [seg_start[i], seg_start[i+1]), longest first
    float2 pl[4], ph[4];       // row pass: {dec[L-1-2q], dec[L-2-2q]}
    float2 vl[8], vh[8];       // column pass: {dec[m], dec[m]}
};

template <int L, int NSTG_ = 3>
struct WPairGeom {
    static constexpr int HALO = L - 2, NA = L / 2;
    static constexpr int HAL = (HALO + 3) / 4 * 4;          // left halo of the staged tile, 16-byte aligned
    static constexpr int OFF1 = HAL - HALO;
    static constexpr int HL1 = HAL;                         // approximation columns left of the owned ones
    static constexpr int OFF2 = HL1 - HALO;
    static constexpr int TW1 = 128;                         // level-1 columns per strip (4 per lane)
    static constexpr int TW2 = (TW1 - HL1) / 2;             // level-2 columns owned by a strip
    static constexpr int NV1 = OFF1 + L + 6, NV1_4 = (NV1 + 3) / 4;
    static constexpr int TILE_W = 8 * 31 + 4 * NV1_4;       // staged input columns
    static constexpr int NV2 = OFF2 + L + 2, NV2_4 = (NV2 + 3) / 4;
    static constexpr int RP1 = TW1;                         // pitch of the two approximation row buffers (the windows of
                                                            // lanes >= TW2/2 run into the ring behind them: don't-care)
    static constexpr int R2P = 128;                         // ring row: 64 low-pass | 64 high-pass row-filtered samples
    static constexpr int RING = 8;                          // >= L rows (the window of one output; boundary sources)
    static constexpr int ROWS = 4, NSTG = NSTG_;
    static constexpr int STAGE_BYTES = ROWS * TILE_W * 4;
    static constexpr int STAGE_STRIDE = (STAGE_BYTES + 127) / 128 * 128;
    static constexpr int SMEM = NSTG * STAGE_STRIDE + 2 * RP1 * 4 + RING * R2P * 4 + 8 * NSTG;
    static_assert(L % 2 == 0 && L >= 2 && L <= 8, "wpair kernel: even filter length <= 8");
    static_assert(TILE_W % 4 == 0 && TILE_W / 2 <= 256, "tile row must fit one TMA box of 8-byte elements");
    static_assert(RING >= L, "ring too small for the window of one output row");
};

// split cluster barrier (a CTA launched without a cluster is a cluster of one)
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.aligned;" ::: "memory"); }

// lo[c], hi[c] for NC consecutive outputs from the register window w (see row_filter)
template <int L, int NC, int OFF, int NW>
__device__ __forceinline__ void wp_rowfilt(const float (&w)[NW], const float2* __restrict__ pl,
                                           const float2* __restrict__ ph, float (&lo)[NC], float (&hi)[NC]) {
#pragma unroll
    for (int c = 0; c < NC; ++c) {
        float2 a = make_float2(0.f, 0.f), h = make_float2(0.f, 0.f);
#pragma unroll
        for (int q = 0; q < L / 2; ++q) {
            const float2 x = make_float2(w[2 * c + 2 * q + OFF], w[2 * c + 2 * q + OFF + 1]);
            a = ffma2(pl[q], x, a);
            h = ffma2(ph[q], x, h);
        }
        lo[c] = a.x + a.y;
        hi[c] = h.x + h.y;
    }
}

// Scatter one pair of row-filtered rows (index 0: even row 2k, 1: odd row 2k+1) into the L/2 output rows
// k .. k+L/2-1 it contributes to.  Slot s completes with this pair, slot (s + L/2 - 1) % (L/2) starts.
// acc[slot][band][column pair]; band = 0: lo_H lo_W, 1: lo_H hi_W, 2: hi_H lo_W, 3: hi_H hi_W.
// s must be a compile-time constant after unrolling (the accumulators live in registers).
template <int L, int NCP>
__device__ __forceinline__ void wp_scatter(float2 (&acc)[L / 2][4][NCP], const float2 (&lo)[2][NCP],
                                           const float2 (&hi)[2][NCP], const WPairParams& p, const int s) {
    constexpr int NA = L / 2;
#pragma unroll
    for (int d = 0; d < NA; ++d) {
        const int slot = (s + d) % NA;
        const float2 tl0 = p.vl[2 * d + 1], tl1 = p.vl[2 * d], th0 = p.vh[2 * d + 1], th1 = p.vh[2 * d];
#pragma unroll
        for (int cp = 0; cp < NCP; ++cp) {
            const float2 z = make_float2(0.f, 0.f);
            const float2 a0 = d == NA - 1 ? z : acc[slot][0][cp], a1 = d == NA - 1 ? z : acc[slot][1][cp];
            const float2 a2 = d == NA - 1 ? z : acc[slot][2][cp], a3 = d == NA - 1 ? z : acc[slot][3][cp];
            acc[slot][0][cp] = ffma2(tl1, lo[1][cp], ffma2(tl0, lo[0][cp], a0));
            acc[slot][1][cp] = ffma2(tl1, hi[1][cp], ffma2(tl0, hi[0][cp], a1));
            acc[slot][2][cp] = ffma2(th1, lo[1][cp], ffma2(th0, lo[0][cp], a2));
            acc[slot][3][cp] = ffma2(th1, hi[1][cp], ffma2(th0, hi[0][cp], a3));
        }
    }
}

// Row pass + scatter of one level-1 step: rows tr, tr + TILE_W of the staged tile (lane window)
template <int L>
__device__ __forceinline__ void wp_l1_compute(const float* __restrict__ tr, float2 (&acc)[L / 2][4][2],
                                              const WPairParams& p, const int s) {
    using Gm = WPairGeom<L>;
    float2 lo[2][2], hi[2][2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float w[4 * Gm::NV1_4];
#pragma unroll
        for (int q = 0; q < Gm::NV1_4; ++q) {
            const float4 t = *reinterpret_cast<const float4*>(tr + r * Gm::TILE_W + 4 * q);
            w[4 * q] = t.x; w[4 * q + 1] = t.y; w[4 * q + 2] = t.z; w[4 * q + 3] = t.w;
        }
        float l4[4], h4[4];
        wp_rowfilt<L, 4, Gm::OFF1>(w, p.pl, p.ph, l4, h4);
        lo[r][0] = make_float2(l4[0], l4[1]); lo[r][1] = make_float2(l4[2], l4[3]);
        hi[r][0] = make_float2(h4[0], h4[1]); hi[r][1] = make_float2(h4[2], h4[3]);
    }
    wp_scatter<L, 2>(acc, lo, hi, p, s);
}

template <int L, int NSTG, int MINB>
__global__ void __launch_bounds__(32, MINB)
fwd2d_wpair_kernel(const __grid_constant__ WPairParams p, const __grid_constant__ CUtensorMap tmap) {
    using Gm = WPairGeom<L, NSTG>;
    constexpr int HALO = Gm::HALO, NA = Gm::NA, HAL = Gm::HAL, HL1 = Gm::HL1, TW1 = Gm::TW1, TW2 = Gm::TW2;
    constexpr int TILE_W = Gm::TILE_W, RP1 = Gm::RP1, R2P = Gm::R2P, RING = Gm::RING, ROWS = Gm::ROWS;
    constexpr int STG_F = Gm::STAGE_STRIDE / 4;
    constexpr int UNR = (NA & 1) ? NA : (NA / 2 > 0 ? NA / 2 : 1);   // groups per unrolled block: whole slot rotations

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_tile = reinterpret_cast<float*>(smem_raw);                              // [NSTG][ROWS][TILE_W]
    float* s_row = reinterpret_cast<float*>(smem_raw + NSTG * Gm::STAGE_STRIDE);     // [2][RP1] approximation rows
    float* s_ring = s_row + 2 * RP1;                                                 // [RING][R2P] row-filtered lines
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_ring + RING * R2P);

    const int lane = threadIdx.x;
    const int b = p.batch0 + blockIdx.y;

    // ---- strip -------------------------------------------------------------------------------------
    const int X0n = blockIdx.x * TW2;                 // nominal first owned level-2 column
    int X0 = X0n;
    {   // every extension source of the approximation columns level 2 reads must lie inside the strip:
        // the right-most strip is shifted left when needed (it still stores its nominal columns only)
        const int lim = (p.Mw1 - L + HL1) / 2;
        if (X0 > lim) X0 = max(lim & ~1, 0);
    }
    const int cA0 = 2 * X0 - HL1;                     // first approximation column computed (multiple of 4)
    const int c_in0 = 2 * cA0 - HAL;                  // first staged input column (multiple of 4)
    const int own1_lo = 2 * X0n, own1_hi = min(2 * (X0n + TW2), p.Mw1);
    const int own2_lo = X0n, own2_hi = min(X0n + TW2, p.Mw2);

    // ---- segment (long segments come first in the grid, the short ones fill the tail) ---------------
    const int Y0 = p.seg_start[blockIdx.z], Y1 = p.seg_start[blockIdx.z + 1];
    // Approximation rows [a_start, a_end) are computed here (a_start = -1 is a dummy row that is never written).
    // The first row is chosen such that every TMA group completes an (even, odd) pair of rows -- the window of a
    // level-2 output row ends on an odd row, so level 2 runs once per group -- and such that the bottom extension
    // sources (the last RING rows) are included even when the segment is short.
    int a_start = 2 * Y0 - HALO - ((NA - 1) & 1);
    {
        int amax = p.Mh1 - RING;
        if ((amax - (NA - 1)) & 1) --amax;
        a_start = max(min(a_start, amax), -((NA - 1) & 1));
    }
    const int a_end = min(p.Mh1, 2 * Y1);
    const int a_lo = max(a_start, 0);                 // first row really written
    const int n1 = a_end - a_start + NA - 1;          // level-1 steps (pairs of input rows)
    const int ngroups = (n1 + 1) / 2;                 // TMA groups of 4 input rows
    const int r_in0 = 2 * a_start - HALO;             // first staged input row

    if (lane == 0) {
        tma_prefetch_desc(&tmap);
#pragma unroll
        for (int s = 0; s < NSTG; ++s) mbar_init(&bars[s], 1);
        fence_mbar_init();
    }
    __syncwarp();
    if (lane == 0) {
        for (int s = 0; s < NSTG && s < ngroups; ++s) {
            mbar_expect_tx(&bars[s], (uint32_t)Gm::STAGE_BYTES);
            tma_load_3d(s_tile + s * STG_F, &tmap, &bars[s], c_in0 / 2, r_in0 + s * ROWS, b);
        }
    }

    const float* __restrict__ xb = p.x + (int64_t)b * p.x_bs;
    const bool need_patch = (p.mode != WT_MODE_ZERO) || (p.W & 1);
    const bool edge_in = need_patch && (c_in0 < 0 || c_in0 + TILE_W > p.W);   // warp-uniform
    const bool edge_a = cA0 < 0 || cA0 + TW1 > p.Mw1;                         // warp-uniform
    // Column patch of the edge strips' staged rows (rows in range): the L samples next to each border are all any valid
    // output reads.  The same for every row and group: lane q < (at most 2L) patches position cp_t of each staged row
    // from position cp_s of the same row (-1: zero).  The sources are in-range samples, normally staged in the tile
    // already, so the patch is a shared-memory copy; a global-memory round trip in every group of the edge strips
    // would hold back their whole cluster (the cluster barrier waits for its slowest strip).  When a source lies outside
    // the tile, the whole warp reads its sources from global memory instead.
    int cp_t = -1, cp_s = -1;
    bool cpatch_staged = true;
    if (edge_in) {
        const int nl = c_in0 < 0 ? -c_in0 : 0;
        const int l0 = max(nl - L, 0);
        const int r0 = min(max(p.W - c_in0, 0), TILE_W), r1 = min(r0 + L, TILE_W);
        const int wl = nl - l0, wb = wl + (r1 - r0);
        bool staged = true;
        if (lane < wb) {   // wb <= 2L <= 32
            cp_t = lane < wl ? l0 + lane : r0 + (lane - wl);
            const int sc = ext_index32(c_in0 + cp_t, p.W, p.mode);
            cp_s = sc < 0 ? -1 : sc - c_in0;   // an in-range column: never a patched position
            staged = sc < 0 || (cp_s >= 0 && cp_s < TILE_W);
        }
        cpatch_staged = __all_sync(0xffffffffu, staged);
    }

    // level-1 stores: this lane's 4 columns, running pointer = row `produced` of band 1
    const int col1 = cA0 + 4 * lane;
    const bool store1 = col1 >= own1_lo && col1 < own1_hi;
    float* const pd1 = p.d1 + (int64_t)b * p.d1_bs + (int64_t)a_start * p.d1_rs + col1;
    // level-2 stores: this lane's 2 columns, running pointers = row K2 of the four bands
    const int col2 = X0 + 2 * lane;
    const bool store2 = col2 >= own2_lo && col2 < own2_hi;
    float* po2[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) po2[k] = p.o2[k] + (int64_t)b * p.o2_bs[k] + (int64_t)Y0 * p.o2_rs[k] + col2;
    // patch table of the edge strips: source index (within the approximation row) of each out-of-range column
    int psrc[4] = {-2, -2, -2, -2};
    if (edge_a) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int col = col1 + j;
            if (col < 0 || col >= p.Mw1) {
                const int s = ext_index32(col, p.Mw1, p.mode);
                psrc[j] = (s >= cA0 && s < cA0 + TW1) ? s - cA0 : -1;
            }
        }
    }

    float2 acc1[NA][4][2];
#pragma unroll
    for (int s = 0; s < NA; ++s)
#pragma unroll
        for (int k = 0; k < 4; ++k) { acc1[s][k][0] = make_float2(0.f, 0.f); acc1[s][k][1] = make_float2(0.f, 0.f); }

    int K2 = Y0;                       // next level-2 output row
    int produced = a_lo;               // approximation rows [.., produced) are in the ring
    int stage = 0;
    uint32_t par = 0;
    float* const row_lane = s_row + 4 * lane;
    float* const ring_lane = s_ring + 2 * lane;

    for (int g0 = 0; g0 < ngroups; g0 += UNR) {
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            const int g = g0 + u;
            if (g >= ngroups) break;
            // Adjacent strips of one segment form a cluster and march in step, at most one group apart: their
            // row pieces then reach DRAM together as long contiguous runs.  Left to drift apart, the same
            // traffic streams at about 2.1 instead of 2.7 TB/s on an H100 (tools/time_wpair_ceiling.py).
            if (g > 0) cluster_wait();
            float* tile = s_tile + stage * STG_F;
            mbar_wait(&bars[stage], par);
            const int rbase = r_in0 + g * ROWS;

            // ---- boundary extension of the staged input -------------------------------------------------
            if (need_patch) {
                const bool rows_oob = rbase < 0 || rbase + ROWS > p.H;
                if (rows_oob) {
                    for (int idx = lane; idx < ROWS * TILE_W; idx += 32) {
                        const int rr = idx / TILE_W, t = idx - rr * TILE_W;
                        const int r = rbase + rr, c = c_in0 + t;
                        if (r < 0 || r >= p.H || c < 0 || c >= p.W) {
                            const int sr = ext_index32(r, p.H, p.mode), sc = ext_index32(c, p.W, p.mode);
                            tile[idx] = (sr >= 0 && sc >= 0) ? __ldg(xb + (int64_t)sr * p.x_rs + sc) : 0.f;
                        }
                    }
                    __syncwarp();
                } else if (edge_in) {
                    if (cpatch_staged) {
                        if (cp_t >= 0) {
#pragma unroll
                            for (int rr = 0; rr < ROWS; ++rr)
                                tile[rr * TILE_W + cp_t] = cp_s >= 0 ? tile[rr * TILE_W + cp_s] : 0.f;
                        }
                    } else if (cp_t >= 0) {
                        const int sc = ext_index32(c_in0 + cp_t, p.W, p.mode);
                        for (int rr = 0; rr < ROWS; ++rr)
                            tile[rr * TILE_W + cp_t] = sc >= 0 ? __ldg(xb + (int64_t)(rbase + rr) * p.x_rs + sc) : 0.f;
                    }
                    __syncwarp();
                }
            }

            // ---- level 1: two steps = one (even, odd) pair of approximation rows, straight-line code; accumulator
            //      slots are compile-time constants, row validity only predicates the stores -------------------------
            const int a0 = a_start + 2 * g - (NA - 1);             // rows completed by the two steps: a0 (even), a0 + 1
            {
                const int sl0 = (2 * u) % NA, sl1 = (2 * u + 1) % NA;
                const float* tl = tile + 8 * lane;
                wp_l1_compute<L>(tl, acc1, p, sl0);
                const bool v0 = a0 >= a_lo && a0 < a_end;
                const bool v1 = a0 + 1 >= a_lo && a0 + 1 < a_end;
                float* rrow0 = row_lane + (a0 & 1) * RP1;
                float* rrow1 = row_lane + ((a0 + 1) & 1) * RP1;
                float* pdA = pd1 + (int64_t)(a0 - a_start) * p.d1_rs;
                if (v0) {
                    *reinterpret_cast<float4*>(rrow0) =
                        make_float4(acc1[sl0][0][0].x, acc1[sl0][0][0].y, acc1[sl0][0][1].x, acc1[sl0][0][1].y);
                    if (store1 && a0 >= 2 * Y0) {
                        *reinterpret_cast<float4*>(pdA) =
                            make_float4(acc1[sl0][1][0].x, acc1[sl0][1][0].y, acc1[sl0][1][1].x, acc1[sl0][1][1].y);
                        *reinterpret_cast<float4*>(pdA + p.d1_band) =
                            make_float4(acc1[sl0][2][0].x, acc1[sl0][2][0].y, acc1[sl0][2][1].x, acc1[sl0][2][1].y);
                        *reinterpret_cast<float4*>(pdA + 2 * p.d1_band) =
                            make_float4(acc1[sl0][3][0].x, acc1[sl0][3][0].y, acc1[sl0][3][1].x, acc1[sl0][3][1].y);
                    }
                }
                wp_l1_compute<L>(tl + 2 * TILE_W, acc1, p, sl1);
                if (v1) {
                    *reinterpret_cast<float4*>(rrow1) =
                        make_float4(acc1[sl1][0][0].x, acc1[sl1][0][0].y, acc1[sl1][0][1].x, acc1[sl1][0][1].y);
                    if (store1 && a0 + 1 >= 2 * Y0) {
                        float* pdB = pdA + p.d1_rs;
                        *reinterpret_cast<float4*>(pdB) =
                            make_float4(acc1[sl1][1][0].x, acc1[sl1][1][0].y, acc1[sl1][1][1].x, acc1[sl1][1][1].y);
                        *reinterpret_cast<float4*>(pdB + p.d1_band) =
                            make_float4(acc1[sl1][2][0].x, acc1[sl1][2][0].y, acc1[sl1][2][1].x, acc1[sl1][2][1].y);
                        *reinterpret_cast<float4*>(pdB + 2 * p.d1_band) =
                            make_float4(acc1[sl1][3][0].x, acc1[sl1][3][0].y, acc1[sl1][3][1].x, acc1[sl1][3][1].y);
                    }
                }
                __syncwarp();
                if (edge_a) {
                    // boundary extension of the approximation band along the columns (edge strips)
                    if (psrc[0] != -2 || psrc[3] != -2) {
                        float* r0 = rrow0 - 4 * lane;
                        float* r1 = rrow1 - 4 * lane;
#pragma unroll
                        for (int jj = 0; jj < 4; ++jj)
                            if (psrc[jj] != -2) {
                                rrow0[jj] = psrc[jj] >= 0 ? r0[psrc[jj]] : 0.f;
                                rrow1[jj] = psrc[jj] >= 0 ? r1[psrc[jj]] : 0.f;
                            }
                    }
                    __syncwarp();
                }
                // level-2 row pass of both rows -> ring lines
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float* rrow = h ? rrow1 : rrow0;
                    float w[4 * Gm::NV2_4];
#pragma unroll
                    for (int q = 0; q < Gm::NV2_4; ++q) {
                        const float4 t = *reinterpret_cast<const float4*>(rrow + 4 * q);
                        w[4 * q] = t.x; w[4 * q + 1] = t.y; w[4 * q + 2] = t.z; w[4 * q + 3] = t.w;
                    }
                    float l2[2], h2[2];
                    wp_rowfilt<L, 2, Gm::OFF2>(w, p.pl, p.ph, l2, h2);
                    if (h ? v1 : v0) {
                        float* dst = ring_lane + ((a0 + h) & (RING - 1)) * R2P;
                        *reinterpret_cast<float2*>(dst) = make_float2(l2[0], l2[1]);
                        *reinterpret_cast<float2*>(dst + 64) = make_float2(h2[0], h2[1]);
                    }
                }
                produced = min(max(a0 + 2, a_lo), a_end);
            }
            __syncwarp();   // tile consumed by every lane; ring lines visible

            if (lane == 0 && g + NSTG < ngroups) {
                fence_proxy_async();
                mbar_expect_tx(&bars[stage], (uint32_t)Gm::STAGE_BYTES);
                tma_load_3d(tile, &tmap, &bars[stage], c_in0 / 2, r_in0 + (g + NSTG) * ROWS, b);
            }
            if (++stage == NSTG) { stage = 0; par ^= 1u; }
            cluster_arrive();

            // ---- level 2 column pass: every output row whose L ring lines exist ----------------------------
            while (K2 < Y1) {
                const int vb = 2 * K2 - HALO;                      // first row of the window
                float2 o[4] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
                if (vb >= 0 && vb + L <= p.Mh1) {
                    if (vb + L > produced) break;
#pragma unroll
                    for (int j = 0; j < L; ++j) {
                        const float* rr = ring_lane + ((vb + j) & (RING - 1)) * R2P;
                        const float2 lo = *reinterpret_cast<const float2*>(rr), hi = *reinterpret_cast<const float2*>(rr + 64);
                        o[0] = ffma2(p.vl[L - 1 - j], lo, o[0]); o[1] = ffma2(p.vl[L - 1 - j], hi, o[1]);
                        o[2] = ffma2(p.vh[L - 1 - j], lo, o[2]); o[3] = ffma2(p.vh[L - 1 - j], hi, o[3]);
                    }
                } else {
                    // window reaches over the top / bottom border of the approximation band
                    int src[L], mx = -1;
#pragma unroll
                    for (int j = 0; j < L; ++j) { src[j] = ext_index32(vb + j, p.Mh1, p.mode); mx = max(mx, src[j]); }
                    if (mx >= produced) break;
#pragma unroll
                    for (int j = 0; j < L; ++j) {
                        if (src[j] < 0) continue;
                        const float* rr = ring_lane + (src[j] & (RING - 1)) * R2P;
                        const float2 lo = *reinterpret_cast<const float2*>(rr), hi = *reinterpret_cast<const float2*>(rr + 64);
                        o[0] = ffma2(p.vl[L - 1 - j], lo, o[0]); o[1] = ffma2(p.vl[L - 1 - j], hi, o[1]);
                        o[2] = ffma2(p.vh[L - 1 - j], lo, o[2]); o[3] = ffma2(p.vh[L - 1 - j], hi, o[3]);
                    }
                }
                if (store2) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) *reinterpret_cast<float2*>(po2[k]) = o[k];
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) po2[k] += p.o2_rs[k];
                ++K2;
            }
        }
    }
    if (ngroups > 0) cluster_wait();   // pairs the last arrive
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static bool make_tmap_3d_pairs(CUtensorMap* map, const float* base, int64_t B, int64_t H, int64_t W, int64_t bs, int64_t rs,
                               int box_w_pairs, int box_h) {
    PFN_encodeTiled enc = get_encode_tiled();
    if (!enc) return false;
    if (((uintptr_t)base & 15) || (rs & 3) || (bs & 3)) return false;
    if ((W & 1) && rs <= W) return false;             // the odd sample's partner must be addressable
    if (box_w_pairs > 256 || box_h > 256 || ((box_w_pairs * 8) & 15)) return false;
    cuuint64_t dims[3] = {(cuuint64_t)((W + 1) / 2), (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)(rs * 4), (cuuint64_t)(bs * 4)};
    cuuint32_t box[3] = {(cuuint32_t)box_w_pairs, (cuuint32_t)box_h, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    if (B == 1) strides[1] = (cuuint64_t)H * strides[0];
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, (void*)base, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// Parameters, tensor map and strip count of one levels-1-2 call; false when the kernel does not take these shapes,
// strides or mode.  The grid is (nstrip, batch, p.nseg).
template <int L, int NSTG>
static bool wpair_plan(const float* x, int64_t B, int H, int W, int64_t x_bs, int64_t x_rs, const wt_level& l1,
                       const wt_level& l2, int mode, const Taps<float>& taps, WPairParams& p, CUtensorMap& tmap,
                       int& nstrip) {
    using Gm = WPairGeom<L, NSTG>;
    memset(&p, 0, sizeof(p));
    p.x = x; p.x_bs = x_bs; p.x_rs = x_rs; p.H = H; p.W = W;
    p.Mh1 = (int)l1.dims[0]; p.Mw1 = (int)l1.dims[1]; p.Mh2 = (int)l2.dims[0]; p.Mw2 = (int)l2.dims[1];
    if (mode == WT_MODE_PERIODIC) return false;
    if (p.Mh1 < 2 * Gm::RING + 2 || p.Mw1 < 4 * L || p.Mh2 < L || p.Mw2 < L) return false;
    // level-1 details: three bands with common strides, 128-bit stores
    p.d1 = (float*)l1.details; p.d1_bs = l1.details_batch_stride; p.d1_rs = l1.strides[0]; p.d1_band = l1.band_stride;
    if (l1.strides[1] != 1 || ((uintptr_t)p.d1 & 15) || (p.d1_bs & 3) || (p.d1_rs & 3) || (p.d1_band & 3) ||
        p.d1_rs < (p.Mw1 + 3) / 4 * 4)
        return false;
    // level-2 bands: 64-bit stores
    if (l2.strides[1] != 1 || l2.approx_strides[1] != 1) return false;
    p.o2[0] = (float*)l2.approx; p.o2_bs[0] = l2.approx_batch_stride; p.o2_rs[0] = l2.approx_strides[0];
    for (int k = 1; k < 4; ++k) {
        p.o2[k] = (float*)l2.details + (int64_t)(k - 1) * l2.band_stride;
        p.o2_bs[k] = l2.details_batch_stride; p.o2_rs[k] = l2.strides[0];
    }
    for (int k = 0; k < 4; ++k)
        if (((uintptr_t)p.o2[k] & 7) || (p.o2_bs[k] & 1) || (p.o2_rs[k] & 1) || p.o2_rs[k] < (p.Mw2 + 1) / 2 * 2) return false;
    // strips: the (possibly shifted) last strip must still reach the last level-2 column
    nstrip = (p.Mw2 + Gm::TW2 - 1) / Gm::TW2;
    {
        int X0 = (nstrip - 1) * Gm::TW2;
        const int lim = (p.Mw1 - L + Gm::HL1) / 2;
        if (X0 > lim) X0 = lim & ~1;
        if (X0 < 0 || X0 + Gm::TW2 < p.Mw2) return false;
        if (nstrip > 1 && X0 < (nstrip - 2) * Gm::TW2) return false;
    }
    p.mode = mode;
    for (int q = 0; q < L / 2; ++q) {
        p.pl[q] = make_float2(taps.lo[L - 1 - 2 * q], taps.lo[L - 2 - 2 * q]);
        p.ph[q] = make_float2(taps.hi[L - 1 - 2 * q], taps.hi[L - 2 - 2 * q]);
    }
    for (int m = 0; m < L; ++m) {
        p.vl[m] = make_float2(taps.lo[m], taps.lo[m]);
        p.vh[m] = make_float2(taps.hi[m], taps.hi[m]);
    }
    memset(&tmap, 0, sizeof(tmap));
    if (!make_tmap_3d_pairs(&tmap, x, B, H, W, x_bs, x_rs, Gm::TILE_W / 2, Gm::ROWS)) return false;
    // segments: long ones (restart overhead ~3 %) first, then geometrically shorter ones that fill the tail of the
    // grid (the segment index is the slowest grid dimension, so the short tasks are dispatched last)
    {
        const int forced = (int)knob_val(K_WPAIR_SEG, 0);
        int big = forced > 0 ? forced : 144;
        // enough tasks to fill the machine a few times
        const int64_t want = 3 * (int64_t)sm_count() * 12;
        while (forced <= 0 && big > 32 && (int64_t)((p.Mh2 + big - 1) / big) * nstrip * B < want) big -= 16;
        int y = 0, n = 0;
        p.seg_start[0] = 0;
        while (y < p.Mh2 && n < WPAIR_MAXSEG - 1) {
            const int left = p.Mh2 - y;
            int sz = big;
            if (forced <= 0 && left <= 3 * big) sz = left / 3 > 16 ? (left + 2) / 3 : (left > 24 ? 16 : left);
            if (sz > left || left - sz < 8) sz = left;
            y += sz;
            p.seg_start[++n] = y;
        }
        if (y < p.Mh2) p.seg_start[n] = p.Mh2;   // table full: the last segment takes the rest
        p.nseg = n;
    }
    return true;
}

// Returns true when the two levels were launched here (*err carries the launch status).
template <int L, int NSTG, int MINB>
static bool launch_fwd2d_wpair_t(const float* x, int64_t B, int H, int W, int64_t x_bs, int64_t x_rs, const wt_level& l1,
                                 const wt_level& l2, int mode, const Taps<float>& taps, cudaStream_t st,
                                 uint64_t* launches, cudaError_t* err) {
    using Gm = WPairGeom<L, NSTG>;
    WPairParams p;
    CUtensorMap tmap;
    int nstrip = 0;
    if (!wpair_plan<L, NSTG>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, p, tmap, nstrip)) return false;
    const int nseg = p.nseg;
    auto kern = fwd2d_wpair_kernel<L, NSTG, MINB>;
    const cudaError_t attr_err = ensure_dyn_smem(kern, (size_t)Gm::SMEM);
    if (attr_err != cudaSuccess) { *err = attr_err; return true; }
    *err = cudaSuccess;
    // clusters of adjacent strips (see the cluster barrier in the kernel): the largest of 6, 3, 2 that divides nstrip
    const int cl = nstrip % 6 == 0 ? 6 : nstrip % 3 == 0 ? 3 : nstrip % 2 == 0 ? 2 : 1;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cl; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    for (int64_t b0 = 0; b0 < B; b0 += 65535) {
        p.batch0 = (int)b0;
        const int nb = (int)((B - b0) < 65535 ? (B - b0) : 65535);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(nstrip, nb, nseg);
        cfg.blockDim = dim3(32, 1, 1);
        cfg.dynamicSmemBytes = Gm::SMEM;
        cfg.stream = st;
        cfg.attrs = &attr;
        cfg.numAttrs = 1;
        cudaLaunchKernelEx(&cfg, kern, p, tmap);
        ++*launches;
        *err = cudaGetLastError();
        if (*err != cudaSuccess) return true;
    }
    return true;
}

template <typename T>
static bool try_wpair(const T*, int64_t, int, int, int64_t, int64_t, const wt_level&, const wt_level&, int, int,
                      const Taps<T>&, cudaStream_t, uint64_t*, cudaError_t*) {
    return false;
}
template <>
bool try_wpair<float>(const float* x, int64_t B, int H, int W, int64_t x_bs, int64_t x_rs, const wt_level& l1,
                      const wt_level& l2, int L, int mode, const Taps<float>& taps, cudaStream_t st,
                      uint64_t* launches, cudaError_t* err) {
    // Default for levels (1, 2) of batches of >= 8 images of >= WPAIR_MIN = 2^24 samples (the caller checks): cA1
    // never reaches HBM.  On an H100 80GB HBM3 at a 400 W power limit (tools/time_fwd2d_pairs.py), db4 level 4 takes
    // 4.64 ms against 5.67 ms with one strip-kernel launch per level for 64 x 4096^2 and 0.68 against 0.76 ms for
    // 8 x 4096^2; one 4096^2 image (0.25 against 0.17 ms) and images of 2048^2 and smaller (up to 40 % slower) are
    // faster with one launch per level.  WPAIR=0 or NO_WPAIR=1 (environment
    // WTB200_<NAME> or wt_set_knob) forces one launch per level.
    if ((knob_is_set(K_WPAIR) && !knob_on(K_WPAIR)) || knob_on(K_NO_WPAIR) || knob_on(K_DISABLE_FUSED)) return false;
    switch (L) {
        case 2: return launch_fwd2d_wpair_t<2, 3, 12>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
        case 4: return launch_fwd2d_wpair_t<4, 3, 12>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
        case 6: return launch_fwd2d_wpair_t<6, 3, 12>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
        case 8:
            if (knob_val(K_WPAIR_VAR, 0) == 1)
                return launch_fwd2d_wpair_t<8, 2, 15>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
            if (knob_val(K_WPAIR_VAR, 0) == 3)
                return launch_fwd2d_wpair_t<8, 3, 12>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
            return launch_fwd2d_wpair_t<8, 2, 12>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
        default: return false;
    }
}

}  // namespace wtb
