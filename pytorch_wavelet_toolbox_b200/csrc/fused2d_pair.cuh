// fused2d_pair.cuh -- TWO analysis levels of the 2-D transform in one kernel (float32).
//
// The level-1 approximation band is the only data the reference's level loop
// (src/ptwt/conv_transform_2.py:142-149) carries from one level to the next.  With one launch per
// level it makes a round trip through HBM (+25 % traffic at level 1).  Here a CTA keeps rolling down
// a strip exactly like fwd2d_strip_kernel, but the level-1 column pass hands the approximation rows
// to a second, smaller filter bank through shared memory:
//
//   warps 0 .. NW1-1   level 1: TMA-staged input chunk -> row pass -> ring1 -> column pass
//                               (details to HBM, approximation rows -> tile2 in shared memory)
//   warps NW1, NW1+1   level 2, one chunk behind: tile2 -> (border patch) -> row pass -> ring2 ->
//                               column pass -> all four level-2 bands to HBM
//
// Both groups meet at the same two CTA barriers per chunk, so level 2 costs no extra phases.
// Strip geometry: a CTA owns 32 level-2 columns = 64 level-1 columns and computes HL1 extra level-1
// approximation columns on the left (the horizontal halo of level 2); level-1 details are stored for
// the owned 64 columns only.  The last strip is shifted left so that every boundary-extension source
// of the level-1 approximation lies inside the strip (duplicate stores carry identical values).
// Vertically both levels roll; level 2 lags by HALO rows so that the top-border sources exist.
// Periodic extension needs samples from the far side of the approximation band and is therefore
// left to the one-level kernel.
#pragma once

#include "fused2d.cuh"

namespace wtb {

struct Pair2dParams {
    const float* x;          // level-1 input [batch, H, W]
    int64_t x_bs, x_rs;
    float* d1[3];            // level-1 detail bands k = 1, 2, 3
    int64_t d1_bs, d1_rs;
    float* o2[4];            // level-2 bands k = 0 (approx), 1, 2, 3
    int64_t o2_bs[4], o2_rs[4];
    int H, W, Mh1, Mw1, Mh2, Mw2;
    int seg2_rows;           // level-2 output rows per segment
    int mode;
    int batch0;
    int vec1, vec2;          // 128-bit stores allowed for level-1 details / level-2 bands
    // filter taps packed in pairs for ffma2: polyphase pairs for the row passes,
    // broadcast pairs for the column passes (index j = tap applied to ring row j of the window)
    float2 pl[8], ph[8];     // {dec[L-1-2m], dec[L-2-2m]}
    float2 bl[16], bh[16];   // {dec[L-1-j], dec[L-1-j]}
};

template <int L, int TW2_ = 32>
struct Pair2dGeom {
    static constexpr int HALO = L - 2;
    static constexpr int HAL = (HALO + 3) / 4 * 4;            // 16-byte aligned halo (float)
    static constexpr int HL1 = (HALO + 1 + 7) / 8 * 8;        // extra level-1 approximation columns (left)
    static constexpr int OWN1 = 2 * TW2_;                      // level-1 columns whose details this CTA stores
    static constexpr int TW1 = OWN1 + HL1;                     // level-1 columns computed
    static constexpr int TW2 = TW2_;                           // level-2 columns owned
    static constexpr int CH = 16, IN_ROWS = 32;
    static constexpr int NEED1 = 2 * TW1 + HAL;
    static constexpr int SW1 = ((NEED1 - 4 + 7) / 8) * 8 + 4;  // staged tile pitch, == 4 (mod 8)
    static constexpr int OFF1 = HAL - HALO;
    static constexpr int MP1 = TW1 + 4;
    static constexpr int RING1 = IN_ROWS + HALO;
    static constexpr int MIR = L + 2;                          // mirror rows appended to the rings (no wrap in reads)
    static constexpr int T2P = TW1 + 4;                        // pitch of the approximation tile
    static constexpr int OFF2 = HL1 - HALO;
    static constexpr int MP2 = TW2 + 4;
    static constexpr int RING2 = (CH + 2 * HALO + 2) <= 32 ? 32 : 64;
    static constexpr int NW1 = TW1 / 8, NW2 = TW2 / 16, NT2 = 32 * NW2;
    static constexpr int NT1 = 32 * NW1, NT = 32 * (NW1 + NW2);
    static constexpr int NV1 = 16 + HAL, NV1_4 = (NV1 + 3) / 4;
    static constexpr int NV2 = 16 + HALO + OFF2, NV2_4 = (NV2 + 3) / 4;
    // level-2 rows that become computable after level-1 chunk c: Y <= Y0 + 8 c + D
    static constexpr int D2 = (14 - 5 * HALO / 2 >= 0) ? (14 - 5 * HALO / 2) / 2 : -((5 * HALO / 2 - 14 + 1) / 2);
    static constexpr size_t STAGE_BYTES = (size_t)IN_ROWS * SW1 * 4;
    static constexpr size_t SMEM = 2 * STAGE_BYTES + 2 * (size_t)(RING1 + MIR) * MP1 * 4 + (size_t)CH * T2P * 4 +
                                   2 * (size_t)(RING2 + MIR) * MP2 * 4 + 64;
    static_assert(L % 2 == 0 && L >= 2 && L <= 16, "pair kernel: even filter length <= 16");
    static_assert(16 * (NW1 - 1) + 4 * NV1_4 <= SW1, "level-1 row pass reads past the tile");
    static_assert(16 * (TW2 / 8 - 1) + 4 * NV2_4 <= T2P, "level-2 row pass reads past the approximation tile");
    static_assert(TW2 == 16 || TW2 == 32, "TW2 must be 16 or 32");
    static_assert(CH + 2 * HALO + 2 <= RING2, "ring2 too small");
};

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

template <int L, bool USE_TMA, int TW2_ = 32>
__global__ void __launch_bounds__((Pair2dGeom<L, TW2_>::NT), (TW2_ == 32 ? 2 : 4))
fwd2d_pair_kernel(const __grid_constant__ Pair2dParams p, const __grid_constant__ CUtensorMap tmap) {
    using Gm = Pair2dGeom<L, TW2_>;
    constexpr int NT2 = Gm::NT2;
    constexpr int HALO = Gm::HALO, HAL = Gm::HAL, HL1 = Gm::HL1, TW1 = Gm::TW1, TW2 = Gm::TW2, CH = Gm::CH;
    constexpr int IN_ROWS = Gm::IN_ROWS, SW1 = Gm::SW1, OFF1 = Gm::OFF1, MP1 = Gm::MP1, RING1 = Gm::RING1;
    constexpr int T2P = Gm::T2P, OFF2 = Gm::OFF2, MP2 = Gm::MP2, RING2 = Gm::RING2, MIR = Gm::MIR;
    constexpr int NW1 = Gm::NW1, NT1 = Gm::NT1, NV1_4 = Gm::NV1_4, NV2_4 = Gm::NV2_4, D2 = Gm::D2;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_in = reinterpret_cast<float*>(smem_raw);                        // [2][IN_ROWS][SW1]
    float* s_lo1 = s_in + 2 * IN_ROWS * SW1;                                 // [RING1 + MIR][MP1]
    float* s_hi1 = s_lo1 + (RING1 + MIR) * MP1;
    float* s_t2 = s_hi1 + (RING1 + MIR) * MP1;                               // [CH][T2P]
    float* s_lo2 = s_t2 + CH * T2P;                                          // [RING2 + MIR][MP2]
    float* s_hi2 = s_lo2 + (RING2 + MIR) * MP2;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_hi2 + (RING2 + MIR) * MP2);   // [2]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool is_l1 = warp < NW1;
    const int b = p.batch0 + blockIdx.z;

    // ---- strip / segment geometry -----------------------------------------------------------
    int X0 = blockIdx.x * TW2;                         // first owned level-2 column
    if (X0 + TW2 > p.Mw2) X0 = max(p.Mw2 - TW2, 0);    // last strip: shifted left, overlaps its neighbour
    const int x0 = 2 * X0;                             // first owned level-1 column
    const bool vec1 = p.vec1 && !(x0 & 3), vec2 = p.vec2 && !(X0 & 3);   // the shifted strip may be misaligned
    const int Y0 = blockIdx.y * p.seg2_rows;
    if (Y0 >= p.Mh2) return;
    const int Y1 = min(Y0 + p.seg2_rows, p.Mh2);
    const int own1_y0 = 2 * Y0, own1_y1 = min(2 * Y1, p.Mh1);    // level-1 detail rows stored here
    const int yb1 = 2 * Y0 - HALO - HALO / 2;          // level-1 chunk c covers rows [yb1 + 16 c, +16)
    const int c_in0 = 2 * (x0 - HL1) - HAL;            // first staged input column (16-byte aligned)
    const int r_in0 = 2 * yb1;                         // first staged input row of chunk 0
    // level-2 rows Y <= Y0 + 8 c + D2 are computable once level-1 chunk c is done
    const int c_last = max((Y1 - 1 - Y0 - D2 + 7) / 8, 0);
    const int nchunks = c_last + 1;                    // level-1 chunks; the loop runs one more iteration
    const int c_need1 = 2 * min(x0 + Gm::OWN1, p.Mw1); // one past the last input column a valid output reads
    const int r_need1 = 2 * min(yb1 + nchunks * CH, p.Mh1);

    if (USE_TMA) {
        if (tid == 0) {
            tma_prefetch_desc(&tmap);
            mbar_init(&bars[0], 1);
            mbar_init(&bars[1], 1);
            fence_mbar_init();
        }
        __syncthreads();
        if (tid == 0) {
            for (int s = 0; s < 2 && s < nchunks; ++s) {
                mbar_expect_tx(&bars[s], (uint32_t)Gm::STAGE_BYTES);
                tma_load_3d(s_in + s * IN_ROWS * SW1, &tmap, &bars[s], c_in0, r_in0 + s * IN_ROWS, b);
            }
        }
    }
    const float* __restrict__ xb = p.x + (int64_t)b * p.x_bs;

    // ---- per-thread constants of the level-1 column pass --------------------------------------
    constexpr int NCG1 = TW1 / 4;
    const int c1_half = tid / (NT1 / 2);
    const int c1_rem = tid - c1_half * (NT1 / 2);
    const int c1_rp = c1_rem / NCG1, c1_cg = c1_rem - c1_rp * NCG1;
    const int c1_yl = 2 * c1_rp;
    const bool c1_halo = c1_cg < HL1 / 4;
    const bool c1_skip = (c1_half == 1 && c1_halo) || !is_l1;
    const float* c1_ring = (c1_half ? s_hi1 : s_lo1) + 4 * c1_cg;
    const int c1_gx = x0 + 4 * c1_cg - HL1;
    const bool c1_store = !c1_halo && c1_gx < p.Mw1 && is_l1;
    // global pointers of output row (yb1 + yl) of the two detail bands this thread stores
    float* c1_pA = nullptr;
    float* c1_pB = nullptr;
    if (c1_store) {
        const int64_t o = (int64_t)b * p.d1_bs + (int64_t)(yb1 + c1_yl) * p.d1_rs + c1_gx;
        c1_pA = c1_half ? p.d1[0] + o : nullptr;                 // lo_H hi_W  (band 1)
        c1_pB = (c1_half ? p.d1[2] : p.d1[1]) + o;               // hi_H hi_W (3) | hi_H lo_W (2)
    }
    // ---- per-thread constants of the level-2 passes (threads NT1 .. NT1+63) ---------------------
    const int t2 = tid - NT1;
    const int r2_row = t2 & 15, r2_grp = (t2 >> 4) & (TW2 / 8 - 1);
    constexpr int NCG2 = TW2 / 4;
    const int c2_half = (t2 / (NT2 / 2)) & 1, c2_rp = ((t2 % (NT2 / 2)) / NCG2) & 3, c2_cg = t2 % NCG2;
    const float* c2_ring = (c2_half ? s_hi2 : s_lo2) + 4 * c2_cg;
    const int c2_gx = X0 + 4 * c2_cg;

    int ring1_base = 0;
    for (int c = 0; c <= nchunks; ++c) {
        const bool l1_active = c < nchunks;
        const int stage = c & 1;
        float* tile = s_in + stage * IN_ROWS * SW1;

        // =============================== phase A ===============================================
        if (is_l1) {
            if (l1_active) {
                const int r_base = r_in0 + c * IN_ROWS;
                if (USE_TMA) {
                    mbar_wait(&bars[stage], (uint32_t)((c >> 1) & 1));
                    if (p.mode != WT_MODE_ZERO) {
                        // patch the out-of-range input samples valid outputs read (see fwd2d_strip_kernel)
                        const int cl0 = c_in0 < 0 ? max(-c_in0 - HALO, 0) : 0;
                        const int nl = c_in0 < 0 ? -c_in0 - cl0 : 0;
                        const int cr1 = min(c_need1 - c_in0, SW1);
                        const int cr0 = max(min(p.W - c_in0, cr1), cl0 + nl);
                        const int nt = r_base < 0 ? min(-r_base, IN_ROWS) : 0;
                        const int rb1 = min(r_need1 - r_base, IN_ROWS);
                        const int rb0 = max(min(p.H - r_base, rb1), nt);
                        const int wb = nl + max(cr1 - cr0, 0);
                        const bool patch = (wb > 0 && rb0 > nt) || (nt > 0) || (rb1 > rb0);
                        if (patch) {
                            const int n_in = max(rb0 - nt, 0);
                            for (int idx = tid; idx < n_in * wb; idx += NT1) {
                                const int rr = nt + idx / wb, q = idx % wb;
                                const int cc = q < nl ? cl0 + q : cr0 + (q - nl);
                                const int sc = ext_index32(c_in0 + cc, p.W, p.mode);
                                tile[rr * SW1 + cc] = __ldg(xb + (int64_t)(r_base + rr) * p.x_rs + sc);
                            }
                            const int n_oob = nt + max(rb1 - rb0, 0);
                            const int wn = cr1 - cl0;
                            if (n_oob > 0 && wn > 0) {
                                for (int idx = tid; idx < n_oob * wn; idx += NT1) {
                                    const int q = idx / wn, cc = cl0 + idx % wn;
                                    const int rr = q < nt ? q : rb0 + (q - nt);
                                    const int sr = ext_index32(r_base + rr, p.H, p.mode);
                                    const int sc = ext_index32(c_in0 + cc, p.W, p.mode);
                                    tile[rr * SW1 + cc] = __ldg(xb + (int64_t)sr * p.x_rs + sc);
                                }
                            }
                            named_bar_sync(1, NT1);
                        }
                    }
                } else {
                    for (int idx = tid; idx < IN_ROWS * SW1; idx += NT1) {
                        const int rr = idx / SW1, cc = idx - rr * SW1;
                        const int sr = ext_index32(r_base + rr, p.H, p.mode), sc = ext_index32(c_in0 + cc, p.W, p.mode);
                        tile[idx] = (sr >= 0 && sc >= 0) ? __ldg(xb + (int64_t)sr * p.x_rs + sc) : 0.f;
                    }
                    named_bar_sync(1, NT1);
                }
                // ---- level-1 row pass: lane <-> tile row, warp <-> 8 output columns --------------
                const float* src = tile + lane * SW1 + 16 * warp;
                float v[4 * NV1_4];
#pragma unroll
                for (int q = 0; q < NV1_4; ++q) {
                    const float4 t = *reinterpret_cast<const float4*>(src + 4 * q);
                    v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
                }
                float lo[8], hi[8];
                row_filter8<L, OFF1>(v, p.pl, p.ph, lo, hi);
                int slot = ring1_base + lane;
                if (slot >= RING1) slot -= RING1;
                float* dlo = s_lo1 + slot * MP1 + 8 * warp;
                float* dhi = s_hi1 + slot * MP1 + 8 * warp;
                const float4 l0 = make_float4(lo[0], lo[1], lo[2], lo[3]), l1v = make_float4(lo[4], lo[5], lo[6], lo[7]);
                const float4 h0 = make_float4(hi[0], hi[1], hi[2], hi[3]), h1v = make_float4(hi[4], hi[5], hi[6], hi[7]);
                *reinterpret_cast<float4*>(dlo) = l0; *reinterpret_cast<float4*>(dlo + 4) = l1v;
                *reinterpret_cast<float4*>(dhi) = h0; *reinterpret_cast<float4*>(dhi + 4) = h1v;
                if (slot < MIR) {   // mirror copy so that column-pass windows never wrap
                    *reinterpret_cast<float4*>(dlo + RING1 * MP1) = l0; *reinterpret_cast<float4*>(dlo + RING1 * MP1 + 4) = l1v;
                    *reinterpret_cast<float4*>(dhi + RING1 * MP1) = h0; *reinterpret_cast<float4*>(dhi + RING1 * MP1 + 4) = h1v;
                }
            }
        } else if (c >= 1) {
            // ---- level 2, fed by the approximation rows of level-1 chunk c - 1 (in s_t2) ----------
            const int rowbase = yb1 + (c - 1) * CH;         // level-1 row index of tile2 row 0
            const int col0 = x0 - HL1;                      // level-1 column of tile2 column 0
            // (1) boundary extension of the approximation band along the columns
            {
                const int need1 = 2 * min(X0 + TW2, p.Mw2); // one past the last approximation column level 2 reads
                const int tl0 = max((x0 - HALO) - col0, 0), tl1 = max(min(0 - col0, TW1), tl0);   // columns < 0
                const int tr0 = max(p.Mw1 - col0, 0), tr1 = max(min(need1 - col0, TW1), tr0);     // columns >= Mw1
                const int wpatch = (tl1 - tl0) + (tr1 - tr0);
                if (wpatch > 0) {
                    for (int idx = t2; idx < CH * wpatch; idx += NT2) {
                        const int rr = idx / wpatch, q = idx % wpatch;
                        const int t = q < (tl1 - tl0) ? tl0 + q : tr0 + (q - (tl1 - tl0));
                        const int sc = ext_index32(col0 + t, p.Mw1, p.mode);
                        s_t2[rr * T2P + t] = sc >= 0 ? s_t2[rr * T2P + (sc - col0)] : 0.f;
                    }
                    named_bar_sync(2, NT2);
                }
            }
            // (2) level-2 row pass: 16 rows x 4 groups of 8 outputs
            {
                const int rr = rowbase + r2_row;            // level-1 approximation row index
                if (rr >= 0 && rr < p.Mh1) {
                    const float* src = s_t2 + r2_row * T2P + 16 * r2_grp;
                    float v[4 * NV2_4];
#pragma unroll
                    for (int q = 0; q < NV2_4; ++q) {
                        const float4 t = *reinterpret_cast<const float4*>(src + 4 * q);
                        v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
                    }
                    float lo[8], hi[8];
                    row_filter8<L, OFF2>(v, p.pl, p.ph, lo, hi);
                    const int slot = rr & (RING2 - 1);
                    float* dlo = s_lo2 + slot * MP2 + 8 * r2_grp;
                    float* dhi = s_hi2 + slot * MP2 + 8 * r2_grp;
                    const float4 l0 = make_float4(lo[0], lo[1], lo[2], lo[3]), l1v = make_float4(lo[4], lo[5], lo[6], lo[7]);
                    const float4 h0 = make_float4(hi[0], hi[1], hi[2], hi[3]), h1v = make_float4(hi[4], hi[5], hi[6], hi[7]);
                    *reinterpret_cast<float4*>(dlo) = l0; *reinterpret_cast<float4*>(dlo + 4) = l1v;
                    *reinterpret_cast<float4*>(dhi) = h0; *reinterpret_cast<float4*>(dhi + 4) = h1v;
                    if (slot < MIR) {
                        *reinterpret_cast<float4*>(dlo + RING2 * MP2) = l0; *reinterpret_cast<float4*>(dlo + RING2 * MP2 + 4) = l1v;
                        *reinterpret_cast<float4*>(dhi + RING2 * MP2) = h0; *reinterpret_cast<float4*>(dhi + RING2 * MP2 + 4) = h1v;
                    }
                }
            }
        }
        __syncthreads();   // B1: ring1 rows of chunk c and ring2 rows of chunk c-1 are visible

        if (USE_TMA && tid == 0 && c + 2 < nchunks) {
            fence_proxy_async();
            mbar_expect_tx(&bars[stage], (uint32_t)Gm::STAGE_BYTES);
            tma_load_3d(tile, &tmap, &bars[stage], c_in0, r_in0 + (c + 2) * IN_ROWS, b);
        }

        // =============================== phase B ===============================================
        if (is_l1) {
            if (l1_active && !c1_skip) {
                // level-1 column pass: thread <-> (lo|hi array, 2 output rows, 4 output columns)
                int row0 = ring1_base + 2 * c1_yl - HALO;   // in (-RING1, 2 RING1): one wrap suffices
                if (row0 < 0) row0 += RING1;
                else if (row0 >= RING1) row0 -= RING1;
                float2 accL[2][2], accH[2][2];
                col_filter2x4<L>(c1_ring + row0 * MP1, MP1, p.bl, p.bh, accL, accH);
                if (c1_half == 0) {
                    // approximation rows stay on chip
                    *reinterpret_cast<float4*>(s_t2 + c1_yl * T2P + 4 * c1_cg) = make_float4(accL[0][0].x, accL[0][0].y, accL[0][1].x, accL[0][1].y);
                    *reinterpret_cast<float4*>(s_t2 + (c1_yl + 1) * T2P + 4 * c1_cg) = make_float4(accL[1][0].x, accL[1][0].y, accL[1][1].x, accL[1][1].y);
                }
                if (c1_store) {
                    const int gyc = yb1 + c * CH + c1_yl;
                    const int64_t adv = (int64_t)c * CH * p.d1_rs;
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const int gy = gyc + r;
                        if (gy < own1_y0 || gy >= own1_y1) continue;
                        float* qB = c1_pB + adv + (int64_t)r * p.d1_rs;
                        if (vec1) {
                            if (c1_half) *reinterpret_cast<float4*>(c1_pA + adv + (int64_t)r * p.d1_rs) = make_float4(accL[r][0].x, accL[r][0].y, accL[r][1].x, accL[r][1].y);
                            *reinterpret_cast<float4*>(qB) = make_float4(accH[r][0].x, accH[r][0].y, accH[r][1].x, accH[r][1].y);
                        } else {
                            const float aL[4] = {accL[r][0].x, accL[r][0].y, accL[r][1].x, accL[r][1].y};
                            const float aH[4] = {accH[r][0].x, accH[r][0].y, accH[r][1].x, accH[r][1].y};
#pragma unroll
                            for (int e = 0; e < 4; ++e)
                                if (c1_gx + e < p.Mw1) {
                                    if (c1_half) (c1_pA + adv + (int64_t)r * p.d1_rs)[e] = aL[e];
                                    qB[e] = aH[e];
                                }
                        }
                    }
                }
            }
        } else if (c >= 1) {
            // level-2 column pass: rows Y in [Yhi - 7, Yhi], Yhi = Y0 + 8 (c - 1) + D2
            const int Ya = Y0 + 8 * (c - 1) + D2 - 7 + 2 * c2_rp;    // first of the two output rows
            if (Ya + 1 >= Y0 && Ya < Y1 && c2_gx < p.Mw2) {
                float2 accL[2][2], accH[2][2];
                const int ra = 2 * Ya - HALO;                          // first approximation row of the window
                if (ra >= 0 && ra + L + 1 < p.Mh1) {
                    col_filter2x4<L>(c2_ring + (ra & (RING2 - 1)) * MP2, MP2, p.bl, p.bh, accL, accH);
                } else {
                    // window touches the top / bottom border of the approximation band
#pragma unroll
                    for (int r = 0; r < 2; ++r)
#pragma unroll
                        for (int e = 0; e < 2; ++e) { accL[r][e] = make_float2(0.f, 0.f); accH[r][e] = make_float2(0.f, 0.f); }
#pragma unroll
                    for (int j = 0; j < L + 2; ++j) {
                        int rr = ra + j;
                        if (rr < 0 || rr >= p.Mh1) rr = ext_index32(rr, p.Mh1, p.mode);
                        float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (rr >= 0) f = *reinterpret_cast<const float4*>(c2_ring + (rr & (RING2 - 1)) * MP2);
                        const float2 w0 = make_float2(f.x, f.y), w1 = make_float2(f.z, f.w);
                        if (j < L) {
                            accL[0][0] = ffma2(p.bl[j], w0, accL[0][0]); accL[0][1] = ffma2(p.bl[j], w1, accL[0][1]);
                            accH[0][0] = ffma2(p.bh[j], w0, accH[0][0]); accH[0][1] = ffma2(p.bh[j], w1, accH[0][1]);
                        }
                        if (j >= 2) {
                            accL[1][0] = ffma2(p.bl[j - 2], w0, accL[1][0]); accL[1][1] = ffma2(p.bl[j - 2], w1, accL[1][1]);
                            accH[1][0] = ffma2(p.bh[j - 2], w0, accH[1][0]); accH[1][1] = ffma2(p.bh[j - 2], w1, accH[1][1]);
                        }
                    }
                }
                float* oL = p.o2[c2_half] + (int64_t)b * p.o2_bs[c2_half] + c2_gx;
                float* oH = p.o2[2 + c2_half] + (int64_t)b * p.o2_bs[2 + c2_half] + c2_gx;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int gy = Ya + r;
                    if (gy < Y0 || gy >= Y1) continue;
                    float* dl = oL + (int64_t)gy * p.o2_rs[c2_half];
                    float* dh = oH + (int64_t)gy * p.o2_rs[2 + c2_half];
                    if (vec2) {
                        *reinterpret_cast<float4*>(dl) = make_float4(accL[r][0].x, accL[r][0].y, accL[r][1].x, accL[r][1].y);
                        *reinterpret_cast<float4*>(dh) = make_float4(accH[r][0].x, accH[r][0].y, accH[r][1].x, accH[r][1].y);
                    } else {
                        const float aL[4] = {accL[r][0].x, accL[r][0].y, accL[r][1].x, accL[r][1].y};
                        const float aH[4] = {accH[r][0].x, accH[r][0].y, accH[r][1].x, accH[r][1].y};
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            if (c2_gx + e < p.Mw2) { dl[e] = aL[e]; dh[e] = aH[e]; }
                    }
                }
            }
        }
        __syncthreads();   // B2: tile2 (chunk c) complete; ring1 / ring2 rows may be overwritten
        ring1_base += IN_ROWS;
        if (ring1_base >= RING1) ring1_base -= RING1;
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static bool pair2d_supported(int L, int mode) {
    // experimental: correct (tests run it with WTB200_ENABLE_PAIR=1) but at 2 CTAs/SM it is not yet
    // faster than two one-level launches, so it is off by default
    return !(L & 1) && L >= 2 && L <= 8 && mode != WT_MODE_PERIODIC && knob_on(K_ENABLE_PAIR);
}

template <int L, int TW2_>
static cudaError_t launch_fwd2d_pair_t(const float* x, int64_t B, int H, int W, int64_t x_bs, int64_t x_rs,
                                       const wt_level& l1, const wt_level& l2, int mode, const Taps<float>& taps,
                                       cudaStream_t st, uint64_t* launches) {
    using Gm = Pair2dGeom<L, TW2_>;
    Pair2dParams p;
    p.x = x; p.x_bs = x_bs; p.x_rs = x_rs;
    p.H = H; p.W = W;
    p.Mh1 = (int)l1.dims[0]; p.Mw1 = (int)l1.dims[1]; p.Mh2 = (int)l2.dims[0]; p.Mw2 = (int)l2.dims[1];
    for (int k = 0; k < 3; ++k) p.d1[k] = (float*)l1.details + (int64_t)k * l1.band_stride;
    p.d1_bs = l1.details_batch_stride; p.d1_rs = l1.strides[0];
    p.o2[0] = (float*)l2.approx; p.o2_bs[0] = l2.approx_batch_stride; p.o2_rs[0] = l2.approx_strides[0];
    for (int k = 1; k < 4; ++k) {
        p.o2[k] = (float*)l2.details + (int64_t)(k - 1) * l2.band_stride;
        p.o2_bs[k] = l2.details_batch_stride; p.o2_rs[k] = l2.strides[0];
    }
    p.mode = mode;
    for (int m = 0; m < L / 2; ++m) {
        p.pl[m] = make_float2(taps.lo[L - 1 - 2 * m], taps.lo[L - 2 - 2 * m]);
        p.ph[m] = make_float2(taps.hi[L - 1 - 2 * m], taps.hi[L - 2 - 2 * m]);
    }
    for (int j = 0; j < L; ++j) {
        p.bl[j] = make_float2(taps.lo[L - 1 - j], taps.lo[L - 1 - j]);
        p.bh[j] = make_float2(taps.hi[L - 1 - j], taps.hi[L - 1 - j]);
    }
    p.vec1 = 1;
    for (int k = 0; k < 3; ++k)
        if (((uintptr_t)p.d1[k] & 15) || (p.d1_bs & 3) || (p.d1_rs & 3) || p.d1_rs < (p.Mw1 + 3) / 4 * 4) p.vec1 = 0;
    p.vec2 = 1;
    for (int k = 0; k < 4; ++k)
        if (((uintptr_t)p.o2[k] & 15) || (p.o2_bs[k] & 3) || (p.o2_rs[k] & 3) || p.o2_rs[k] < (p.Mw2 + 3) / 4 * 4) p.vec2 = 0;
    const int nstrip0 = (p.Mw2 + Gm::TW2 - 1) / Gm::TW2;
    int nseg = (p.Mh2 + 255) / 256;
    // small levels: shorter segments so that the grid still fills the machine a few times
    while ((int64_t)nseg * nstrip0 * B < 4 * 296 && (p.Mh2 + nseg - 1) / nseg > 48) ++nseg;
    int seg = ((p.Mh2 + nseg - 1) / nseg + 7) / 8 * 8;
    nseg = (p.Mh2 + seg - 1) / seg;
    p.seg2_rows = seg;
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof(tmap));
    const bool tma = make_tmap_3d<float>(&tmap, x, B, H, W, x_bs, x_rs, Gm::SW1, Gm::IN_ROWS);
    auto kern = tma ? fwd2d_pair_kernel<L, true, TW2_> : fwd2d_pair_kernel<L, false, TW2_>;
    cudaError_t e = ensure_dyn_smem(kern, (size_t)Gm::SMEM);
    if (e != cudaSuccess) return e;
    const int nstrip = (p.Mw2 + Gm::TW2 - 1) / Gm::TW2;
    for (int64_t b0 = 0; b0 < B; b0 += 65535) {
        p.batch0 = (int)b0;
        const int nb = (int)((B - b0) < 65535 ? (B - b0) : 65535);
        dim3 grid(nstrip, nseg, nb);
        kern<<<grid, Gm::NT, Gm::SMEM, st>>>(p, tmap);
        ++*launches;
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

template <int L>
static cudaError_t launch_fwd2d_pair(const float* x, int64_t B, int H, int W, int64_t x_bs, int64_t x_rs,
                                     const wt_level& l1, const wt_level& l2, int mode, const Taps<float>& taps,
                                     cudaStream_t st, uint64_t* launches) {
    if (knob_val(K_PAIR_TW2, 32) == 16)
        return launch_fwd2d_pair_t<L, 16>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches);
    return launch_fwd2d_pair_t<L, 32>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches);
}

}  // namespace wtb
