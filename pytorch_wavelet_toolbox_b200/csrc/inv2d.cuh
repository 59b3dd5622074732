// inv2d.cuh -- one 2-D synthesis level as ONE kernel (float32): rolling column strips, mirror image
// of fwd2d_strip_f32_kernel.
//
// Replaces the reference's  stack([ll, lh, hl, hh]) -> conv_transpose2d(4 x [L x L], stride 2) -> crop
// (src/ptwt/conv_transform_2.py:224-249): no stacked copy, no full-size uncropped intermediate; the
// four sub-bands are read once and the reconstruction is written once.
//
//   y[t] = sum_i lo[i] rec_lo[t + L-2 - 2i] + hi[i] rec_hi[t + L-2 - 2i]          (per axis)
//
//   * a CTA owns 128 output columns (64 + L/2 - 1 coefficient columns) and a segment of output rows and
//     marches down in chunks of 16 coefficient rows = 32 output rows;
//   * the 4 band tiles [16 x CP] of a chunk are staged by TMA (one tensor map per band, out-of-range
//     coefficients = zero fill, which is exactly what a transposed convolution needs: no boundary
//     extension exists on the synthesis side), 2-stage mbarrier ring;
//   * row pass (synthesis along W): lane <-> (band pair, coefficient row), warp <-> 16 output columns;
//     (ll, hl) -> Lh and (lh, hh) -> Hh, written to a ring of 16 + L/2 - 1 rows (+ mirror rows);
//   * column pass (synthesis along H): thread <-> (4 output rows, 4 output columns): L/2 + 1 ring rows
//     of Lh and Hh (LDS.128, no wrap), 64 paired FMAs (ffma2), 4 coalesced STG.128.
//
// Algorithmic bytes per level: 4 B * (4 Mh Mw read + OH OW written).
#pragma once

#include "fused2d.cuh"

namespace wtb {

struct Inv2dParams {
    const float* in[4];      // sub-bands k = 0..3 of this level, [batch, Mh, Mw]
    int64_t in_bs[4], in_rs[4];
    float* y;                // reconstruction [batch, OH, OW]
    int64_t y_bs, y_rs;
    int Mh, Mw, OH, OW;
    int seg_rows;            // output rows per segment (even)
    int batch0;
    int vec_store;
    float rlo[16], rhi[16];  // un-flipped rec_lo / rec_hi (row pass, scalar FMAs)
    float2 bl[16], bh[16];   // {rec_lo[k], rec_lo[k]}, {rec_hi[k], rec_hi[k]} (column pass, ffma2)
};

struct Inv2dMaps {
    CUtensorMap m[4];
};

constexpr int INV2D_TWO = 128;                                  // output columns per strip

template <int L>
struct Inv2dGeom {
    static constexpr int HALF = L / 2;
    static constexpr int TWO = INV2D_TWO;
    static constexpr int NC = TWO / 2 + HALF - 1;               // coefficient columns a strip reads
    static constexpr int CP = ((NC - 4 + 7) / 8) * 8 + 4;       // staged pitch, == 4 (mod 8), multiple of 4
    static constexpr int CR = 16;                               // coefficient rows per chunk
    static constexpr int RING = CR + HALF - 1;
    static constexpr int MIR = HALF + 1;
    static constexpr int RP = TWO + 4;
    static constexpr int NT = 256;
    static constexpr int NVC = 8 + HALF - 1;                    // coefficient samples per row-pass thread
    static constexpr int NVC4 = (NVC + 3) / 4;
    static constexpr size_t BAND_BYTES = (size_t)CR * CP * 4;
    static constexpr size_t STAGE_BYTES = 4 * BAND_BYTES;
    static constexpr size_t SMEM = 2 * STAGE_BYTES + 2 * (size_t)(RING + MIR) * RP * 4 + 64;
    static_assert(L % 2 == 0 && L >= 2 && L <= 16, "even filter length <= 16");
    static_assert(8 * 7 + 4 * NVC4 <= CP, "row pass reads past the staged tile");
};

template <int L, bool USE_TMA>
__global__ void __launch_bounds__(256, 3)
inv2d_strip_kernel(const __grid_constant__ Inv2dParams p, const __grid_constant__ Inv2dMaps maps) {
    using Gm = Inv2dGeom<L>;
    constexpr int HALF = Gm::HALF, TWO = Gm::TWO, CP = Gm::CP, CR = Gm::CR, RING = Gm::RING, MIR = Gm::MIR;
    constexpr int RP = Gm::RP, NT = Gm::NT, NVC4 = Gm::NVC4;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_in = reinterpret_cast<float*>(smem_raw);                 // [2][4][CR][CP]
    float* s_l = s_in + 2 * 4 * CR * CP;                              // Lh ring [RING + MIR][RP]
    float* s_h = s_l + (RING + MIR) * RP;                             // Hh ring
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_h + (RING + MIR) * RP);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = p.batch0 + blockIdx.z;
    const int X0 = blockIdx.x * TWO;                  // first output column of the strip
    const int T0 = blockIdx.y * p.seg_rows;           // first output row of the segment (even)
    if (T0 >= p.OH) return;
    const int T1 = min(T0 + p.seg_rows, p.OH);
    const int S0 = T0 / 2, S1 = (T1 + 1) / 2;         // output row pairs [S0, S1)
    const int rb = S0;                                // first coefficient row staged
    const int sb = S0 - (HALF - 1);                   // chunk c yields row pairs [sb + 16 c, sb + 16 c + 16)
    const int nchunks = (S1 - sb + CR - 1) / CR;
    const int c0 = X0 / 2;                            // first coefficient column staged

    if (USE_TMA) {
        if (tid == 0) {
            for (int k = 0; k < 4; ++k) tma_prefetch_desc(&maps.m[k]);
            mbar_init(&bars[0], 1);
            mbar_init(&bars[1], 1);
            fence_mbar_init();
        }
        __syncthreads();
        if (tid == 0) {
            for (int s = 0; s < 2 && s < nchunks; ++s) {
                mbar_expect_tx(&bars[s], (uint32_t)Gm::STAGE_BYTES);
                for (int k = 0; k < 4; ++k)
                    tma_load_3d(s_in + (s * 4 + k) * CR * CP, &maps.m[k], &bars[s], c0, rb + s * CR, b);
            }
        }
    }

    // per-thread constants of the column pass: 8 row groups (4 output rows each) x 32 column groups
    const int rg = tid >> 5, cg = tid & 31;
    const int gx = X0 + 4 * cg;
    const bool col_ok = gx < p.OW;
    float* ybase = p.y + (int64_t)b * p.y_bs + gx;

    int ring_base = 0;
    for (int c = 0; c < nchunks; ++c) {
        const int stage = c & 1;
        float* tile = s_in + stage * 4 * CR * CP;
        const int r_base = rb + c * CR;
        if (USE_TMA) {
            mbar_wait(&bars[stage], (uint32_t)((c >> 1) & 1));
        } else {
            for (int idx = tid; idx < 4 * CR * CP; idx += NT) {
                const int k = idx / (CR * CP), r2 = idx - k * (CR * CP);
                const int rr = r2 / CP, cc = r2 - rr * CP;
                const int gr = r_base + rr, gc = c0 + cc;
                float v = 0.f;
                if (gr >= 0 && gr < p.Mh && gc < p.Mw)
                    v = __ldg(p.in[k] + (int64_t)b * p.in_bs[k] + (int64_t)gr * p.in_rs[k] + gc);
                tile[idx] = v;
            }
            __syncthreads();
        }

        // ---- row pass: synthesis along W --------------------------------------------------------
        {
            const int pair = lane >> 4, row = lane & 15;          // pair 0: (k0, k1) -> Lh; pair 1: (k2, k3) -> Hh
            const float* a = tile + (2 * pair) * CR * CP + row * CP + 8 * warp;        // lo_W band
            const float* d = tile + (2 * pair + 1) * CR * CP + row * CP + 8 * warp;    // hi_W band
            float va[4 * NVC4], vd[4 * NVC4];
#pragma unroll
            for (int q = 0; q < NVC4; ++q) {
                const float4 t = *reinterpret_cast<const float4*>(a + 4 * q);
                va[4 * q] = t.x; va[4 * q + 1] = t.y; va[4 * q + 2] = t.z; va[4 * q + 3] = t.w;
                const float4 u = *reinterpret_cast<const float4*>(d + 4 * q);
                vd[4 * q] = u.x; vd[4 * q + 1] = u.y; vd[4 * q + 2] = u.z; vd[4 * q + 3] = u.w;
            }
            float o[16];
#pragma unroll
            for (int s = 0; s < 8; ++s) {
                float e0 = 0.f, e1 = 0.f;
#pragma unroll
                for (int j = 0; j < HALF; ++j) {
                    e0 = fmaf(p.rlo[L - 2 - 2 * j], va[s + j], e0);
                    e0 = fmaf(p.rhi[L - 2 - 2 * j], vd[s + j], e0);
                    e1 = fmaf(p.rlo[L - 1 - 2 * j], va[s + j], e1);
                    e1 = fmaf(p.rhi[L - 1 - 2 * j], vd[s + j], e1);
                }
                o[2 * s] = e0; o[2 * s + 1] = e1;
            }
            int slot = ring_base + row;
            if (slot >= RING) slot -= RING;
            float* dst = (pair ? s_h : s_l) + slot * RP + 16 * warp;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float4 t = make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
                *reinterpret_cast<float4*>(dst + 4 * q) = t;
                if (slot < MIR) *reinterpret_cast<float4*>(dst + RING * RP + 4 * q) = t;
            }
        }
        __syncthreads();

        if (USE_TMA && tid == 0 && c + 2 < nchunks) {
            fence_proxy_async();
            mbar_expect_tx(&bars[stage], (uint32_t)Gm::STAGE_BYTES);
            for (int k = 0; k < 4; ++k)
                tma_load_3d(tile + k * CR * CP, &maps.m[k], &bars[stage], c0, rb + (c + 2) * CR, b);
        }

        // ---- column pass: synthesis along H, 4 output rows x 4 columns per thread ------------------
        {
            int row0 = ring_base + 2 * rg - (HALF - 1);       // ring row of coefficient row s
            if (row0 < 0) row0 += RING;
            else if (row0 >= RING) row0 -= RING;
            const float* pl = s_l + row0 * RP + 4 * cg;
            const float* ph = s_h + row0 * RP + 4 * cg;
            float2 acc[4][2];
#pragma unroll
            for (int r = 0; r < 4; ++r) { acc[r][0] = make_float2(0.f, 0.f); acc[r][1] = make_float2(0.f, 0.f); }
#pragma unroll
            for (int m = 0; m <= HALF; ++m) {
                const float4 fl = *reinterpret_cast<const float4*>(pl + m * RP);
                const float4 fh = *reinterpret_cast<const float4*>(ph + m * RP);
                const float2 l0 = make_float2(fl.x, fl.y), l1 = make_float2(fl.z, fl.w);
                const float2 h0 = make_float2(fh.x, fh.y), h1 = make_float2(fh.z, fh.w);
                if (m < HALF) {       // rows 2s, 2s+1: j = m
                    acc[0][0] = ffma2(p.bl[L - 2 - 2 * m], l0, acc[0][0]); acc[0][1] = ffma2(p.bl[L - 2 - 2 * m], l1, acc[0][1]);
                    acc[0][0] = ffma2(p.bh[L - 2 - 2 * m], h0, acc[0][0]); acc[0][1] = ffma2(p.bh[L - 2 - 2 * m], h1, acc[0][1]);
                    acc[1][0] = ffma2(p.bl[L - 1 - 2 * m], l0, acc[1][0]); acc[1][1] = ffma2(p.bl[L - 1 - 2 * m], l1, acc[1][1]);
                    acc[1][0] = ffma2(p.bh[L - 1 - 2 * m], h0, acc[1][0]); acc[1][1] = ffma2(p.bh[L - 1 - 2 * m], h1, acc[1][1]);
                }
                if (m >= 1) {         // rows 2(s+1), 2(s+1)+1: j = m - 1
                    acc[2][0] = ffma2(p.bl[L - 2 * m], l0, acc[2][0]); acc[2][1] = ffma2(p.bl[L - 2 * m], l1, acc[2][1]);
                    acc[2][0] = ffma2(p.bh[L - 2 * m], h0, acc[2][0]); acc[2][1] = ffma2(p.bh[L - 2 * m], h1, acc[2][1]);
                    acc[3][0] = ffma2(p.bl[L + 1 - 2 * m], l0, acc[3][0]); acc[3][1] = ffma2(p.bl[L + 1 - 2 * m], l1, acc[3][1]);
                    acc[3][0] = ffma2(p.bh[L + 1 - 2 * m], h0, acc[3][0]); acc[3][1] = ffma2(p.bh[L + 1 - 2 * m], h1, acc[3][1]);
                }
            }
            if (col_ok) {
                const int s = sb + c * CR + 2 * rg;           // first row pair of this thread
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int ty = 2 * s + r;
                    if (ty < T0 || ty >= T1) continue;
                    float* dst = ybase + (int64_t)ty * p.y_rs;
                    if (p.vec_store) {
                        *reinterpret_cast<float4*>(dst) = make_float4(acc[r][0].x, acc[r][0].y, acc[r][1].x, acc[r][1].y);
                    } else {
                        const float a4[4] = {acc[r][0].x, acc[r][0].y, acc[r][1].x, acc[r][1].y};
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            if (gx + e < p.OW) dst[e] = a4[e];
                    }
                }
            }
        }
        __syncthreads();
        ring_base += CR;
        if (ring_base >= RING) ring_base -= RING;
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// Synthesis level of OH x OW outputs per image, B images per launch.  Segments of 32 k - 2 (HALF - 1) output rows keep
// the chunking free of an idle tail; small levels get shorter ones so that the grid still fills the machine.
static StripGrid inv2d_grid(int64_t OH, int64_t OW, int64_t B, int L) {
    const int H1 = L / 2 - 1;   // Inv2dGeom::HALF - 1
    const int64_t nstrip = (OW + INV2D_TWO - 1) / INV2D_TWO;
    int64_t nseg = (OH + 511) / 512;
    while (nseg * nstrip * B < 4 * 444 && (OH + nseg - 1) / nseg > 96) ++nseg;
    int64_t seg = ((OH + nseg - 1) / nseg + 2 * H1 + 31) / 32 * 32 - 2 * H1;
    if (seg < 2) seg = 2;
    return {(int)nstrip, (int)((OH + seg - 1) / seg), (int)seg};
}

template <int L>
static cudaError_t launch_inv2d_level(const float* const in[4], const int64_t in_bs[4], const int64_t in_rs[4], int64_t B,
                                      int Mh, int Mw, float* y, int64_t y_bs, int64_t y_rs, int OH, int OW,
                                      const double* rlo, const double* rhi, cudaStream_t st, uint64_t* launches) {
    using Gm = Inv2dGeom<L>;
    Inv2dParams p;
    Inv2dMaps maps;
    memset(&maps, 0, sizeof(maps));
    bool tma = true;
    for (int k = 0; k < 4; ++k) {
        p.in[k] = in[k]; p.in_bs[k] = in_bs[k]; p.in_rs[k] = in_rs[k];
        if (tma) tma = make_tmap_3d<float>(&maps.m[k], in[k], B, Mh, Mw, in_bs[k], in_rs[k], Gm::CP, Gm::CR);
    }
    p.y = y; p.y_bs = y_bs; p.y_rs = y_rs;
    p.Mh = Mh; p.Mw = Mw; p.OH = OH; p.OW = OW;
    for (int k = 0; k < L; ++k) {
        p.rlo[k] = (float)rlo[k]; p.rhi[k] = (float)rhi[k];
        p.bl[k] = make_float2((float)rlo[k], (float)rlo[k]);
        p.bh[k] = make_float2((float)rhi[k], (float)rhi[k]);
    }
    p.vec_store = !(((uintptr_t)y & 15) || (y_bs & 3) || (y_rs & 3) || y_rs < (OW + 3) / 4 * 4);
    const StripGrid g = inv2d_grid(OH, OW, B, L);
    assert(g.nseg <= 65535 && "dwt_route sends levels whose segments overflow gridDim.y to the general path");
    p.seg_rows = g.seg;
    auto kern = tma ? inv2d_strip_kernel<L, true> : inv2d_strip_kernel<L, false>;
    cudaError_t e = ensure_dyn_smem(kern, (size_t)Gm::SMEM);
    if (e != cudaSuccess) return e;
    for (int64_t b0 = 0; b0 < B; b0 += 65535) {
        p.batch0 = (int)b0;
        const int nb = (int)((B - b0) < 65535 ? (B - b0) : 65535);
        dim3 grid(g.nstrip, g.nseg, nb);
        kern<<<grid, Gm::NT, Gm::SMEM, st>>>(p, maps);
        ++*launches;
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// All levels of a float32 2-D synthesis on the strip kernel (dwt_route chose it).
static int fused2d_inv(int levels, int L, const double* rlo, const double* rhi, float* y, int64_t batch,
                       const int64_t* out_dims, const int64_t* ys, int64_t ybs, const wt_level* lv, cudaStream_t st) {
    uint64_t launches = 0;
    for (int l = levels - 1; l >= 0; --l) {
        const wt_level& d = lv[l];
        const float* in[4];
        int64_t ibs[4], irs[4];
        in[0] = (const float*)d.approx; ibs[0] = d.approx_batch_stride; irs[0] = d.approx_strides[0];
        for (int k = 1; k < 4; ++k) {
            in[k] = (const float*)d.details + (int64_t)(k - 1) * d.band_stride;
            ibs[k] = d.details_batch_stride; irs[k] = d.strides[0];
        }
        float* dst; int64_t dbs, drs; int OH, OW;
        if (l > 0) {
            dst = (float*)lv[l - 1].approx; dbs = lv[l - 1].approx_batch_stride; drs = lv[l - 1].approx_strides[0];
            OH = (int)lv[l - 1].dims[0]; OW = (int)lv[l - 1].dims[1];
        } else {
            dst = y; dbs = ybs; drs = ys[0]; OH = (int)out_dims[0]; OW = (int)out_dims[1];
        }
        cudaError_t e = cudaSuccess;
#define WTB_I2D_CASE(LL)                                                                                         \
    case LL:                                                                                                     \
        e = launch_inv2d_level<LL>(in, ibs, irs, batch, (int)d.dims[0], (int)d.dims[1], dst, dbs, drs, OH, OW, rlo, rhi, st, \
                                   &launches);                                                                   \
        break;
        switch (L) {
            WTB_I2D_CASE(2) WTB_I2D_CASE(4) WTB_I2D_CASE(6) WTB_I2D_CASE(8)
            WTB_I2D_CASE(10) WTB_I2D_CASE(12) WTB_I2D_CASE(14) WTB_I2D_CASE(16)
            default: return 0;
        }
#undef WTB_I2D_CASE
        g_launches.fetch_add(launches, std::memory_order_relaxed);
        launches = 0;
        if (e != cudaSuccess) return cuda_fail(e, "inv2d_strip_kernel");
    }
    return 0;
}

}  // namespace wtb
