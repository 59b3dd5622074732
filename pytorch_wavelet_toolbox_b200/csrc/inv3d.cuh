// inv3d.cuh -- one 3-D synthesis level as ONE kernel (float32): coefficient planes streamed along D.
//
// Replaces the reference's  stack(8 bands) -> conv_transpose3d(8 x [L x L x L], stride 2) -> crop
// (src/ptwt/conv_transform_3.py:205-249): the eight sub-bands are read once, the reconstruction is
// written once, no stacked copy and no uncropped intermediate.
//
//   * a CTA owns a 16 x 64 tile of the (H, W) output plane (8+L/2-1 x 32+L/2-1 coefficients) and a
//     segment of output planes; it consumes coefficient planes one by one (4-D TMA, one tensor map per
//     band, out-of-range = zero fill -- transposed convolutions have no boundary extension);
//   * per coefficient plane: synthesis along W (8 bands -> 4 arrays), synthesis along H (-> 2 arrays:
//     low / high along D) kept in a ring of L/2 planes;
//   * depth pass: the last L/2 ring planes -> two output planes, 128-bit coalesced stores.
//
// Algorithmic bytes per level: 4 B * (8 Md Mh Mw + OD OH OW).
#pragma once

#include "fwd3d.cuh"

namespace wtb {

struct Inv3dParams {
    const float* in[8];
    int64_t in_bs[8], in_ps[8], in_rs[8];
    float* y;
    int64_t y_bs, y_ps, y_rs;
    int Md, Mh, Mw, OD, OH, OW;
    int seg_pairs;           // output plane pairs per segment
    int nty;
    int vec_store;
    float rlo[16], rhi[16];
    float2 bl[16], bh[16];   // {rec_lo[k], rec_lo[k]}, {rec_hi[k], rec_hi[k]}
};

struct Inv3dMaps {
    CUtensorMap m[8];
};

constexpr int INV3D_TOH = 16, INV3D_TOW = 64;                   // output tile

template <int L>
struct Inv3dGeom {
    static constexpr int HALF = L / 2;
    static constexpr int TOH = INV3D_TOH, TOW = INV3D_TOW;
    static constexpr int CRW = TOH / 2 + HALF - 1;              // coefficient rows per tile
    static constexpr int NCC = TOW / 2 + HALF - 1;              // coefficient columns per tile
    static constexpr int CP = ((NCC - 4 + 7) / 8) * 8 + 4;      // staged pitch (== 4 mod 8)
    static constexpr int BAND_ELEMS = (CRW * CP + 31) / 32 * 32; // 128-byte aligned band tile
    static constexpr int MPW = TOW + 4;                         // pitch of the W-synthesised arrays
    static constexpr int RINGD = 4;                             // planes kept for the depth pass (>= HALF)
    static constexpr int NT = 256;
    static constexpr int NVC = 8 + HALF - 1, NVC4 = (NVC + 3) / 4;
    static constexpr size_t BAND_BYTES = (size_t)CRW * CP * 4;
    static constexpr size_t SMEM = 2 * 8 * (size_t)BAND_ELEMS * 4 + 4 * (size_t)CRW * MPW * 4 +
                                   (size_t)RINGD * 2 * TOH * TOW * 4 + 64;
    static_assert(L % 2 == 0 && L >= 2 && L <= 8, "3-D fused synthesis: even filter length <= 8");
    static_assert(HALF <= RINGD, "depth ring too small");
    static_assert(8 * 3 + 4 * NVC4 <= CP, "row pass reads past the staged tile");
};

template <int L, bool USE_TMA>
__global__ void __launch_bounds__(256, 3)
inv3d_tile_kernel(const __grid_constant__ Inv3dParams p, const __grid_constant__ Inv3dMaps maps) {
    using Gm = Inv3dGeom<L>;
    constexpr int HALF = Gm::HALF, TOH = Gm::TOH, TOW = Gm::TOW, CRW = Gm::CRW, CP = Gm::CP, BE = Gm::BAND_ELEMS;
    constexpr int MPW = Gm::MPW, RINGD = Gm::RINGD, NT = Gm::NT, NVC4 = Gm::NVC4;
    constexpr int PLANE = TOH * TOW;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_in = reinterpret_cast<float*>(smem_raw);          // [2 stages][8 bands][BE]
    float* s_w = s_in + 2 * 8 * BE;                            // [4][CRW][MPW]: index 2 d + h (d: D band, h: H band)
    float* s_ring = s_w + 4 * CRW * MPW;                       // [RINGD][2][TOH][TOW]: P_lo / P_hi (bands along D)
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_ring + RINGD * 2 * PLANE);

    const int tid = threadIdx.x;
    const int b = blockIdx.z;
    const int X0 = blockIdx.x * TOW;
    const int ty = blockIdx.y % p.nty, sg = blockIdx.y / p.nty;
    const int Y0 = ty * TOH;
    const int S0 = sg * p.seg_pairs;                           // first output plane pair
    const int npairs_total = (p.OD + 1) / 2;
    if (S0 >= npairs_total) return;
    const int S1 = min(S0 + p.seg_pairs, npairs_total);
    const int nplanes = (S1 - S0) + HALF - 1;                  // coefficient planes consumed: S0 .. S1 + HALF - 2
    const int c0 = X0 / 2, r0 = Y0 / 2;

    if (USE_TMA) {
        if (tid == 0) {
            for (int k = 0; k < 8; ++k) tma_prefetch_desc(&maps.m[k]);
            mbar_init(&bars[0], 1);
            mbar_init(&bars[1], 1);
            fence_mbar_init();
        }
        __syncthreads();
        if (tid == 0) {
            for (int s = 0; s < 2 && s < nplanes; ++s) {
                mbar_expect_tx(&bars[s], (uint32_t)(8 * Gm::BAND_BYTES));
                for (int k = 0; k < 8; ++k) tma_load_4d(s_in + (s * 8 + k) * BE, &maps.m[k], &bars[s], c0, r0, S0 + s, b);
            }
        }
    }

    for (int t = 0; t < nplanes; ++t) {
        const int z = S0 + t;                                  // coefficient plane index
        const int stage = t & 1;
        float* tile = s_in + stage * 8 * BE;
        if (USE_TMA) {
            mbar_wait(&bars[stage], (uint32_t)((t >> 1) & 1));
        } else {
            for (int idx = tid; idx < 8 * CRW * CP; idx += NT) {
                const int k = idx / (CRW * CP), r2 = idx - k * (CRW * CP);
                const int rr = r2 / CP, cc = r2 - rr * CP;
                const int gr = r0 + rr, gc = c0 + cc;
                float v = 0.f;
                if (z < p.Md && gr < p.Mh && gc < p.Mw)
                    v = __ldg(p.in[k] + (int64_t)b * p.in_bs[k] + (int64_t)z * p.in_ps[k] + (int64_t)gr * p.in_rs[k] + gc);
                tile[k * BE + rr * CP + cc] = v;
            }
            __syncthreads();
        }

        // ---- synthesis along W: (pair = 2 d + h, coefficient row, group of 16 outputs) ---------------
        for (int item = tid; item < 4 * CRW * (TOW / 16); item += NT) {
            const int row = item % CRW, rest = item / CRW;
            const int pair = rest & 3, grp = rest >> 2;
            // bands of the pair: k = 4 d + 2 h + w ; pair = 2 d + h
            const float* a = tile + (2 * pair) * BE + row * CP + 8 * grp;         // lo along W
            const float* d = tile + (2 * pair + 1) * BE + row * CP + 8 * grp;     // hi along W
            float va[4 * NVC4], vd[4 * NVC4];
#pragma unroll
            for (int q = 0; q < NVC4; ++q) {
                const float4 f = *reinterpret_cast<const float4*>(a + 4 * q);
                va[4 * q] = f.x; va[4 * q + 1] = f.y; va[4 * q + 2] = f.z; va[4 * q + 3] = f.w;
                const float4 g = *reinterpret_cast<const float4*>(d + 4 * q);
                vd[4 * q] = g.x; vd[4 * q + 1] = g.y; vd[4 * q + 2] = g.z; vd[4 * q + 3] = g.w;
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
            float* dst = s_w + pair * CRW * MPW + row * MPW + 16 * grp;
#pragma unroll
            for (int q = 0; q < 4; ++q)
                *reinterpret_cast<float4*>(dst + 4 * q) = make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
        }
        __syncthreads();

        if (USE_TMA && tid == 0 && t + 2 < nplanes) {
            fence_proxy_async();
            mbar_expect_tx(&bars[stage], (uint32_t)(8 * Gm::BAND_BYTES));
            for (int k = 0; k < 8; ++k) tma_load_4d(tile + k * BE, &maps.m[k], &bars[stage], c0, r0, S0 + t + 2, b);
        }

        // ---- synthesis along H: (d, 4 output rows, 4 columns) -> ring plane z -----------------------
        if (tid < 2 * (TOH / 4) * (TOW / 4)) {
            const int dd = tid / ((TOH / 4) * (TOW / 4));
            const int rem = tid - dd * ((TOH / 4) * (TOW / 4));
            const int rg = rem / (TOW / 4), cg = rem - rg * (TOW / 4);
            const float* pl = s_w + (2 * dd) * CRW * MPW + (2 * rg) * MPW + 4 * cg;       // low along H
            const float* ph = s_w + (2 * dd + 1) * CRW * MPW + (2 * rg) * MPW + 4 * cg;   // high along H
            float2 acc[4][2];
#pragma unroll
            for (int r = 0; r < 4; ++r) { acc[r][0] = make_float2(0.f, 0.f); acc[r][1] = make_float2(0.f, 0.f); }
#pragma unroll
            for (int m = 0; m <= HALF; ++m) {
                const float4 fl = *reinterpret_cast<const float4*>(pl + m * MPW);
                const float4 fh = *reinterpret_cast<const float4*>(ph + m * MPW);
                const float2 l0 = make_float2(fl.x, fl.y), l1 = make_float2(fl.z, fl.w);
                const float2 h0 = make_float2(fh.x, fh.y), h1 = make_float2(fh.z, fh.w);
                if (m < HALF) {
                    acc[0][0] = ffma2(p.bl[L - 2 - 2 * m], l0, acc[0][0]); acc[0][1] = ffma2(p.bl[L - 2 - 2 * m], l1, acc[0][1]);
                    acc[0][0] = ffma2(p.bh[L - 2 - 2 * m], h0, acc[0][0]); acc[0][1] = ffma2(p.bh[L - 2 - 2 * m], h1, acc[0][1]);
                    acc[1][0] = ffma2(p.bl[L - 1 - 2 * m], l0, acc[1][0]); acc[1][1] = ffma2(p.bl[L - 1 - 2 * m], l1, acc[1][1]);
                    acc[1][0] = ffma2(p.bh[L - 1 - 2 * m], h0, acc[1][0]); acc[1][1] = ffma2(p.bh[L - 1 - 2 * m], h1, acc[1][1]);
                }
                if (m >= 1) {
                    acc[2][0] = ffma2(p.bl[L - 2 * m], l0, acc[2][0]); acc[2][1] = ffma2(p.bl[L - 2 * m], l1, acc[2][1]);
                    acc[2][0] = ffma2(p.bh[L - 2 * m], h0, acc[2][0]); acc[2][1] = ffma2(p.bh[L - 2 * m], h1, acc[2][1]);
                    acc[3][0] = ffma2(p.bl[L + 1 - 2 * m], l0, acc[3][0]); acc[3][1] = ffma2(p.bl[L + 1 - 2 * m], l1, acc[3][1]);
                    acc[3][0] = ffma2(p.bh[L + 1 - 2 * m], h0, acc[3][0]); acc[3][1] = ffma2(p.bh[L + 1 - 2 * m], h1, acc[3][1]);
                }
            }
            float* rp = s_ring + ((z & (RINGD - 1)) * 2 + dd) * PLANE + (4 * rg) * TOW + 4 * cg;
#pragma unroll
            for (int r = 0; r < 4; ++r)
                *reinterpret_cast<float4*>(rp + r * TOW) = make_float4(acc[r][0].x, acc[r][0].y, acc[r][1].x, acc[r][1].y);
        }
        __syncthreads();

        // ---- depth pass: planes z-HALF+1 .. z -> output planes 2 s, 2 s + 1 with s = z - HALF + 1 ---
        if (t >= HALF - 1) {
            const int s = z - (HALF - 1);
            const int row = tid >> 4, cg = tid & 15;
            float2 e0[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
            float2 e1[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
#pragma unroll
            for (int j = 0; j < HALF; ++j) {
                const float* rp = s_ring + (((s + j) & (RINGD - 1)) * 2) * PLANE + row * TOW + 4 * cg;
                const float4 fl = *reinterpret_cast<const float4*>(rp);
                const float4 fh = *reinterpret_cast<const float4*>(rp + PLANE);
                const float2 l0 = make_float2(fl.x, fl.y), l1 = make_float2(fl.z, fl.w);
                const float2 h0 = make_float2(fh.x, fh.y), h1 = make_float2(fh.z, fh.w);
                e0[0] = ffma2(p.bl[L - 2 - 2 * j], l0, e0[0]); e0[1] = ffma2(p.bl[L - 2 - 2 * j], l1, e0[1]);
                e0[0] = ffma2(p.bh[L - 2 - 2 * j], h0, e0[0]); e0[1] = ffma2(p.bh[L - 2 - 2 * j], h1, e0[1]);
                e1[0] = ffma2(p.bl[L - 1 - 2 * j], l0, e1[0]); e1[1] = ffma2(p.bl[L - 1 - 2 * j], l1, e1[1]);
                e1[0] = ffma2(p.bh[L - 1 - 2 * j], h0, e1[0]); e1[1] = ffma2(p.bh[L - 1 - 2 * j], h1, e1[1]);
            }
            const int gy = Y0 + row, gx = X0 + 4 * cg;
            if (gy < p.OH && gx < p.OW) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int tz = 2 * s + e;
                    if (tz >= p.OD) continue;
                    float* dst = p.y + (int64_t)b * p.y_bs + (int64_t)tz * p.y_ps + (int64_t)gy * p.y_rs + gx;
                    const float2 a0 = e ? e1[0] : e0[0], a1 = e ? e1[1] : e0[1];
                    if (p.vec_store) {
                        *reinterpret_cast<float4*>(dst) = make_float4(a0.x, a0.y, a1.x, a1.y);
                    } else {
                        const float v4[4] = {a0.x, a0.y, a1.x, a1.y};
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            if (gx + q < p.OW) dst[q] = v4[q];
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// Synthesis level of OD x OH x OW outputs per volume: segments along depth only while the grid would not fill the
// machine a few times.
static TileGrid3d inv3d_grid(int64_t OD, int64_t OH, int64_t OW, int64_t B) {
    const int64_t ntx = (OW + INV3D_TOW - 1) / INV3D_TOW, nty = (OH + INV3D_TOH - 1) / INV3D_TOH, npairs = (OD + 1) / 2;
    int64_t nseg = 1;
    while (nseg * ntx * nty * B < 4 * 296 && (npairs + nseg - 1) / nseg > 16) ++nseg;
    const int64_t seg = (npairs + nseg - 1) / nseg;
    return {(int)ntx, (int)nty, (int)((npairs + seg - 1) / seg), (int)seg};
}

template <int L>
static cudaError_t launch_inv3d_level(const wt_level& d, int64_t B, float* y, int64_t y_bs, int64_t y_ps, int64_t y_rs, int OD,
                                      int OH, int OW, const double* rlo, const double* rhi, cudaStream_t st, uint64_t* launches) {
    using Gm = Inv3dGeom<L>;
    Inv3dParams p;
    Inv3dMaps maps;
    memset(&maps, 0, sizeof(maps));
    p.Md = (int)d.dims[0]; p.Mh = (int)d.dims[1]; p.Mw = (int)d.dims[2];
    bool tma = true;
    for (int k = 0; k < 8; ++k) {
        if (k == 0) {
            p.in[0] = (const float*)d.approx; p.in_bs[0] = d.approx_batch_stride; p.in_ps[0] = d.approx_strides[0]; p.in_rs[0] = d.approx_strides[1];
        } else {
            p.in[k] = (const float*)d.details + (int64_t)(k - 1) * d.band_stride;
            p.in_bs[k] = d.details_batch_stride; p.in_ps[k] = d.strides[0]; p.in_rs[k] = d.strides[1];
        }
        if (tma) tma = make_tmap_4d(&maps.m[k], p.in[k], B, p.Md, p.Mh, p.Mw, p.in_bs[k], p.in_ps[k], p.in_rs[k], Gm::CP, Gm::CRW);
    }
    p.y = y; p.y_bs = y_bs; p.y_ps = y_ps; p.y_rs = y_rs;
    p.OD = OD; p.OH = OH; p.OW = OW;
    for (int k = 0; k < L; ++k) {
        p.rlo[k] = (float)rlo[k]; p.rhi[k] = (float)rhi[k];
        p.bl[k] = make_float2((float)rlo[k], (float)rlo[k]);
        p.bh[k] = make_float2((float)rhi[k], (float)rhi[k]);
    }
    p.vec_store = !(((uintptr_t)y & 15) || (y_bs & 3) || (y_ps & 3) || (y_rs & 3) || y_rs < (OW + 3) / 4 * 4);
    const TileGrid3d g = inv3d_grid(OD, OH, OW, B);
    assert(g.fits(B) && "dwt_route sends levels whose tiles overflow the grid to the general path");
    p.seg_pairs = g.seg;
    p.nty = g.nty;
    auto kern = tma ? inv3d_tile_kernel<L, true> : inv3d_tile_kernel<L, false>;
    cudaError_t e = ensure_dyn_smem(kern, (size_t)Gm::SMEM);
    if (e != cudaSuccess) return e;
    dim3 grid(g.ntx, g.nty * g.nseg, (unsigned)B);
    kern<<<grid, Gm::NT, Gm::SMEM, st>>>(p, maps);
    ++*launches;
    return cudaGetLastError();
}

// All levels of a float32 3-D synthesis on the tile kernel (dwt_route chose it).
static int fused3d_inv(int levels, int L, const double* rlo, const double* rhi, float* y, int64_t batch,
                       const int64_t* out_dims, const int64_t* ys, int64_t ybs, const wt_level* lv, cudaStream_t st) {
    uint64_t launches = 0;
    for (int l = levels - 1; l >= 0; --l) {
        float* dst; int64_t dbs, dps, drs; int OD, OH, OW;
        if (l > 0) {
            dst = (float*)lv[l - 1].approx; dbs = lv[l - 1].approx_batch_stride; dps = lv[l - 1].approx_strides[0]; drs = lv[l - 1].approx_strides[1];
            OD = (int)lv[l - 1].dims[0]; OH = (int)lv[l - 1].dims[1]; OW = (int)lv[l - 1].dims[2];
        } else {
            dst = y; dbs = ybs; dps = ys[0]; drs = ys[1]; OD = (int)out_dims[0]; OH = (int)out_dims[1]; OW = (int)out_dims[2];
        }
        cudaError_t e;
        switch (L) {
            case 2: e = launch_inv3d_level<2>(lv[l], batch, dst, dbs, dps, drs, OD, OH, OW, rlo, rhi, st, &launches); break;
            case 4: e = launch_inv3d_level<4>(lv[l], batch, dst, dbs, dps, drs, OD, OH, OW, rlo, rhi, st, &launches); break;
            case 6: e = launch_inv3d_level<6>(lv[l], batch, dst, dbs, dps, drs, OD, OH, OW, rlo, rhi, st, &launches); break;
            case 8: e = launch_inv3d_level<8>(lv[l], batch, dst, dbs, dps, drs, OD, OH, OW, rlo, rhi, st, &launches); break;
            default: return 0;
        }
        g_launches.fetch_add(launches, std::memory_order_relaxed);
        launches = 0;
        if (e != cudaSuccess) return cuda_fail(e, "inv3d_tile_kernel");
    }
    return 0;
}

}  // namespace wtb
