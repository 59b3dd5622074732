// fwd3d.cuh -- one 3-D analysis level as ONE kernel (float32): in-plane tiles streamed along the
// slowest axis.
//
// Replaces the reference's  F.pad -> conv3d(8 x [L x L x L], stride 2) -> split
// (src/ptwt/conv_transform_3.py:122-141): the input volume is read once and the eight sub-bands are
// written once; the reference's L^3 = 512 MACs per output collapse to 3 L = 24 (separable).
//
//   * a CTA owns a TH x TW tile of the (H, W) output plane (16 x 32, 11 x 44 or 8 x 64 -- the host picks
//     the shape that wastes the fewest computed-but-discarded outputs, e.g. 11 x 44 for the 131 x 131
//     planes of a 256^3 volume with an 8-tap filter) and a segment of output planes; it consumes the
//     input volume plane by plane (axis D), each plane tile [2 TH + L-2, 2 TW + HAL] staged by a 4-D TMA
//     tensor map over [batch, D, H, W] (out-of-range = zero fill = ptwt's default "zero" mode of
//     wavedec3; other modes patch the halo in-kernel / redirect the plane index);
//   * per input plane: row pass (along W) into a double-buffered pair of shared arrays, ONE barrier,
//     column pass (along H) by the thread that owns the (row, 4-column) result;
//   * that thread also owns the result along D: the last 8 planes of its two float4 results live in
//     registers (fixed slots, the TAPS rotate instead of the data), so the depth pass reads no shared
//     memory; every second plane it emits low / high along D -> all eight sub-bands of one output
//     plane, 128-bit stores.  Nothing but input and output touches HBM.
//
// Algorithmic bytes per level: 4 B * (D H W + 8 Md Mh Mw).
#pragma once

#include "fused2d.cuh"

namespace wtb {

struct Fwd3dParams {
    const float* x;              // [batch, D, H, W]
    int64_t x_bs, x_ps, x_rs;    // element strides: batch, plane, row
    float* out[8];               // sub-bands k = 4 hD + 2 hH + hW
    int64_t out_bs[8], out_ps[8], out_rs[8];
    int D, H, W, Md, Mh, Mw;
    int seg_planes;              // output planes per segment
    int mode;
    int nty;                     // tiles along H (blockIdx.y = segment * nty + tile)
    int vec_store;
    float2 pl[8], ph[8], bl[16], bh[16];
    float2 dl[8], dh[8];         // depth taps {c, c}, zero-padded to the 8-plane register window
};

template <int L, int TH_, int TW_>
struct Fwd3dGeom {
    static constexpr int HALO = L - 2;
    static constexpr int HAL = (HALO + 3) / 4 * 4;
    static constexpr int OFF = HAL - HALO;
    static constexpr int TH = TH_, TW = TW_;
    static constexpr int TW4 = TW / 4;                            // float4 column groups of the tile
    static constexpr int NG8 = (TW + 7) / 8;                      // row-pass groups of 8 outputs
    static constexpr int ROWS = 2 * TH + HALO;                    // staged tile rows
    static constexpr int NV4 = (16 + HAL + 3) / 4;                // float4 loads of one row-pass item
    static constexpr int NEED = 16 * (NG8 - 1) + 4 * NV4;         // columns the row pass touches (>= 2 TW + HAL)
    static constexpr int SW = ((NEED - 4 + 7) / 8) * 8 + 4;       // staged pitch, == 4 (mod 8)
    static constexpr int MP = 8 * NG8 + 4;                        // pitch of the row-filtered arrays, == 4 (mod 8)
    static constexpr int NSTAGE = 3;
    static constexpr int NT = 256;
    static constexpr size_t STAGE_BYTES = (size_t)ROWS * SW * 4;               // bytes one TMA box delivers
    static constexpr int STAGE_ELEMS = (ROWS * SW + 31) / 32 * 32;            // stage stride: 128-byte aligned
    static constexpr size_t SMEM = NSTAGE * (size_t)STAGE_ELEMS * 4 + 4 * (size_t)ROWS * MP * 4 + 64;
    static_assert(L % 2 == 0 && L >= 2 && L <= 8, "3-D fused path: even filter length <= 8");
    static_assert(TW % 4 == 0 && 2 * TH * TW4 <= NT, "one (band, row, 4-column) item per thread");
    static_assert(NEED >= 2 * TW + HAL && SW <= 256, "staged tile too narrow / TMA box too wide");
};

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

template <int L, int TH_, int TW_, bool USE_TMA>
__global__ void __launch_bounds__(256, 2)
fwd3d_tile_kernel(const __grid_constant__ Fwd3dParams p, const __grid_constant__ CUtensorMap tmap) {
    using Gm = Fwd3dGeom<L, TH_, TW_>;
    constexpr int HALO = Gm::HALO, HAL = Gm::HAL, OFF = Gm::OFF, TH = Gm::TH, TW = Gm::TW, ROWS = Gm::ROWS;
    constexpr int SW = Gm::SW, MP = Gm::MP, NSTAGE = Gm::NSTAGE, NT = Gm::NT, NV4 = Gm::NV4;
    constexpr int SE = Gm::STAGE_ELEMS, TW4 = Gm::TW4, NG8 = Gm::NG8;
    constexpr int WN = 8;                                          // register window (planes), >= L

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_in = reinterpret_cast<float*>(smem_raw);              // [NSTAGE][ROWS][SW]
    float* s_row = s_in + NSTAGE * SE;                             // [2 buffers][lo | hi][ROWS][MP]
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_row + 4 * ROWS * MP);

    const int tid = threadIdx.x;
    const int b = blockIdx.z;
    const int x0 = blockIdx.x * TW;
    const int ty = blockIdx.y % p.nty, sg = blockIdx.y / p.nty;
    const int y0 = ty * TH;
    const int z0 = sg * p.seg_planes;
    if (z0 >= p.Md) return;
    const int z1 = min(z0 + p.seg_planes, p.Md);
    const int q0 = 2 * z0 - HALO;
    const int nplanes = 2 * (z1 - z0) + HALO;
    const int c_in0 = 2 * x0 - HAL, r_in0 = 2 * y0 - HALO;
    const int c_need1 = 2 * min(x0 + TW, p.Mw), r_need1 = 2 * min(y0 + TH, p.Mh);

    auto plane_src = [&](int q) -> int {
        if (q >= 0 && q < p.D) return q;
        if (p.mode == WT_MODE_ZERO) return q;
        return ext_index32(q, p.D, p.mode);
    };

    if (USE_TMA) {
        if (tid == 0) {
            tma_prefetch_desc(&tmap);
            for (int s = 0; s < NSTAGE; ++s) mbar_init(&bars[s], 1);
            fence_mbar_init();
        }
        __syncthreads();
        if (tid == 0) {
            for (int s = 0; s < NSTAGE - 1 && s < nplanes; ++s) {
                mbar_expect_tx(&bars[s], (uint32_t)Gm::STAGE_BYTES);
                tma_load_4d(s_in + s * SE, &tmap, &bars[s], c_in0, r_in0, plane_src(q0 + s), b);
            }
        }
    }
    const float* __restrict__ xb = p.x + (int64_t)b * p.x_bs;

    // column / depth item of this thread: (array half = W band, output row, 4-column group)
    const bool owner = tid < 2 * TH * TW4;
    const int cp_half = owner ? tid / (TH * TW4) : 0;
    const int cp_row = owner ? (tid % (TH * TW4)) / TW4 : 0, cp_cg = tid % TW4;
    const int gy = y0 + cp_row, gx = x0 + 4 * cp_cg;
    const bool live = owner && gy < p.Mh && gx < p.Mw;
    // window slot k holds {low-H.xy, low-H.zw, high-H.xy, high-H.zw} of plane index == k (mod 8)
    float2 win[WN][4];
#pragma unroll
    for (int k = 0; k < WN; ++k)
#pragma unroll
        for (int i = 0; i < 4; ++i) win[k][i] = make_float2(0.f, 0.f);

    for (int t = 0; t < nplanes; ++t) {
        const int q = q0 + t;
        const int stage = t % NSTAGE;
        float* tile = s_in + stage * SE;
        float* s_lo = s_row + (t & 1) * 2 * ROWS * MP;
        float* s_hi = s_lo + ROWS * MP;
        if (USE_TMA) {
            if (tid == 0 && t + NSTAGE - 1 < nplanes) {
                const int tn = t + NSTAGE - 1, sn = tn % NSTAGE;
                fence_proxy_async();
                mbar_expect_tx(&bars[sn], (uint32_t)Gm::STAGE_BYTES);
                tma_load_4d(s_in + sn * SE, &tmap, &bars[sn], c_in0, r_in0, plane_src(q0 + tn), b);
            }
            mbar_wait(&bars[stage], (uint32_t)((t / NSTAGE) & 1));
            if (p.mode != WT_MODE_ZERO) {
                const int nl = c_in0 < 0 ? -c_in0 : 0;
                const int cr1 = min(c_need1 - c_in0, SW);
                const int cr0 = max(min(p.W - c_in0, cr1), nl);
                const int nt = r_in0 < 0 ? min(-r_in0, ROWS) : 0;
                const int rb1 = min(r_need1 - r_in0, ROWS);
                const int rb0 = max(min(p.H - r_in0, rb1), nt);
                const int wb = nl + (cr1 - cr0);
                if ((wb > 0) || (nt > 0) || (rb1 > rb0)) {
                    const float* xp = xb + (int64_t)plane_src(q) * p.x_ps;
                    const int n_in = rb0 - nt;
                    for (int idx = tid; idx < n_in * wb; idx += NT) {
                        const int rr = nt + idx / wb, qq = idx % wb;
                        const int cc = qq < nl ? qq : cr0 + (qq - nl);
                        const int sc = ext_index32(c_in0 + cc, p.W, p.mode);
                        tile[rr * SW + cc] = __ldg(xp + (int64_t)(r_in0 + rr) * p.x_rs + sc);
                    }
                    const int n_oob = nt + (rb1 - rb0);
                    if (n_oob > 0 && cr1 > 0) {
                        for (int idx = tid; idx < n_oob * cr1; idx += NT) {
                            const int qq = idx / cr1, cc = idx % cr1;
                            const int rr = qq < nt ? qq : rb0 + (qq - nt);
                            const int sr = ext_index32(r_in0 + rr, p.H, p.mode);
                            const int sc = ext_index32(c_in0 + cc, p.W, p.mode);
                            tile[rr * SW + cc] = __ldg(xp + (int64_t)sr * p.x_rs + sc);
                        }
                    }
                    __syncthreads();
                }
            }
        } else {
            const int qs = plane_src(q);
            const bool pz = qs < 0 || qs >= p.D;
            for (int idx = tid; idx < ROWS * SW; idx += NT) {
                const int rr = idx / SW, cc = idx - rr * SW;
                const int sr = ext_index32(r_in0 + rr, p.H, p.mode), sc = ext_index32(c_in0 + cc, p.W, p.mode);
                tile[idx] = (!pz && sr >= 0 && sc >= 0) ? __ldg(xb + (int64_t)qs * p.x_ps + (int64_t)sr * p.x_rs + sc) : 0.f;
            }
            __syncthreads();
        }

        // ---- row pass (along W) into buffer t & 1 -------------------------------------------------
        for (int item = tid; item < ROWS * NG8; item += NT) {
            const int row = item % ROWS, grp = item / ROWS;
            const float* src = tile + row * SW + 16 * grp;
            float v[4 * NV4];
#pragma unroll
            for (int qd = 0; qd < NV4; ++qd) {
                const float4 f = *reinterpret_cast<const float4*>(src + 4 * qd);
                v[4 * qd] = f.x; v[4 * qd + 1] = f.y; v[4 * qd + 2] = f.z; v[4 * qd + 3] = f.w;
            }
            float lo[8], hi[8];
            row_filter<L, OFF>(v, p.pl, p.ph, lo, hi);
            float* dlo = s_lo + row * MP + 8 * grp;
            float* dhi = s_hi + row * MP + 8 * grp;
            *reinterpret_cast<float4*>(dlo) = make_float4(lo[0], lo[1], lo[2], lo[3]);
            *reinterpret_cast<float4*>(dlo + 4) = make_float4(lo[4], lo[5], lo[6], lo[7]);
            *reinterpret_cast<float4*>(dhi) = make_float4(hi[0], hi[1], hi[2], hi[3]);
            *reinterpret_cast<float4*>(dhi + 4) = make_float4(hi[4], hi[5], hi[6], hi[7]);
        }
        // the only barrier of the plane: row results visible; the previous plane's column pass read the
        // OTHER buffer, and the stage that the next TMA overwrites was consumed before the previous barrier
        __syncthreads();

        // ---- column pass (along H) -> window slot t & 7 ---------------------------------------------
        {
            const float* src = (cp_half ? s_hi : s_lo) + (2 * cp_row) * MP + 4 * cp_cg;
            float2 aL[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
            float2 aH[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
#pragma unroll
            for (int j = 0; j < L; ++j) {
                const float4 f = *reinterpret_cast<const float4*>(src + j * MP);
                const float2 w0 = make_float2(f.x, f.y), w1 = make_float2(f.z, f.w);
                aL[0] = ffma2(p.bl[j], w0, aL[0]); aL[1] = ffma2(p.bl[j], w1, aL[1]);
                aH[0] = ffma2(p.bh[j], w0, aH[0]); aH[1] = ffma2(p.bh[j], w1, aH[1]);
            }
            switch (t & (WN - 1)) {                                  // uniform branch: fixed register slots
#define WTB_SLOT(K) case K: win[K][0] = aL[0]; win[K][1] = aL[1]; win[K][2] = aH[0]; win[K][3] = aH[1]; break;
                WTB_SLOT(0) WTB_SLOT(1) WTB_SLOT(2) WTB_SLOT(3) WTB_SLOT(4) WTB_SLOT(5) WTB_SLOT(6) WTB_SLOT(7)
#undef WTB_SLOT
            }
        }

        // ---- depth pass from registers: after plane t = HALO + 1 + 2 m the window t-L+1 .. t is complete ---
        if (t >= HALO + 1 && ((t - HALO) & 1)) {
            const int z = z0 + (t - HALO - 1) / 2;
            const int base = (t - L + 1) & (WN - 1);                  // slot of tap 0
            float2 accL[4], accH[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { accL[i] = make_float2(0.f, 0.f); accH[i] = make_float2(0.f, 0.f); }
#pragma unroll
            for (int k = 0; k < WN; ++k) {
                const int j = (k - base) & (WN - 1);                  // tap index of slot k (taps >= L are zero)
                const float2 cl = p.dl[j], ch = p.dh[j];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    accL[i] = ffma2(cl, win[k][i], accL[i]);
                    accH[i] = ffma2(ch, win[k][i], accH[i]);
                }
            }
            if (live) {
                // sub-band k = 4 hD + 2 hH + hW: this thread holds hW = cp_half, hH = 0 (i = 0, 1) and 1 (i = 2, 3)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int sb = 2 * hh + cp_half;
                    float* oL = p.out[sb] + (int64_t)b * p.out_bs[sb] + (int64_t)z * p.out_ps[sb] + (int64_t)gy * p.out_rs[sb] + gx;
                    float* oH = p.out[4 + sb] + (int64_t)b * p.out_bs[4 + sb] + (int64_t)z * p.out_ps[4 + sb] + (int64_t)gy * p.out_rs[4 + sb] + gx;
                    const float2 l0 = accL[2 * hh], l1 = accL[2 * hh + 1], h0 = accH[2 * hh], h1 = accH[2 * hh + 1];
                    if (p.vec_store) {
                        *reinterpret_cast<float4*>(oL) = make_float4(l0.x, l0.y, l1.x, l1.y);
                        *reinterpret_cast<float4*>(oH) = make_float4(h0.x, h0.y, h1.x, h1.y);
                    } else {
                        const float l4[4] = {l0.x, l0.y, l1.x, l1.y};
                        const float h4[4] = {h0.x, h0.y, h1.x, h1.y};
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            if (gx + e < p.Mw) { oL[e] = l4[e]; oH[e] = h4[e]; }
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static bool make_tmap_4d(CUtensorMap* map, const float* base, int64_t B, int64_t D, int64_t H, int64_t W, int64_t bs,
                         int64_t ps, int64_t rs, int box_w, int box_h) {
    PFN_encodeTiled enc = get_encode_tiled();
    if (!enc) return false;
    if (((uintptr_t)base & 15) || ((rs * 4) & 15) || ((ps * 4) & 15) || ((bs * 4) & 15)) return false;
    if (box_w > 256 || box_h > 256) return false;
    cuuint64_t dims[4] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)D, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)(rs * 4), (cuuint64_t)(ps * 4), (cuuint64_t)(bs * 4)};
    if (B == 1) strides[2] = (cuuint64_t)D * strides[1];
    cuuint32_t box[4] = {(cuuint32_t)box_w, (cuuint32_t)box_h, 1, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Grid of a 3-D tile-kernel launch: ntx x (nty * nseg) x B CTAs, segments of seg planes (analysis) or plane pairs
// (synthesis).
struct TileGrid3d {
    int ntx, nty, nseg, seg;
    bool fits(int64_t B) const { return (int64_t)nty * nseg <= 65535 && B <= 65535; }
};

// Output tiles (rows x columns) of fwd3d_tile_kernel.
static const int FWD3D_TILES[3][2] = {{16, 32}, {11, 44}, {8, 64}};

// Tile of an analysis level with Mh x Mw output planes: 16 x 32 unless another shape stages at least 25 % fewer input
// elements per plane (narrow or short planes); FWD3D_TILE forces one.
static int fwd3d_tile_shape(int64_t Mh, int64_t Mw, int L) {
    int best = 0;
    int64_t cost[3];
    for (int c = 0; c < 3; ++c) {
        const int th_ = FWD3D_TILES[c][0], tw_ = FWD3D_TILES[c][1];
        cost[c] = ((Mh + th_ - 1) / th_) * ((Mw + tw_ - 1) / tw_) * (2 * th_ + L - 2) * (2 * tw_ + L - 2);
    }
    for (int c = 1; c < 3; ++c)
        if (4 * cost[c] <= 3 * cost[0] && cost[c] < cost[best]) best = c;
    if (knob_is_set(K_FWD3D_TILE)) {
        const int forced = (int)knob_val(K_FWD3D_TILE, -1);
        if (forced >= 0 && forced < 3) best = forced;
    }
    return best;
}

// Analysis level of Md x Mh x Mw outputs per volume: segments along depth only while the grid would not fill the
// machine a few times.
static TileGrid3d fwd3d_grid(int64_t Md, int64_t Mh, int64_t Mw, int64_t B, int TH, int TW) {
    const int64_t ntx = (Mw + TW - 1) / TW, nty = (Mh + TH - 1) / TH;
    int64_t nseg = 1;
    while (nseg * ntx * nty * B < 4 * 296 && (Md + nseg - 1) / nseg > 24) ++nseg;
    const int64_t seg = (Md + nseg - 1) / nseg;
    return {(int)ntx, (int)nty, (int)((Md + seg - 1) / seg), (int)seg};
}

template <int L, int TH, int TW>
static cudaError_t launch_fwd3d_tiles(Fwd3dParams& p, const float* x, int64_t B, int D, int H, int W, int64_t x_bs, int64_t x_ps,
                                      int64_t x_rs, cudaStream_t st, uint64_t* launches) {
    using Gm = Fwd3dGeom<L, TH, TW>;
    const TileGrid3d g = fwd3d_grid(p.Md, p.Mh, p.Mw, B, TH, TW);
    assert(g.fits(B) && "dwt_route sends levels whose tiles overflow the grid to the general path");
    p.seg_planes = g.seg;
    p.nty = g.nty;
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof(tmap));
    const bool tma = make_tmap_4d(&tmap, x, B, D, H, W, x_bs, x_ps, x_rs, Gm::SW, Gm::ROWS);
    auto kern = tma ? fwd3d_tile_kernel<L, TH, TW, true> : fwd3d_tile_kernel<L, TH, TW, false>;
    cudaError_t e = ensure_dyn_smem(kern, (size_t)Gm::SMEM);
    if (e != cudaSuccess) return e;
    dim3 grid(g.ntx, g.nty * g.nseg, (unsigned)B);
    kern<<<grid, Gm::NT, Gm::SMEM, st>>>(p, tmap);
    ++*launches;
    return cudaGetLastError();
}

template <int L>
static cudaError_t launch_fwd3d_level(const float* x, int64_t B, int D, int H, int W, int64_t x_bs, int64_t x_ps, int64_t x_rs,
                                      const wt_level& d, int mode, const double* dlo, const double* dhi, cudaStream_t st,
                                      uint64_t* launches) {
    Fwd3dParams p;
    p.x = x; p.x_bs = x_bs; p.x_ps = x_ps; p.x_rs = x_rs;
    p.D = D; p.H = H; p.W = W;
    p.Md = (int)d.dims[0]; p.Mh = (int)d.dims[1]; p.Mw = (int)d.dims[2];
    p.out[0] = (float*)d.approx; p.out_bs[0] = d.approx_batch_stride; p.out_ps[0] = d.approx_strides[0]; p.out_rs[0] = d.approx_strides[1];
    for (int k = 1; k < 8; ++k) {
        p.out[k] = (float*)d.details + (int64_t)(k - 1) * d.band_stride;
        p.out_bs[k] = d.details_batch_stride; p.out_ps[k] = d.strides[0]; p.out_rs[k] = d.strides[1];
    }
    p.mode = mode;
    p.vec_store = 1;
    for (int k = 0; k < 8; ++k)
        if (((uintptr_t)p.out[k] & 15) || (p.out_bs[k] & 3) || (p.out_ps[k] & 3) || (p.out_rs[k] & 3) ||
            p.out_rs[k] < (p.Mw + 3) / 4 * 4)
            p.vec_store = 0;
    float tl[16], th[16];
    for (int k = 0; k < L; ++k) { tl[k] = (float)dlo[k]; th[k] = (float)dhi[k]; }
    for (int m = 0; m < L / 2; ++m) {
        p.pl[m] = make_float2(tl[L - 1 - 2 * m], tl[L - 2 - 2 * m]);
        p.ph[m] = make_float2(th[L - 1 - 2 * m], th[L - 2 - 2 * m]);
    }
    for (int j = 0; j < L; ++j) {
        p.bl[j] = make_float2(tl[L - 1 - j], tl[L - 1 - j]);
        p.bh[j] = make_float2(th[L - 1 - j], th[L - 1 - j]);
    }
    for (int j = 0; j < 8; ++j) {
        p.dl[j] = j < L ? p.bl[j] : make_float2(0.f, 0.f);
        p.dh[j] = j < L ? p.bh[j] : make_float2(0.f, 0.f);
    }
    switch (fwd3d_tile_shape(p.Mh, p.Mw, L)) {
        case 1: return launch_fwd3d_tiles<L, 11, 44>(p, x, B, D, H, W, x_bs, x_ps, x_rs, st, launches);
        case 2: return launch_fwd3d_tiles<L, 8, 64>(p, x, B, D, H, W, x_bs, x_ps, x_rs, st, launches);
        default: return launch_fwd3d_tiles<L, 16, 32>(p, x, B, D, H, W, x_bs, x_ps, x_rs, st, launches);
    }
}

// All levels of a float32 3-D analysis on the tile kernel (dwt_route chose it).
static int fused3d_fwd(int mode, int levels, int L, const double* dlo, const double* dhi, const float* x, int64_t batch,
                       const int64_t* dims, const int64_t* xs, int64_t xbs, const wt_level* lv, cudaStream_t st) {
    const float* src = x;
    int64_t sbs = xbs, sps = xs[0], srs = xs[1];
    int D = (int)dims[0], H = (int)dims[1], W = (int)dims[2];
    uint64_t launches = 0;
    for (int l = 0; l < levels; ++l) {
        cudaError_t e;
        switch (L) {
            case 2: e = launch_fwd3d_level<2>(src, batch, D, H, W, sbs, sps, srs, lv[l], mode, dlo, dhi, st, &launches); break;
            case 4: e = launch_fwd3d_level<4>(src, batch, D, H, W, sbs, sps, srs, lv[l], mode, dlo, dhi, st, &launches); break;
            case 6: e = launch_fwd3d_level<6>(src, batch, D, H, W, sbs, sps, srs, lv[l], mode, dlo, dhi, st, &launches); break;
            case 8: e = launch_fwd3d_level<8>(src, batch, D, H, W, sbs, sps, srs, lv[l], mode, dlo, dhi, st, &launches); break;
            default: return 0;
        }
        g_launches.fetch_add(launches, std::memory_order_relaxed);
        launches = 0;
        if (e != cudaSuccess) return cuda_fail(e, "fwd3d_tile_kernel");
        src = (const float*)lv[l].approx; sbs = lv[l].approx_batch_stride; sps = lv[l].approx_strides[0]; srs = lv[l].approx_strides[1];
        D = (int)lv[l].dims[0]; H = (int)lv[l].dims[1]; W = (int)lv[l].dims[2];
    }
    return 0;
}

}  // namespace wtb
