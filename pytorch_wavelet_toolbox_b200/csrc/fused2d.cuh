// fused2d.cuh -- 2-D analysis level as ONE kernel: rolling column strips on sm_90a.
//
// Replaces, per level, the reference's  F.pad -> conv2d(4 x [L x L], stride 2) -> split
// (src/ptwt/conv_transform_2.py:142-149) by a separable polyphase filter bank that reads the
// level input once and writes the four sub-bands once:
//
//   * a CTA owns a strip of TW output columns and a segment of output rows of one image and
//     marches down the strip in chunks of CH output rows (2 CH input rows);
//   * input chunks [2 CH x SW] are staged in shared memory by TMA (cp.async.bulk.tensor, 3-D
//     tensor map over [batch, H, W], out-of-bounds = zero fill) into an NSTAGE ring, completion
//     on mbarriers, so the next chunks are in flight while the current one is filtered;
//     border CTAs patch the out-of-range halo with the boundary extension (ext_index32);
//   * row pass: lane <-> input row, warp <-> group of 8 output columns; each thread slides the
//     L-tap window over 2*8+L-2 register-resident samples (LDS.128, conflict-free pitch) and
//     writes lo/hi rows into a ring of row-filtered lines;
//   * column pass: lane <-> output column; each thread slides down 4 output rows of the ring and
//     emits ll, lh, hl, hh -- coalesced 128-byte rows to HBM.  The vertical halo never leaves
//     shared memory (rolling ring), the horizontal halo costs (L-2)/(2 TW) extra L2 reads.
//
// Algorithmic bytes per level: 4 B * (H*W read + 4*Mh*Mw written).
#pragma once

#include <cassert>
#include <cuda.h>

#include "common.cuh"

namespace wtb {

// ------------------------------------------------------------------------------------------
// PTX helpers (mbarrier + TMA)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// ------------------------------------------------------------------------------------------
// paired-FP32 filter helpers: taps and samples travel as float2 pairs (even / odd polyphase halves).
// sm_90a has no packed FP32 FMA, so a pair is two round-to-nearest FMAs.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 ffma2(const float2 a, const float2 b, const float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// Row filter of one thread: NG consecutive (lo, hi) outputs from the register window v[].
// out[g] = sum_k dec[L-1-k] v[2g+k+OFF], evaluated as an even-tap and an odd-tap partial sum in the
// two halves of one paired accumulator.
template <int L, int OFF, int NV, int NG>
__device__ __forceinline__ void row_filter(const float (&v)[NV], const float2* __restrict__ pl,
                                           const float2* __restrict__ ph, float (&lo)[NG], float (&hi)[NG]) {
#pragma unroll
    for (int g = 0; g < NG; ++g) {
        float2 a = make_float2(0.f, 0.f), h = make_float2(0.f, 0.f);
#pragma unroll
        for (int m = 0; m < L / 2; ++m) {
            const float2 x = make_float2(v[2 * g + 2 * m + OFF], v[2 * g + 2 * m + OFF + 1]);
            a = ffma2(pl[m], x, a);
            h = ffma2(ph[m], x, h);
        }
        lo[g] = a.x + a.y;
        hi[g] = h.x + h.y;
    }
}

// Column filter of one thread: 2 output rows x 4 columns from L+2 consecutive ring rows (no wrap:
// the ring carries mirror rows), vertical low-pass into accL, high-pass into accH.
template <int L>
__device__ __forceinline__ void col_filter2x4(const float* __restrict__ rows, int pitch, const float2* __restrict__ bl,
                                              const float2* __restrict__ bh, float2 (&accL)[2][2], float2 (&accH)[2][2]) {
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int e = 0; e < 2; ++e) { accL[r][e] = make_float2(0.f, 0.f); accH[r][e] = make_float2(0.f, 0.f); }
#pragma unroll
    for (int j = 0; j < L + 2; ++j) {
        const float4 f = *reinterpret_cast<const float4*>(rows + j * pitch);
        const float2 w0 = make_float2(f.x, f.y), w1 = make_float2(f.z, f.w);
        if (j < L) {
            accL[0][0] = ffma2(bl[j], w0, accL[0][0]); accL[0][1] = ffma2(bl[j], w1, accL[0][1]);
            accH[0][0] = ffma2(bh[j], w0, accH[0][0]); accH[0][1] = ffma2(bh[j], w1, accH[0][1]);
        }
        if (j >= 2) {
            accL[1][0] = ffma2(bl[j - 2], w0, accL[1][0]); accL[1][1] = ffma2(bl[j - 2], w1, accL[1][1]);
            accH[1][0] = ffma2(bh[j - 2], w0, accH[1][0]); accH[1][1] = ffma2(bh[j - 2], w1, accH[1][1]);
        }
    }
}


// ------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------
template <typename T>
struct Fwd2dParams {
    const T* x;              // level input [batch, H, W]
    int64_t x_bs, x_rs;      // element strides (batch, row); column stride 1
    T* out[4];               // k = 0 (approx), 1, 2, 3 (sub-band index of include/wtb200.h)
    int64_t out_bs[4], out_rs[4];
    int H, W, Mh, Mw;
    int seg_rows;            // output rows per segment
    int mode;
    int batch0;              // batch offset of this launch (gridDim.z chunking)
    int vec_store;           // 1: every output row start is 16-byte aligned -> 128-bit stores
    Taps<T> taps;            // un-flipped dec_lo / dec_hi
    // float32 fast kernel: taps packed in pairs (see row_filter / col_filter2x4)
    float2 pl[8], ph[8], bl[16], bh[16];
};

template <int L, int TW, int ES = 4>
struct Fwd2dGeom {
    static constexpr int HALO = L - 2;
    // TMA needs the box to start on a 16-byte boundary: the staged tile begins HAL >= HALO columns
    // left of the first output's window, HAL * ES a multiple of 16.
    static constexpr int HAL = ((HALO * ES + 15) / 16) * 16 / ES;
    static constexpr int OFF = HAL - HALO;        // columns skipped at the left of the tile
    static constexpr int CH = 16;                 // output rows per chunk
    static constexpr int IN_ROWS = 2 * CH;        // input rows per chunk (= 32 = one row per lane)
    static constexpr int NEED = 2 * TW + HAL;     // input columns staged per strip
    static constexpr int SW = ((NEED - 4 + 7) / 8) * 8 + 4;  // smem pitch: >= NEED, == 4 (mod 8)
    static constexpr int MP = TW + 4;             // pitch of the row-filtered ring (== 4 mod 8 for TW % 8 == 0)
    static constexpr int RING = IN_ROWS + HALO;   // ring rows: one chunk plus the vertical halo
    static constexpr int NSTAGE = 2;              // input stages: one being filtered, one in flight
    static constexpr int G = 8;                   // output columns per thread in the row pass
    static constexpr int NWARP = TW / G;
    static constexpr int NTHREADS = 32 * NWARP;
    static constexpr int NV = 2 * G + HAL;        // samples a row-pass thread loads
    static constexpr int NV4 = (NV + 3) / 4;
    static constexpr int VEC = 16 / ES;           // output columns per thread in the column pass
    static constexpr int NCG = TW / VEC;          // column groups per output row
    static_assert(L % 2 == 0 && L >= 2 && L <= 18, "fused path: even filter length <= 18");
    static_assert(TW % 8 == 0, "TW must be a multiple of 8");
    static_assert(16 * (NWARP - 1) + 4 * NV4 <= SW, "row pass would read past the staged tile");
    static constexpr size_t stage_bytes(size_t es) { return (size_t)IN_ROWS * SW * es; }
    static constexpr size_t smem_bytes(size_t es) {
        return NSTAGE * stage_bytes(es) + 2 * (size_t)RING * MP * es + 64;
    }
};

template <typename T> struct VecOf;
template <> struct VecOf<float> { using type = float4; };
template <> struct VecOf<double> { using type = double2; };

template <typename T, int L, int TW, bool USE_TMA>
__global__ void __launch_bounds__((Fwd2dGeom<L, TW, sizeof(T)>::NTHREADS), (sizeof(T) == 4 ? 4 : 2))
fwd2d_strip_kernel(const __grid_constant__ Fwd2dParams<T> p, const __grid_constant__ CUtensorMap tmap) {
    using Gm = Fwd2dGeom<L, TW, sizeof(T)>;
    using V = typename VecOf<T>::type;
    constexpr int OFF = Gm::OFF, HAL = Gm::HAL;
    constexpr int HALO = Gm::HALO, CH = Gm::CH, IN_ROWS = Gm::IN_ROWS, SW = Gm::SW, MP = Gm::MP;
    constexpr int RING = Gm::RING, NSTAGE = Gm::NSTAGE, G = Gm::G, NT = Gm::NTHREADS, NV4 = Gm::NV4;
    constexpr int VEC = Gm::VEC, NCG = Gm::NCG;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    T* s_in = reinterpret_cast<T*>(smem_raw);                                   // [NSTAGE][IN_ROWS][SW]
    T* s_lo = reinterpret_cast<T*>(smem_raw + NSTAGE * Gm::stage_bytes(sizeof(T)));  // [RING][MP]
    T* s_hi = s_lo + RING * MP;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_hi + RING * MP);             // [NSTAGE]

    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int b = p.batch0 + blockIdx.z;
    const int x0 = blockIdx.x * TW;                 // first output column of the strip
    const int y0 = blockIdx.y * p.seg_rows;         // first output row of the segment
    const int y1 = min(y0 + p.seg_rows, p.Mh);
    if (y0 >= p.Mh) return;
    const int yb = y0 - HALO / 2;                   // chunk c covers output rows [yb + CH c, yb + CH (c+1))
    const int c_in0 = 2 * x0 - HAL;                 // first input column staged (16-byte aligned)
    const int r_in0 = 2 * yb;                       // first input row of chunk 0
    const int nchunks = (y1 - yb + CH - 1) / CH;
    const int c_need1 = 2 * min(x0 + TW, p.Mw);      // one past the last input column any output reads
    const int r_need1 = 2 * y1;                      // one past the last input row any output reads

    if (USE_TMA) {
        if (tid == 0) {
            tma_prefetch_desc(&tmap);
            for (int s = 0; s < NSTAGE; ++s) mbar_init(&bars[s], 1);
            fence_mbar_init();
        }
        __syncthreads();
        if (tid == 0) {
            // both stages are filled up front; a stage is refilled once its chunk has been row-filtered
            for (int s = 0; s < NSTAGE && s < nchunks; ++s) {
                mbar_expect_tx(&bars[s], (uint32_t)Gm::stage_bytes(sizeof(T)));
                tma_load_3d(s_in + (size_t)s * IN_ROWS * SW, &tmap, &bars[s], c_in0, r_in0 + s * IN_ROWS, b);
            }
        }
    }

    const T* __restrict__ xb = p.x + (int64_t)b * p.x_bs;

    // column-pass work decomposition (fixed per thread when NT == 2 * (CH/2) * NCG)
    constexpr int CP_ITEMS = 2 * (CH / 2) * NCG;    // (array half) x (row pair) x (column group)

    int ring_base = 0;                              // ring row that holds tile row 0 of the current chunk
    for (int c = 0; c < nchunks; ++c) {
        const int stage = c % NSTAGE;
        T* tile = s_in + (size_t)stage * IN_ROWS * SW;
        const int r_base = r_in0 + c * IN_ROWS;     // absolute input row of tile row 0

        if (USE_TMA) {
            mbar_wait(&bars[stage], (uint32_t)((c / NSTAGE) & 1));
            // border CTAs: replace the zero-filled out-of-range halo by the boundary extension.
            // Only the samples some output of this strip / segment really reads are patched:
            // tile columns [0, nl) and [cr0, cr1) of the in-range rows, and tile columns [0, cr1)
            // of the out-of-range rows [0, nt) and [rb0, rb1).
            if (p.mode != WT_MODE_ZERO) {
                const int nl = c_in0 < 0 ? -c_in0 : 0;
                const int cr1 = c_need1 - c_in0;                    // one past the last needed tile column
                const int cr0 = max(min(p.W - c_in0, cr1), nl);
                const int nt = r_base < 0 ? min(-r_base, IN_ROWS) : 0;
                const int rb1 = min(r_need1 - r_base, IN_ROWS);     // one past the last needed tile row
                const int rb0 = max(min(p.H - r_base, rb1), nt);
                const int wb = nl + (cr1 - cr0);
                const bool patch = (wb > 0) || (nt > 0) || (rb1 > rb0);
                if (patch) {
                    const int n_in = rb0 - nt;                      // in-range tile rows [nt, rb0)
                    for (int idx = tid; idx < n_in * wb; idx += NT) {
                        const int rr = nt + idx / wb, q = idx % wb;
                        const int cc = q < nl ? q : cr0 + (q - nl);
                        const int sc = ext_index32(c_in0 + cc, p.W, p.mode);
                        tile[rr * SW + cc] = __ldg(xb + (int64_t)(r_base + rr) * p.x_rs + sc);
                    }
                    const int n_oob = nt + (rb1 - rb0);
                    if (n_oob > 0 && cr1 > 0) {
                        for (int idx = tid; idx < n_oob * cr1; idx += NT) {
                            const int q = idx / cr1, cc = idx % cr1;
                            const int rr = q < nt ? q : rb0 + (q - nt);
                            const int sr = ext_index32(r_base + rr, p.H, p.mode);
                            const int sc = ext_index32(c_in0 + cc, p.W, p.mode);
                            tile[rr * SW + cc] = __ldg(xb + (int64_t)sr * p.x_rs + sc);
                        }
                    }
                    __syncthreads();
                }
            }
        } else {
            // plain cooperative loader (any alignment): coalesced along columns
            for (int idx = tid; idx < IN_ROWS * SW; idx += NT) {
                const int rr = idx / SW, cc = idx - rr * SW;
                const int sr = ext_index32(r_base + rr, p.H, p.mode), sc = ext_index32(c_in0 + cc, p.W, p.mode);
                tile[idx] = (sr >= 0 && sc >= 0) ? __ldg(xb + (int64_t)sr * p.x_rs + sc) : T(0);
            }
            __syncthreads();
        }

        // ---------------- row pass: lane <-> tile row, warp <-> 8 output columns -----------------
        {
            const T* src = tile + lane * SW + 2 * G * warp;
            T v[4 * NV4];
#pragma unroll
            for (int q = 0; q < NV4; ++q) {
                if (sizeof(T) == 4) {
                    const float4 t = *reinterpret_cast<const float4*>(src + 4 * q);
                    v[4 * q + 0] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
                } else {
                    const double2 t0 = *reinterpret_cast<const double2*>(src + 4 * q);
                    const double2 t1 = *reinterpret_cast<const double2*>(src + 4 * q + 2);
                    v[4 * q + 0] = t0.x; v[4 * q + 1] = t0.y; v[4 * q + 2] = t1.x; v[4 * q + 3] = t1.y;
                }
            }
            T lo[G], hi[G];
#pragma unroll
            for (int g = 0; g < G; ++g) {
                T a = T(0), h = T(0);
#pragma unroll
                for (int k = 0; k < L; ++k) {
                    a = fma(p.taps.lo[L - 1 - k], v[2 * g + k + OFF], a);
                    h = fma(p.taps.hi[L - 1 - k], v[2 * g + k + OFF], h);
                }
                lo[g] = a; hi[g] = h;
            }
            int slot = ring_base + lane;              // ring row of this tile row
            if (slot >= RING) slot -= RING;
            T* dlo = s_lo + slot * MP + G * warp;
            T* dhi = s_hi + slot * MP + G * warp;
            if (sizeof(T) == 4) {
                *reinterpret_cast<float4*>(dlo) = make_float4(lo[0], lo[1], lo[2], lo[3]);
                *reinterpret_cast<float4*>(dlo + 4) = make_float4(lo[4], lo[5], lo[6], lo[7]);
                *reinterpret_cast<float4*>(dhi) = make_float4(hi[0], hi[1], hi[2], hi[3]);
                *reinterpret_cast<float4*>(dhi + 4) = make_float4(hi[4], hi[5], hi[6], hi[7]);
            } else {
#pragma unroll
                for (int g = 0; g < G; g += 2) {
                    *reinterpret_cast<double2*>(dlo + g) = make_double2(lo[g], lo[g + 1]);
                    *reinterpret_cast<double2*>(dhi + g) = make_double2(hi[g], hi[g + 1]);
                }
            }
        }
        __syncthreads();   // ring rows of this chunk visible; the input stage is free again

        if (USE_TMA && tid == 0 && c + NSTAGE < nchunks) {
            fence_proxy_async();   // generic-proxy accesses to this stage precede the async refill
            mbar_expect_tx(&bars[stage], (uint32_t)Gm::stage_bytes(sizeof(T)));
            tma_load_3d(tile, &tmap, &bars[stage], c_in0, r_in0 + (c + NSTAGE) * IN_ROWS, b);
        }

        // ------- column pass: thread <-> (lo|hi array, 2 output rows, VEC output columns) --------
        // the lo array yields bands k = 0 (lo_H) and k = 2 (hi_H); the hi array k = 1 and k = 3
        {
            const int gy_chunk = yb + c * CH;
            for (int item = tid; item < CP_ITEMS; item += NT) {
                const int half = item / (CP_ITEMS / 2);
                const int rem = item - half * (CP_ITEMS / 2);
                const int rp = rem / NCG, cg = rem - rp * NCG;
                const int yl = 2 * rp;
                const T* ring = (half ? s_hi : s_lo) + VEC * cg;
                int row0 = ring_base + 2 * yl - HALO;               // ring row of the first tap
                if (row0 < 0) row0 += RING;
                T accL[2][VEC], accH[2][VEC];
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int e = 0; e < VEC; ++e) { accL[r][e] = T(0); accH[r][e] = T(0); }
#pragma unroll
                for (int j = 0; j < L + 2; ++j) {
                    int rj = row0 + j;
                    if (rj >= RING) rj -= RING;
                    const V t = *reinterpret_cast<const V*>(ring + rj * MP);
                    T w[VEC];
                    if (sizeof(T) == 4) {
                        const float4 f = *reinterpret_cast<const float4*>(&t);
                        w[0] = f.x; w[1] = f.y; w[VEC > 2 ? 2 : 0] = f.z; w[VEC > 2 ? 3 : 1] = f.w;
                    } else {
                        const double2 f = *reinterpret_cast<const double2*>(&t);
                        w[0] = f.x; w[1] = f.y;
                    }
                    if (j < L) {
#pragma unroll
                        for (int e = 0; e < VEC; ++e) {
                            accL[0][e] = fma(p.taps.lo[L - 1 - j], w[e], accL[0][e]);
                            accH[0][e] = fma(p.taps.hi[L - 1 - j], w[e], accH[0][e]);
                        }
                    }
                    if (j >= 2) {
#pragma unroll
                        for (int e = 0; e < VEC; ++e) {
                            accL[1][e] = fma(p.taps.lo[L + 1 - j], w[e], accL[1][e]);
                            accH[1][e] = fma(p.taps.hi[L + 1 - j], w[e], accH[1][e]);
                        }
                    }
                }
                const int gx = x0 + VEC * cg;
                if (gx >= p.Mw) continue;
                T* oL = p.out[half] + (int64_t)b * p.out_bs[half] + gx;          // vertical low-pass
                T* oH = p.out[2 + half] + (int64_t)b * p.out_bs[2 + half] + gx;  // vertical high-pass
                const int64_t rsL = p.out_rs[half], rsH = p.out_rs[2 + half];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int gy = gy_chunk + yl + r;
                    if (gy < y0 || gy >= y1) continue;
                    T* dl = oL + (int64_t)gy * rsL;
                    T* dh = oH + (int64_t)gy * rsH;
                    if (p.vec_store) {
                        if (sizeof(T) == 4) {
                            *reinterpret_cast<float4*>(dl) = make_float4(accL[r][0], accL[r][1], accL[r][VEC > 2 ? 2 : 0], accL[r][VEC > 2 ? 3 : 1]);
                            *reinterpret_cast<float4*>(dh) = make_float4(accH[r][0], accH[r][1], accH[r][VEC > 2 ? 2 : 0], accH[r][VEC > 2 ? 3 : 1]);
                        } else {
                            *reinterpret_cast<double2*>(dl) = make_double2(accL[r][0], accL[r][1]);
                            *reinterpret_cast<double2*>(dh) = make_double2(accH[r][0], accH[r][1]);
                        }
                    } else {
#pragma unroll
                        for (int e = 0; e < VEC; ++e)
                            if (gx + e < p.Mw) { dl[e] = accL[r][e]; dh[e] = accH[r][e]; }
                    }
                }
            }
        }
        __syncthreads();   // ring rows may be overwritten by the next chunk's row pass
        ring_base += IN_ROWS;
        if (ring_base >= RING) ring_base -= RING;
    }
}

// ------------------------------------------------------------------------------------------
// float32 fast variant: same structure as fwd2d_strip_kernel, with paired FP32 taps (ffma2), mirror
// rows behind the ring (column-pass windows never wrap, so their loads use immediate offsets) and
// all per-thread index arithmetic hoisted out of the chunk loop.
// ------------------------------------------------------------------------------------------
template <int L, int TW>
struct Fwd2dGeomF {
    using Base = Fwd2dGeom<L, TW, 4>;
    static constexpr int MIR = L + 2;
    static constexpr size_t SMEM = 2 * Base::stage_bytes(4) + 2 * (size_t)(Base::RING + MIR) * Base::MP * 4 + 64;
};

// Border CTAs of the TMA path: replace the zero-filled out-of-range halo of a staged float32 chunk by the
// boundary extension.  Only the samples some needed output reads are patched: tile columns [0, nl) and
// [cr0, cr1) of the in-range rows, and tile columns [0, cr1) of the out-of-range rows [0, nt) and [rb0, rb1).
// Ends with a barrier when it wrote anything.
template <int SW, int IN_ROWS, int NT>
__device__ __forceinline__ void patch_tile_f32(float* tile, const float* __restrict__ xb, int64_t x_rs, int H, int W,
                                               int mode, int c_in0, int r_base, int c_need1, int r_need1, int tid) {
    const int nl = c_in0 < 0 ? -c_in0 : 0;
    const int cr1 = min(c_need1 - c_in0, SW);
    const int cr0 = max(min(W - c_in0, cr1), nl);
    const int nt = r_base < 0 ? min(-r_base, IN_ROWS) : 0;
    const int rb1 = min(r_need1 - r_base, IN_ROWS);
    const int rb0 = max(min(H - r_base, rb1), nt);
    const int wb = nl + (cr1 - cr0);
    const bool patch = (wb > 0) || (nt > 0) || (rb1 > rb0);
    if (!patch) return;
    const int n_in = rb0 - nt;
    for (int idx = tid; idx < n_in * wb; idx += NT) {
        const int rr = nt + idx / wb, q = idx % wb;
        const int cc = q < nl ? q : cr0 + (q - nl);
        const int sc = ext_index32(c_in0 + cc, W, mode);
        tile[rr * SW + cc] = __ldg(xb + (int64_t)(r_base + rr) * x_rs + sc);
    }
    const int n_oob = nt + (rb1 - rb0);
    if (n_oob > 0 && cr1 > 0) {
        for (int idx = tid; idx < n_oob * cr1; idx += NT) {
            const int q = idx / cr1, cc = idx % cr1;
            const int rr = q < nt ? q : rb0 + (q - nt);
            const int sr = ext_index32(r_base + rr, H, mode);
            const int sc = ext_index32(c_in0 + cc, W, mode);
            tile[rr * SW + cc] = __ldg(xb + (int64_t)sr * x_rs + sc);
        }
    }
    __syncthreads();
}

// Row pass of the float32 strip kernels: lane <-> tile row, warp <-> 8 output columns; writes the lo / hi lines
// of the chunk into the ring (and into the mirror rows behind it).
template <int L, int TW>
__device__ __forceinline__ void strip_row_pass_f32(const float* tile, float* s_lo, float* s_hi, int ring_base,
                                                   const float2* __restrict__ pl, const float2* __restrict__ ph,
                                                   int lane, int warp) {
    using Gm = Fwd2dGeom<L, TW, 4>;
    constexpr int SW = Gm::SW, MP = Gm::MP, RING = Gm::RING, NV4 = Gm::NV4, MIR = L + 2;
    const float* src = tile + lane * SW + 16 * warp;
    float v[4 * NV4];
#pragma unroll
    for (int q = 0; q < NV4; ++q) {
        const float4 t = *reinterpret_cast<const float4*>(src + 4 * q);
        v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
    }
    float lo[8], hi[8];
    row_filter<L, Gm::OFF>(v, pl, ph, lo, hi);
    int slot = ring_base + lane;
    if (slot >= RING) slot -= RING;
    float* dlo = s_lo + slot * MP + 8 * warp;
    float* dhi = s_hi + slot * MP + 8 * warp;
    const float4 l0 = make_float4(lo[0], lo[1], lo[2], lo[3]), l1 = make_float4(lo[4], lo[5], lo[6], lo[7]);
    const float4 h0 = make_float4(hi[0], hi[1], hi[2], hi[3]), h1 = make_float4(hi[4], hi[5], hi[6], hi[7]);
    *reinterpret_cast<float4*>(dlo) = l0; *reinterpret_cast<float4*>(dlo + 4) = l1;
    *reinterpret_cast<float4*>(dhi) = h0; *reinterpret_cast<float4*>(dhi + 4) = h1;
    if (slot < MIR) {
        *reinterpret_cast<float4*>(dlo + RING * MP) = l0; *reinterpret_cast<float4*>(dlo + RING * MP + 4) = l1;
        *reinterpret_cast<float4*>(dhi + RING * MP) = h0; *reinterpret_cast<float4*>(dhi + RING * MP + 4) = h1;
    }
}

template <int L, int TW, bool USE_TMA>
__global__ void __launch_bounds__((Fwd2dGeom<L, TW, 4>::NTHREADS), 3)
fwd2d_strip_f32_kernel(const __grid_constant__ Fwd2dParams<float> p, const __grid_constant__ CUtensorMap tmap) {
    using Gm = Fwd2dGeom<L, TW, 4>;
    constexpr int HAL = Gm::HAL, HALO = Gm::HALO, CH = Gm::CH, IN_ROWS = Gm::IN_ROWS, SW = Gm::SW;
    constexpr int MP = Gm::MP, RING = Gm::RING, NT = Gm::NTHREADS, MIR = Fwd2dGeomF<L, TW>::MIR;
    constexpr int NCG = TW / 4;
    static_assert(NT == 2 * (CH / 2) * NCG, "one column-pass item per thread");

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_in = reinterpret_cast<float*>(smem_raw);                          // [2][IN_ROWS][SW]
    float* s_lo = s_in + 2 * IN_ROWS * SW;                                     // [RING + MIR][MP]
    float* s_hi = s_lo + (RING + MIR) * MP;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_hi + (RING + MIR) * MP);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = p.batch0 + blockIdx.z;
    const int x0 = blockIdx.x * TW;
    const int y0 = blockIdx.y * p.seg_rows;
    if (y0 >= p.Mh) return;
    const int y1 = min(y0 + p.seg_rows, p.Mh);
    const int yb = y0 - HALO / 2;
    const int c_in0 = 2 * x0 - HAL;
    const int r_in0 = 2 * yb;
    const int nchunks = (y1 - yb + CH - 1) / CH;
    const int c_need1 = 2 * min(x0 + TW, p.Mw);
    const int r_need1 = 2 * y1;

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
                mbar_expect_tx(&bars[s], (uint32_t)Gm::stage_bytes(4));
                tma_load_3d(s_in + s * IN_ROWS * SW, &tmap, &bars[s], c_in0, r_in0 + s * IN_ROWS, b);
            }
        }
    }
    const float* __restrict__ xb = p.x + (int64_t)b * p.x_bs;

    // per-thread constants of the column pass: (lo|hi array, row pair, 4-column group)
    const int half = tid / (NT / 2);
    const int rem = tid - half * (NT / 2);
    const int rp = rem / NCG, cg = rem - rp * NCG;
    const int yl = 2 * rp;
    const float* cring = (half ? s_hi : s_lo) + 4 * cg;
    const int gx = x0 + 4 * cg;
    const bool col_ok = gx < p.Mw;
    // bands: the lo array yields k = 0 (vertical low) and k = 2 (vertical high); the hi array k = 1, 3
    float* pL = p.out[half] + (int64_t)b * p.out_bs[half] + (int64_t)(yb + yl) * p.out_rs[half] + gx;
    float* pH = p.out[2 + half] + (int64_t)b * p.out_bs[2 + half] + (int64_t)(yb + yl) * p.out_rs[2 + half] + gx;
    const int64_t rsL = p.out_rs[half], rsH = p.out_rs[2 + half];

    int ring_base = 0;
    for (int c = 0; c < nchunks; ++c) {
        const int stage = c & 1;
        float* tile = s_in + stage * IN_ROWS * SW;
        const int r_base = r_in0 + c * IN_ROWS;

        if (USE_TMA) {
            mbar_wait(&bars[stage], (uint32_t)((c >> 1) & 1));
            if (p.mode != WT_MODE_ZERO)
                patch_tile_f32<SW, IN_ROWS, NT>(tile, xb, p.x_rs, p.H, p.W, p.mode, c_in0, r_base, c_need1, r_need1, tid);
        } else {
            for (int idx = tid; idx < IN_ROWS * SW; idx += NT) {
                const int rr = idx / SW, cc = idx - rr * SW;
                const int sr = ext_index32(r_base + rr, p.H, p.mode), sc = ext_index32(c_in0 + cc, p.W, p.mode);
                tile[idx] = (sr >= 0 && sc >= 0) ? __ldg(xb + (int64_t)sr * p.x_rs + sc) : 0.f;
            }
            __syncthreads();
        }

        strip_row_pass_f32<L, TW>(tile, s_lo, s_hi, ring_base, p.pl, p.ph, lane, warp);
        __syncthreads();

        if (USE_TMA && tid == 0 && c + 2 < nchunks) {
            fence_proxy_async();
            mbar_expect_tx(&bars[stage], (uint32_t)Gm::stage_bytes(4));
            tma_load_3d(tile, &tmap, &bars[stage], c_in0, r_in0 + (c + 2) * IN_ROWS, b);
        }

        // ---- column pass --------------------------------------------------------------------------
        {
            int row0 = ring_base + 2 * yl - HALO;
            if (row0 < 0) row0 += RING;
            else if (row0 >= RING) row0 -= RING;
            float2 accL[2][2], accH[2][2];
            col_filter2x4<L>(cring + row0 * MP, MP, p.bl, p.bh, accL, accH);
            if (col_ok) {
                const int gyc = yb + c * CH + yl;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int gy = gyc + r;
                    if (gy < y0 || gy >= y1) continue;
                    float* dl = pL + (int64_t)(c * CH + r) * rsL;
                    float* dh = pH + (int64_t)(c * CH + r) * rsH;
                    if (p.vec_store) {
                        *reinterpret_cast<float4*>(dl) = make_float4(accL[r][0].x, accL[r][0].y, accL[r][1].x, accL[r][1].y);
                        *reinterpret_cast<float4*>(dh) = make_float4(accH[r][0].x, accH[r][0].y, accH[r][1].x, accH[r][1].y);
                    } else {
                        const float aL[4] = {accL[r][0].x, accL[r][0].y, accL[r][1].x, accL[r][1].y};
                        const float aH[4] = {accH[r][0].x, accH[r][0].y, accH[r][1].x, accH[r][1].y};
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            if (gx + e < p.Mw) { dl[e] = aL[e]; dh[e] = aH[e]; }
                    }
                }
            }
        }
        __syncthreads();
        ring_base += IN_ROWS;
        if (ring_base >= RING) ring_base -= RING;
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_tiled() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)ptr;
    });
    return fn;
}

template <typename T>
static bool make_tmap_3d(CUtensorMap* map, const T* base, int64_t B, int64_t H, int64_t W, int64_t bs, int64_t rs,
                         int box_w, int box_h) {
    PFN_encodeTiled enc = get_encode_tiled();
    if (!enc) return false;
    if (((uintptr_t)base & 15) || ((rs * sizeof(T)) & 15) || ((bs * sizeof(T)) & 15)) return false;
    if (box_w > 256 || box_h > 256 || ((box_w * sizeof(T)) & 15)) return false;
    cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)(rs * sizeof(T)), (cuuint64_t)(bs * sizeof(T))};
    cuuint32_t box[3] = {(cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    if (B == 1) strides[1] = (cuuint64_t)H * strides[0];  // any valid value
    CUresult r = enc(map, sizeof(T) == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3,
                     (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// Output columns per strip of the strip kernel: 64 in float32, 32 in float64.
constexpr int fwd2d_strip_width(int es) { return es == 4 ? 64 : 32; }

// Grid of a strip-kernel launch: nstrip strips (gridDim.x) by nseg segments of seg output rows (gridDim.y); the batch
// rides on gridDim.z in launches of at most 65535 images.
struct StripGrid { int nstrip, nseg, seg; };

// Analysis level of Mh x Mw outputs per image, B images per launch.  Segments of 16 k - HALO/2 output rows keep the
// chunking free of an idle tail; small levels get shorter ones so that the grid still fills the machine a few times
// (fewer images never give fewer segments).
static StripGrid fwd2d_grid(int64_t Mh, int64_t Mw, int64_t B, int L, int TW) {
    const int HH = (L - 2) / 2;   // Fwd2dGeom::HALO / 2
    const int64_t nstrip = (Mw + TW - 1) / TW;
    int64_t nseg = (Mh + 255) / 256;
    while (nseg * nstrip * B < 4 * 592 && (Mh + nseg - 1) / nseg > 48) ++nseg;
    int64_t seg = ((Mh + nseg - 1) / nseg + HH + 15) / 16 * 16 - HH;
    if (seg < 16 - HH) seg = 16 - HH;
    return {(int)nstrip, (int)((Mh + seg - 1) / seg), (int)seg};
}

template <typename T, int L, int TW>
static cudaError_t launch_fwd2d_level(const T* x, int64_t B, int H, int W, int64_t x_bs, int64_t x_rs, T* const out[4],
                                      const int64_t out_bs[4], const int64_t out_rs[4], int Mh, int Mw, int mode,
                                      const Taps<T>& taps, cudaStream_t st, uint64_t* launches) {
    using Gm = Fwd2dGeom<L, TW, sizeof(T)>;
    Fwd2dParams<T> p;
    p.x = x; p.x_bs = x_bs; p.x_rs = x_rs;
    for (int k = 0; k < 4; ++k) { p.out[k] = out[k]; p.out_bs[k] = out_bs[k]; p.out_rs[k] = out_rs[k]; }
    p.H = H; p.W = W; p.Mh = Mh; p.Mw = Mw; p.mode = mode; p.taps = taps;
    // 128-bit stores need every band row to start on a 16-byte boundary and the row pitch to
    // cover the rounded-up width (the packed layout of the Python side guarantees both)
    constexpr int VEC = 16 / (int)sizeof(T);
    p.vec_store = 1;
    for (int k = 0; k < 4; ++k) {
        if (((uintptr_t)out[k] & 15) || (out_bs[k] % VEC) || (out_rs[k] % VEC) || out_rs[k] < (Mw + VEC - 1) / VEC * VEC)
            p.vec_store = 0;
    }
    const StripGrid g = fwd2d_grid(Mh, Mw, B, L, TW);
    assert(g.nseg <= 65535 && "dwt_route sends levels whose segments overflow gridDim.y to the general path");
    p.seg_rows = g.seg;
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof(tmap));
    const bool tma = make_tmap_3d<T>(&tmap, x, B, H, W, x_bs, x_rs, Gm::SW, Gm::IN_ROWS);
    size_t smem = Gm::smem_bytes(sizeof(T));
    auto kern = tma ? fwd2d_strip_kernel<T, L, TW, true> : fwd2d_strip_kernel<T, L, TW, false>;
    if constexpr (sizeof(T) == 4 && TW == 64) {
        if (!knob_on(K_NO_FFMA2)) {
            for (int m = 0; m < L / 2; ++m) {
                p.pl[m] = make_float2(taps.lo[L - 1 - 2 * m], taps.lo[L - 2 - 2 * m]);
                p.ph[m] = make_float2(taps.hi[L - 1 - 2 * m], taps.hi[L - 2 - 2 * m]);
            }
            for (int j = 0; j < L; ++j) {
                p.bl[j] = make_float2(taps.lo[L - 1 - j], taps.lo[L - 1 - j]);
                p.bh[j] = make_float2(taps.hi[L - 1 - j], taps.hi[L - 1 - j]);
            }
            kern = tma ? fwd2d_strip_f32_kernel<L, TW, true> : fwd2d_strip_f32_kernel<L, TW, false>;
            smem = Fwd2dGeomF<L, TW>::SMEM;
        }
    }
    cudaError_t e = ensure_dyn_smem(kern, smem);
    if (e != cudaSuccess) return e;
    for (int64_t b0 = 0; b0 < B; b0 += 65535) {
        p.batch0 = (int)b0;
        const int nb = (int)((B - b0) < 65535 ? (B - b0) : 65535);
        dim3 grid(g.nstrip, g.nseg, nb);
        kern<<<grid, Gm::NTHREADS, smem, st>>>(p, tmap);
        ++*launches;
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

template <typename T>
static bool try_wpair(const T*, int64_t, int, int, int64_t, int64_t, const wt_level&, const wt_level&, int, int,
                      const Taps<T>&, cudaStream_t, uint64_t*, cudaError_t*);
template <typename T>
static bool try_fuse2(const T*, int64_t, int, int, int64_t, int64_t, const wt_level&, const wt_level&, int, int,
                      const Taps<T>&, cudaStream_t, uint64_t*, cudaError_t*);

// One auxiliary stream per device: the batch is cut into chunks that alternate between the caller's
// stream and this one, so that the small, latency-bound launches of the deep levels of one chunk run
// under the bandwidth-bound level-1 launch of the next (fork / join with events; no host sync).
struct AuxStream {
    cudaStream_t s = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr;   // created once per device, reused by every call
    std::mutex mu;                                // orders the record / wait pairs of concurrent callers
};
static AuxStream* aux_stream_for_current_device() {
    static std::mutex mu;
    static AuxStream aux[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    std::lock_guard<std::mutex> g(mu);
    AuxStream& a = aux[dev];
    if (!a.s) {
        if (cudaStreamCreateWithFlags(&a.s, cudaStreamNonBlocking) != cudaSuccess) { a.s = nullptr; return nullptr; }
        if (cudaEventCreateWithFlags(&a.fork, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&a.join, cudaEventDisableTiming) != cudaSuccess) {
            cudaStreamDestroy(a.s);
            a.s = nullptr;
            return nullptr;
        }
    }
    return &a;
}

template <typename T>
static int fused2d_fwd_run(int mode, int levels, int L, const double* dlo, const double* dhi, const T* x, int64_t batch,
                           const int64_t* dims, const int64_t* xs, int64_t xbs, const wt_level* lv, cudaStream_t st);

// All levels of a 2-D analysis on the strip and level-pair kernels (dwt_route chose them).
template <typename T>
static int fused2d_fwd(int mode, int levels, int L, const double* dlo, const double* dhi, const T* x, int64_t batch,
                       const int64_t* dims, const int64_t* xs, int64_t xbs, const wt_level* lv, cudaStream_t st) {
    // Chunking: the batch is cut into chunks that alternate between the caller's stream and one auxiliary
    // stream, so that the latency-bound deep levels of one chunk run under the bandwidth-bound level-1 launch
    // of the next.  The intermediate approximations cA_1 .. cA_{n-1} are scratch, so every chunk reuses the
    // scratch slots of its stream.  (Small chunks could keep those slots L2-resident, but with one launch per
    // level and chunk the launch tails grow with the chunk count.)
    int64_t chunk = 0;   // images per chunk
    int nstreams = 2;
    if (knob_is_set(K_CHUNK)) chunk = knob_val(K_CHUNK, 0);
    else if (levels >= 2 && batch >= 16 && (int64_t)batch * dims[0] * dims[1] >= (int64_t(1) << 27)) chunk = (batch + 1) / 2;
    if (knob_is_set(K_STREAMS)) nstreams = knob_val(K_STREAMS, 2) >= 2 ? 2 : 1;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (nstreams > 1 && (cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone)) nstreams = 1;
    if (knob_on(K_NO_AUX_STREAM)) nstreams = 1;
    AuxStream* aux = nstreams > 1 ? aux_stream_for_current_device() : nullptr;
    cudaStream_t s2 = aux ? aux->s : nullptr;
    if (!s2) nstreams = 1;
    if (chunk <= 0 || chunk >= batch || levels > 32)
        return fused2d_fwd_run<T>(mode, levels, L, dlo, dhi, x, batch, dims, xs, xbs, lv, st);
    if (nstreams > 1) {
        std::lock_guard<std::mutex> g(aux->mu);
        cudaEventRecord(aux->fork, st);
        cudaStreamWaitEvent(s2, aux->fork, 0);
    }
    int rc = 0;
    wt_level sub[32];
    int c = 0;
    for (int64_t b0 = 0; b0 < batch && rc == 0; b0 += chunk, ++c) {
        const int64_t b1 = b0 + chunk < batch ? b0 + chunk : batch;
        const int which = nstreams > 1 ? (c & 1) : 0;
        const int64_t slot0 = (int64_t)which * chunk;       // scratch slots of this stream (stream order protects reuse)
        for (int l = 0; l < levels; ++l) {
            sub[l] = lv[l];
            sub[l].details = (T*)lv[l].details + b0 * lv[l].details_batch_stride;
            // the last level's approximation is an output; the others are scratch (include/wtb200.h)
            sub[l].approx = (T*)lv[l].approx + (l == levels - 1 ? b0 : slot0) * lv[l].approx_batch_stride;
        }
        rc = fused2d_fwd_run<T>(mode, levels, L, dlo, dhi, x + b0 * xbs, b1 - b0, dims, xs, xbs, sub, which ? s2 : st);
    }
    if (nstreams > 1) {
        std::lock_guard<std::mutex> g(aux->mu);
        cudaEventRecord(aux->join, s2);
        cudaStreamWaitEvent(st, aux->join, 0);
    }
    return rc;
}

template <typename T>
static int fused2d_fwd_run(int mode, int levels, int L, const double* dlo, const double* dhi, const T* x, int64_t batch,
                           const int64_t* dims, const int64_t* xs, int64_t xbs, const wt_level* lv, cudaStream_t st) {
    Taps<T> taps;
    for (int k = 0; k < L; ++k) { taps.lo[k] = (T)dlo[k]; taps.hi[k] = (T)dhi[k]; }
    const T* src = x;
    int64_t sbs = xbs, srs = xs[0];
    int64_t H = dims[0], W = dims[1];
    uint64_t launches = 0;
    for (int l = 0; l < levels; ++l) {
        const wt_level& d = lv[l];
        if (l + 1 < levels) {
            // two levels in one launch, cA_{l+1} stays in shared memory: the kernel of independent warps
            // (fused2d_wpair.cuh) for levels 1-2 of images of >= WPAIR_MIN samples, at least 8 of them, else the
            // opt-in two-level strip kernel (fused2d_fuse2.cuh)
            cudaError_t pe = cudaSuccess;
            const char* pair = nullptr;
            const int64_t wmin = knob_val(K_WPAIR_MIN, int64_t(1) << 24);
            if (H * W >= wmin && batch * H * W >= 8 * wmin && (l == 0 || knob_on(K_WPAIR_DEEP)) &&
                try_wpair<T>(src, batch, (int)H, (int)W, sbs, srs, lv[l], lv[l + 1], L, mode, taps, st, &launches, &pe))
                pair = "fwd2d_wpair_kernel";
            else if (try_fuse2<T>(src, batch, (int)H, (int)W, sbs, srs, lv[l], lv[l + 1], L, mode, taps, st, &launches, &pe))
                pair = "fwd2d_fuse2_f32_kernel";
            if (pair) {
                g_launches.fetch_add(launches, std::memory_order_relaxed);
                launches = 0;
                if (pe != cudaSuccess) return cuda_fail(pe, pair);
                const wt_level& d2 = lv[l + 1];
                src = (const T*)d2.approx; sbs = d2.approx_batch_stride; srs = d2.approx_strides[0];
                H = d2.dims[0]; W = d2.dims[1];
                ++l;
                continue;
            }
        }
        T* out[4];
        int64_t obs[4], ors[4];
        out[0] = (T*)d.approx; obs[0] = d.approx_batch_stride; ors[0] = d.approx_strides[0];
        for (int k = 1; k < 4; ++k) {
            out[k] = (T*)d.details + (int64_t)(k - 1) * d.band_stride;
            obs[k] = d.details_batch_stride; ors[k] = d.strides[0];
        }
        const int Mh = (int)d.dims[0], Mw = (int)d.dims[1];
        cudaError_t e = cudaSuccess;
#define WTB_F2D_CASE(LL)                                                                                       \
    case LL:                                                                                                   \
        e = launch_fwd2d_level<T, LL, fwd2d_strip_width(sizeof(T))>(src, batch, (int)H, (int)W, sbs, srs, out, obs,  \
                                                                     ors, Mh, Mw, mode, taps, st, &launches);  \
        break;
        switch (L) {
            WTB_F2D_CASE(2)
            WTB_F2D_CASE(4)
            WTB_F2D_CASE(6)
            WTB_F2D_CASE(8)
            WTB_F2D_CASE(10)
            WTB_F2D_CASE(12)
            WTB_F2D_CASE(14)
            WTB_F2D_CASE(16)
            default: return 0;
        }
#undef WTB_F2D_CASE
        g_launches.fetch_add(launches, std::memory_order_relaxed);
        launches = 0;
        if (e != cudaSuccess) return cuda_fail(e, "fwd2d_strip_kernel");
        src = out[0]; sbs = obs[0]; srs = ors[0];
        H = Mh; W = Mw;
    }
    return 0;
}

}  // namespace wtb
