// fused2d_mega.cuh -- ALL levels of a float32 2-D analysis in ONE persistent kernel (EXPERIMENTAL, off by
// default: WTB200_MEGA=1).
//
// One launch per level makes every approximation band cA_l a round trip through HBM (+33 % traffic
// for db4 L4).  This kernel runs the per-level strip algorithm of fwd2d_strip_f32_kernel over a work
// queue that interleaves the levels image by image:
//
//     period p :  level-1 items of image p, level-2 items of image p-1, level-3 items of image p-2, ...
//
// The idea is that cA_1 of an image, consumed one period after it was produced, is still resident in L2
// (50 MB on an H100), optionally helped by L2 cache hints (evict_first for streaming loads / detail
// stores, evict_last for approximation stores) and by a ring of 2-4 reused scratch slots
// (WTB200_MEGA_RING).  With hundreds of resident CTAs the in-flight window is larger than L2, so the
// per-level launches stay the default.  The scheduling machinery (queue, completion counters,
// write-after-read protection of the slot ring, TMA reads of data produced by other SMs) is correct,
// tested in every boundary mode, and the starting point for whatever keeps cA on chip next.
//
//   * persistent CTAs (3 per SM) fetch item indices from a global atomic counter; an item of level l+1
//     waits (ld.acquire spin by one thread) until the per-(level, image) completion counter of level l
//     reaches the item count; producers publish with __threadfence + atomicAdd.  Items only ever wait
//     for items with smaller queue indices, which running CTAs hold, so the scheme cannot deadlock
//     regardless of how many CTAs are resident;
//   * approximation data written by other SMs with ordinary stores is read by TMA (async proxy):
//     the consumer issues fence.proxy.async after the acquire.
#pragma once

#include "fused2d.cuh"

namespace wtb {

constexpr int MEGA_MAXLEV = 8;

struct MegaLevel {
    const float* x;
    int64_t x_bs, x_rs;
    float* out[4];
    int64_t out_bs[4], out_rs[4];
    int H, W, Mh, Mw;
    int seg_rows, nstrip, nseg;
    int vec_store;
};

struct MegaParams {
    MegaLevel lv[MEGA_MAXLEV];
    int levels, batch, mode;
    int ring;                    // > 0: the intermediate approximations of image b live in scratch slot b % ring
    int items_per_period;        // sum over levels of nstrip * nseg
    int* counters;               // [0]: work queue; [1 + l * batch + b]: finished items of level l, image b
    float2 pl[8], ph[8], bl[16], bh[16];
};

struct MegaMaps {
    CUtensorMap m[MEGA_MAXLEV];
};

__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void tma_load_3d_hint(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                                 uint64_t pol) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(pol)
        : "memory");
}
__device__ __forceinline__ void st_v4_hint(float* p, float4 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w),
                 "l"(pol)
                 : "memory");
}
__device__ __forceinline__ int ld_acquire(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

template <int L, bool HINTS>
__global__ void __launch_bounds__(256, 3)
fwd2d_mega_kernel(const __grid_constant__ MegaParams p, const __grid_constant__ MegaMaps maps) {
    constexpr int TW = 64;
    using Gm = Fwd2dGeom<L, TW, 4, 2>;
    constexpr int OFF = Gm::OFF, HAL = Gm::HAL, HALO = Gm::HALO, CH = Gm::CH, IN_ROWS = Gm::IN_ROWS, SW = Gm::SW;
    constexpr int MP = Gm::MP, RING = Gm::RING, NT = Gm::NTHREADS, NV4 = Gm::NV4, MIR = Fwd2dGeomF<L, TW>::MIR;
    constexpr int NCG = TW / 4;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_in = reinterpret_cast<float*>(smem_raw);
    float* s_lo = s_in + 2 * IN_ROWS * SW;
    float* s_hi = s_lo + (RING + MIR) * MP;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_hi + (RING + MIR) * MP);
    __shared__ int s_item;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        for (int l = 0; l < p.levels; ++l) tma_prefetch_desc(&maps.m[l]);
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_mbar_init();
    }
    __syncthreads();
    const uint64_t pol_first = l2_policy_evict_first(), pol_last = l2_policy_evict_last();

    // per-thread constants of the column pass
    const int half = tid / (NT / 2);
    const int rem = tid - half * (NT / 2);
    const int rp = rem / NCG, cg = rem - rp * NCG;
    const int yl = 2 * rp;
    const float* cring = (half ? s_hi : s_lo) + 4 * cg;

    const int nperiods = p.batch + p.levels - 1;
    const int total = nperiods * p.items_per_period;
    uint32_t gchunk = 0;                           // chunks consumed by this CTA so far (mbarrier phase bookkeeping)

    for (;;) {
        if (tid == 0) s_item = atomicAdd(p.counters, 1);
        __syncthreads();
        const int item = s_item;
        __syncthreads();
        if (item >= total) break;
        // decode: period, level, (segment, strip).  Queue order inside a period: level 0 first.
        const int period = item / p.items_per_period;
        int r = item - period * p.items_per_period;
        int l = 0;
        for (; l < p.levels - 1; ++l) {
            const int nl = p.lv[l].nstrip * p.lv[l].nseg;
            if (r < nl) break;
            r -= nl;
        }
        const int b = period - l;                  // level l works on the image that entered l periods ago
        if (b < 0 || b >= p.batch) continue;
        const MegaLevel& d = p.lv[l];
        const int sy = r / d.nstrip, sx = r - sy * d.nstrip;

        // ---- wait for the producing level, and for the readers of the scratch slot this item overwrites ----
        const bool writes_scratch = (l + 1 < p.levels);
        const bool war = p.ring > 0 && writes_scratch && b >= p.ring;
        if (l > 0 || war) {
            if (tid == 0) {
                if (l > 0) {
                    const int need = p.lv[l - 1].nstrip * p.lv[l - 1].nseg;
                    const int* cnt = p.counters + 1 + (l - 1) * p.batch + b;
                    while (ld_acquire(cnt) < need) __nanosleep(200);
                }
                if (war) {
                    // slot b % ring still holds cA_{l+1} of image b - ring until all its level-(l+1) items are done;
                    // those items sit `ring - 1` periods earlier in the queue, so running CTAs hold them: no deadlock
                    const int need = p.lv[l + 1].nstrip * p.lv[l + 1].nseg;
                    const int* cnt = p.counters + 1 + (l + 1) * p.batch + (b - p.ring);
                    while (ld_acquire(cnt) < need) __nanosleep(200);
                }
                asm volatile("fence.proxy.async;" ::: "memory");   // generic-proxy writes -> async-proxy (TMA) reads
            }
            __syncthreads();
        }
        // batch index of the input / of the approximation output: scratch slots when the ring is on
        const int b_in = (p.ring > 0 && l > 0) ? b % p.ring : b;
        const int b_ap = (p.ring > 0 && writes_scratch) ? b % p.ring : b;

        // ---- one strip segment of level l (same algorithm as fwd2d_strip_f32_kernel) -----------------
        const int x0 = sx * TW;
        const int y0 = sy * d.seg_rows;
        if (y0 < d.Mh) {
            const int y1 = min(y0 + d.seg_rows, d.Mh);
            const int yb = y0 - HALO / 2;
            const int c_in0 = 2 * x0 - HAL;
            const int r_in0 = 2 * yb;
            const int nchunks = (y1 - yb + CH - 1) / CH;
            const int c_need1 = 2 * min(x0 + TW, d.Mw);
            const int r_need1 = 2 * y1;
            const CUtensorMap* tm = &maps.m[l];
            if (tid == 0) {
                for (int s = 0; s < 2 && s < nchunks; ++s) {
                    const uint32_t st = (gchunk + s) & 1;
                    mbar_expect_tx(&bars[st], (uint32_t)Gm::stage_bytes(4));
                    if (HINTS) tma_load_3d_hint(s_in + st * IN_ROWS * SW, tm, &bars[st], c_in0, r_in0 + s * IN_ROWS, b_in, pol_first);
                    else tma_load_3d(s_in + st * IN_ROWS * SW, tm, &bars[st], c_in0, r_in0 + s * IN_ROWS, b_in);
                }
            }
            const float* __restrict__ xb = d.x + (int64_t)b_in * d.x_bs;
            const int gx = x0 + 4 * cg;
            const bool col_ok = gx < d.Mw;
            float* pL = d.out[half] + (int64_t)(half == 0 ? b_ap : b) * d.out_bs[half] + (int64_t)(yb + yl) * d.out_rs[half] + gx;
            float* pH = d.out[2 + half] + (int64_t)b * d.out_bs[2 + half] + (int64_t)(yb + yl) * d.out_rs[2 + half] + gx;
            const int64_t rsL = d.out_rs[half], rsH = d.out_rs[2 + half];
            // k = 0 is the approximation (re-read by the next level unless this is the last one)
            const bool l_is_approx = (half == 0) && (l + 1 < p.levels);

            int ring_base = 0;
            for (int c = 0; c < nchunks; ++c, ++gchunk) {
                const int stage = gchunk & 1;
                float* tile = s_in + stage * IN_ROWS * SW;
                const int r_base = r_in0 + c * IN_ROWS;
                mbar_wait(&bars[stage], (gchunk >> 1) & 1);
                if (p.mode != WT_MODE_ZERO) {
                    const int nl = c_in0 < 0 ? -c_in0 : 0;
                    const int cr1 = min(c_need1 - c_in0, SW);
                    const int cr0 = max(min(d.W - c_in0, cr1), nl);
                    const int nt = r_base < 0 ? min(-r_base, IN_ROWS) : 0;
                    const int rb1 = min(r_need1 - r_base, IN_ROWS);
                    const int rb0 = max(min(d.H - r_base, rb1), nt);
                    const int wb = nl + (cr1 - cr0);
                    if ((wb > 0) || (nt > 0) || (rb1 > rb0)) {
                        const int n_in = rb0 - nt;
                        for (int idx = tid; idx < n_in * wb; idx += NT) {
                            const int rr = nt + idx / wb, q = idx % wb;
                            const int cc = q < nl ? q : cr0 + (q - nl);
                            const int sc = ext_index32(c_in0 + cc, d.W, p.mode);
                            tile[rr * SW + cc] = __ldcg(xb + (int64_t)(r_base + rr) * d.x_rs + sc);
                        }
                        const int n_oob = nt + (rb1 - rb0);
                        if (n_oob > 0 && cr1 > 0) {
                            for (int idx = tid; idx < n_oob * cr1; idx += NT) {
                                const int q = idx / cr1, cc = idx % cr1;
                                const int rr = q < nt ? q : rb0 + (q - nt);
                                const int sr = ext_index32(r_base + rr, d.H, p.mode);
                                const int sc = ext_index32(c_in0 + cc, d.W, p.mode);
                                tile[rr * SW + cc] = __ldcg(xb + (int64_t)sr * d.x_rs + sc);
                            }
                        }
                        __syncthreads();
                    }
                }
                // row pass
                {
                    const float* src = tile + lane * SW + 16 * warp;
                    float v[4 * NV4];
#pragma unroll
                    for (int q = 0; q < NV4; ++q) {
                        const float4 t = *reinterpret_cast<const float4*>(src + 4 * q);
                        v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
                    }
                    float lo[8], hi[8];
                    row_filter8<L, OFF>(v, p.pl, p.ph, lo, hi);
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
                __syncthreads();
                if (tid == 0 && c + 2 < nchunks) {
                    fence_proxy_async();
                    mbar_expect_tx(&bars[stage], (uint32_t)Gm::stage_bytes(4));
                    if (HINTS) tma_load_3d_hint(tile, tm, &bars[stage], c_in0, r_in0 + (c + 2) * IN_ROWS, b_in, pol_first);
                    else tma_load_3d(tile, tm, &bars[stage], c_in0, r_in0 + (c + 2) * IN_ROWS, b_in);
                }
                // column pass
                {
                    int row0 = ring_base + 2 * yl - HALO;
                    if (row0 < 0) row0 += RING;
                    else if (row0 >= RING) row0 -= RING;
                    float2 accL[2][2], accH[2][2];
                    col_filter2x4<L>(cring + row0 * MP, MP, p.bl, p.bh, accL, accH);
                    if (col_ok) {
                        const int gyc = yb + c * CH + yl;
#pragma unroll
                        for (int rr = 0; rr < 2; ++rr) {
                            const int gy = gyc + rr;
                            if (gy < y0 || gy >= y1) continue;
                            float* dl = pL + (int64_t)(c * CH + rr) * rsL;
                            float* dh = pH + (int64_t)(c * CH + rr) * rsH;
                            const float4 vl = make_float4(accL[rr][0].x, accL[rr][0].y, accL[rr][1].x, accL[rr][1].y);
                            const float4 vh = make_float4(accH[rr][0].x, accH[rr][0].y, accH[rr][1].x, accH[rr][1].y);
                            if (d.vec_store) {
                                if (HINTS) {
                                    st_v4_hint(dl, vl, l_is_approx ? pol_last : pol_first);
                                    st_v4_hint(dh, vh, pol_first);
                                } else {
                                    *reinterpret_cast<float4*>(dl) = vl;
                                    *reinterpret_cast<float4*>(dh) = vh;
                                }
                            } else {
                                const float aL[4] = {vl.x, vl.y, vl.z, vl.w}, aH[4] = {vh.x, vh.y, vh.z, vh.w};
#pragma unroll
                                for (int e = 0; e < 4; ++e)
                                    if (gx + e < d.Mw) { dl[e] = aL[e]; dh[e] = aH[e]; }
                            }
                        }
                    }
                }
                __syncthreads();
                ring_base += IN_ROWS;
                if (ring_base >= RING) ring_base -= RING;
            }
        }
        // ---- publish ---------------------------------------------------------------------------------
        if (writes_scratch || p.ring > 0) {     // consumers wait on it; with the ring also the next writer of the slot
            __syncthreads();
            if (tid == 0) {
                __threadfence();
                atomicAdd(p.counters + 1 + l * p.batch + b, 1);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static size_t mega_workspace_bytes(int levels, int64_t batch) {
    return (size_t)(1 + (int64_t)levels * batch) * sizeof(int);
}

static bool mega2d_enabled() {
    return knob_on(K_MEGA);
}

template <int L>
static int launch_fwd2d_mega(int mode, int levels, const double* dlo, const double* dhi, const float* x, int64_t batch,
                             const int64_t* dims, const int64_t* xs, int64_t xbs, const wt_level* lv, void* ws, size_t ws_bytes,
                             cudaStream_t st, int* done) {
    using Gm = Fwd2dGeom<L, 64, 4, 2>;
    *done = 0;
    if (levels < 2 || levels > MEGA_MAXLEV || batch < 2 || batch >= (1 << 20)) return 0;
    if (!ws || ws_bytes < mega_workspace_bytes(levels, batch)) return 0;
    MegaParams p;
    MegaMaps maps;
    memset(&p, 0, sizeof(p));
    memset(&maps, 0, sizeof(maps));
    p.levels = levels; p.batch = (int)batch; p.mode = mode;
    p.counters = (int*)ws;
    const float* src = x;
    int64_t sbs = xbs, srs = xs[0];
    int64_t H = dims[0], W = dims[1];
    int ipp = 0;
    for (int l = 0; l < levels; ++l) {
        const wt_level& d = lv[l];
        MegaLevel& m = p.lv[l];
        if (H >= (1 << 30) || W >= (1 << 30) || d.strides[1] != 1 || d.approx_strides[1] != 1) return 0;
        m.x = src; m.x_bs = sbs; m.x_rs = srs;
        m.H = (int)H; m.W = (int)W; m.Mh = (int)d.dims[0]; m.Mw = (int)d.dims[1];
        m.out[0] = (float*)d.approx; m.out_bs[0] = d.approx_batch_stride; m.out_rs[0] = d.approx_strides[0];
        for (int k = 1; k < 4; ++k) {
            m.out[k] = (float*)d.details + (int64_t)(k - 1) * d.band_stride;
            m.out_bs[k] = d.details_batch_stride; m.out_rs[k] = d.strides[0];
        }
        m.vec_store = 1;
        for (int k = 0; k < 4; ++k)
            if (((uintptr_t)m.out[k] & 15) || (m.out_bs[k] & 3) || (m.out_rs[k] & 3) || m.out_rs[k] < (m.Mw + 3) / 4 * 4) m.vec_store = 0;
        constexpr int HH = Gm::HALO / 2;
        int seg_target = 256;
        if (knob_is_set(K_MEGA_SEG)) { const int v = (int)knob_val(K_MEGA_SEG, 0); if (v >= 16 && v <= 4096) seg_target = v; }
        int nseg = (m.Mh + seg_target - 1) / seg_target;
        int seg = ((m.Mh + nseg - 1) / nseg + HH + 15) / 16 * 16 - HH;
        if (seg < 16 - HH) seg = 16 - HH;
        nseg = (m.Mh + seg - 1) / seg;
        m.seg_rows = seg; m.nseg = nseg; m.nstrip = (m.Mw + 63) / 64;
        ipp += m.nseg * m.nstrip;
        if (!make_tmap_3d<float>(&maps.m[l], src, batch, H, W, sbs, srs, Gm::SW, Gm::IN_ROWS)) return 0;
        src = m.out[0]; sbs = m.out_bs[0]; srs = m.out_rs[0];
        H = m.Mh; W = m.Mw;
    }
    p.items_per_period = ipp;
    p.ring = 0;
    if (knob_is_set(K_MEGA_RING)) { const int v = (int)knob_val(K_MEGA_RING, 0); if (v >= 2 && v <= batch) p.ring = v; }
    if ((int64_t)ipp * (batch + levels) >= (int64_t(1) << 31)) return 0;
    float tl[16], th[16];
    for (int k = 0; k < L; ++k) { tl[k] = (float)dlo[k]; th[k] = (float)dhi[k]; }
    for (int m2 = 0; m2 < L / 2; ++m2) {
        p.pl[m2] = make_float2(tl[L - 1 - 2 * m2], tl[L - 2 - 2 * m2]);
        p.ph[m2] = make_float2(th[L - 1 - 2 * m2], th[L - 2 - 2 * m2]);
    }
    for (int j = 0; j < L; ++j) {
        p.bl[j] = make_float2(tl[L - 1 - j], tl[L - 1 - j]);
        p.bh[j] = make_float2(th[L - 1 - j], th[L - 1 - j]);
    }
    cudaError_t e = cudaMemsetAsync(ws, 0, mega_workspace_bytes(levels, batch), st);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemsetAsync");
    const bool hints = !knob_on(K_MEGA_NOHINTS);
    auto kern = hints ? fwd2d_mega_kernel<L, true> : fwd2d_mega_kernel<L, false>;
    const size_t smem = Fwd2dGeomF<L, 64>::SMEM;
    e = ensure_dyn_smem(kern, smem);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute");
    const int sms = sm_count();
    int occ = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, smem);
    if (e != cudaSuccess || occ < 1) return 0;
    kern<<<sms * occ, 256, smem, st>>>(p, maps);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "fwd2d_mega_kernel");
    *done = 1;
    return 0;
}

}  // namespace wtb
