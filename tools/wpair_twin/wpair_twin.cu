// wpair_twin.cu -- traffic twin of fwd2d_wpair_kernel (levels 1-2 of the 2-D analysis in one launch).
//
// Same grid, segment table, one-warp CTAs, TMA boxes, stage ring and mbarriers as the real kernel (the host geometry
// is wpair_plan, the device geometry WPairGeom), and the same stores: three 128-bit level-1 detail stores per lane and
// approximation row, four 64-bit level-2 stores per lane and output row, at the same addresses.  It does no
// filtering: every stored value is a plain sum of staged samples.  Its rate is the best this access pattern reaches
// at the given occupancy, which tells the cost of the real kernel's arithmetic and latency apart from that of its
// traffic (tools/time_wpair_ceiling.py).  Boundary patching is left out: it touches a few edge strips only.
// It can keep its strips in step the way the kernel does (one-warp CTAs in a cluster, split cluster barrier) or as
// warps of one CTA (named barrier), and wpair_kernel_fwd launches the real kernel at the same cluster size and
// CTAs per SM, so the three can be timed side by side.
//
// Built as its own shared object (pytorch_wavelet_toolbox_b200/csrc/build.py), never into libwtb200.so.
#include <atomic>

#include "../../pytorch_wavelet_toolbox_b200/csrc/common.cuh"

namespace wtb {
// the launch counter and error hook that wtb200.cu defines for the strip-kernel launchers of fused2d.cuh
[[maybe_unused]] static std::atomic<uint64_t> g_launches{0};
[[maybe_unused]] static int cuda_fail(cudaError_t e, const char*) { return (int)e; }
}  // namespace wtb

#include "../../pytorch_wavelet_toolbox_b200/csrc/fused2d_wpair.cuh"

namespace wtb {

// HINT bit 0: output stores with the streaming (evict-first) cache operator; bit 1: input boxes loaded with an L2
// evict-first policy.
template <int HINT>
__device__ __forceinline__ void twin_st4(float* p, float4 v) {
    if (HINT & 1) __stcs(reinterpret_cast<float4*>(p), v); else *reinterpret_cast<float4*>(p) = v;
}
template <int HINT>
__device__ __forceinline__ void twin_st2(float* p, float2 v) {
    if (HINT & 1) __stcs(reinterpret_cast<float2*>(p), v); else *reinterpret_cast<float2*>(p) = v;
}
template <int HINT>
__device__ __forceinline__ void twin_load(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    if (HINT & 2) {
        uint64_t pol;
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
        asm volatile(
            "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
            " [%0], [%1, {%3, %4, %5}], [%2], %6;"
            ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(pol)
            : "memory");
    } else {
        tma_load_3d(dst, map, bar, c0, c1, c2);
    }
}

// WPC > 1: a CTA of WPC warps runs WPC adjacent strips (each warp with its own ring, as one CTA of the real kernel)
// and a named barrier after every group keeps them in lockstep.
// CSYNC (one-warp CTAs launched as clusters): 1 = the kernel's split cluster barrier (arrive after the refill, wait
// before the next group); 2 = the same barrier not split (wait right after the arrive).
template <int L, int NSTG, int HINT, int WPC = 1, int CSYNC = 0>
__global__ void __launch_bounds__(32 * WPC) wpair_twin_kernel(const __grid_constant__ WPairParams p,
                                                              const __grid_constant__ CUtensorMap tmap) {
    using Gm = WPairGeom<L, NSTG>;
    constexpr int HALO = Gm::HALO, NA = Gm::NA, HL1 = Gm::HL1, TW2 = Gm::TW2;
    constexpr int TILE_W = Gm::TILE_W, RP1 = Gm::RP1, R2P = Gm::R2P, RING = Gm::RING, ROWS = Gm::ROWS;
    constexpr int STG_F = Gm::STAGE_STRIDE / 4;

    extern __shared__ __align__(128) unsigned char smem_all[];
    const int warp = threadIdx.x >> 5;
    unsigned char* smem_raw = smem_all + warp * ((Gm::SMEM + 127) / 128 * 128);
    float* s_tile = reinterpret_cast<float*>(smem_raw);
    float* s_row = reinterpret_cast<float*>(smem_raw + NSTG * Gm::STAGE_STRIDE);
    float* s_ring = s_row + 2 * RP1;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_ring + RING * R2P);

    const int lane = threadIdx.x & 31;
    const int b = p.batch0 + blockIdx.y;

    // strip and segment exactly as fwd2d_wpair_kernel (a strip past the last one repeats the last one)
    const int X0n = min((int)blockIdx.x * WPC + warp, (p.Mw2 + TW2 - 1) / TW2 - 1) * TW2;
    int X0 = X0n;
    {
        const int lim = (p.Mw1 - L + HL1) / 2;
        if (X0 > lim) X0 = max(lim & ~1, 0);
    }
    const int cA0 = 2 * X0 - HL1;
    const int c_in0 = 2 * cA0 - Gm::HAL;
    const int own1_lo = 2 * X0n, own1_hi = min(2 * (X0n + TW2), p.Mw1);
    const int own2_lo = X0n, own2_hi = min(X0n + TW2, p.Mw2);
    const int Y0 = p.seg_start[blockIdx.z], Y1 = p.seg_start[blockIdx.z + 1];
    int a_start = 2 * Y0 - HALO - ((NA - 1) & 1);
    {
        int amax = p.Mh1 - RING;
        if ((amax - (NA - 1)) & 1) --amax;
        a_start = max(min(a_start, amax), -((NA - 1) & 1));
    }
    const int a_end = min(p.Mh1, 2 * Y1);
    const int a_lo = max(a_start, 0);
    const int n1 = a_end - a_start + NA - 1;
    const int ngroups = (n1 + 1) / 2;
    const int r_in0 = 2 * a_start - HALO;

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
            twin_load<HINT>(s_tile + s * STG_F, &tmap, &bars[s], c_in0 / 2, r_in0 + s * ROWS, b);
        }
    }

    const int col1 = cA0 + 4 * lane;
    const bool store1 = col1 >= own1_lo && col1 < own1_hi;
    float* const pd1 = p.d1 + (int64_t)b * p.d1_bs + (int64_t)a_start * p.d1_rs + col1;
    const int col2 = X0 + 2 * lane;
    const bool store2 = col2 >= own2_lo && col2 < own2_hi;
    float* po2[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) po2[k] = p.o2[k] + (int64_t)b * p.o2_bs[k] + (int64_t)Y0 * p.o2_rs[k] + col2;

    int K2 = Y0, produced = a_lo, stage = 0;
    uint32_t par = 0;
    float* const row_lane = s_row + 4 * lane;
    float* const ring_lane = s_ring + 2 * lane;

    for (int g = 0; g < ngroups; ++g) {
        if (CSYNC == 1 && g > 0) cluster_wait();
        float* tile = s_tile + stage * STG_F;
        mbar_wait(&bars[stage], par);
        const int a0 = a_start + 2 * g - (NA - 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            // the lane's window of the two input rows of this step (same LDS.128 as the row pass)
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int q = 0; q < Gm::NV1_4; ++q) {
                    const float4 t = *reinterpret_cast<const float4*>(tile + (2 * h + r) * TILE_W + 8 * lane + 4 * q);
                    v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
                }
            const int a = a0 + h;
            if (a >= a_lo && a < a_end) {
                *reinterpret_cast<float4*>(row_lane + (a & 1) * RP1) = v;
                if (store1 && a >= 2 * Y0) {
                    float* pd = pd1 + (int64_t)(a - a_start) * p.d1_rs;
                    twin_st4<HINT>(pd, v);
                    twin_st4<HINT>(pd + p.d1_band, make_float4(v.y, v.z, v.w, v.x));
                    twin_st4<HINT>(pd + 2 * p.d1_band, make_float4(v.z, v.w, v.x, v.y));
                }
            }
        }
        __syncwarp();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int a = a0 + h;
            const float* rrow = row_lane + (a & 1) * RP1;
            float2 s = make_float2(0.f, 0.f);
#pragma unroll
            for (int q = 0; q < Gm::NV2_4; ++q) {
                const float4 t = *reinterpret_cast<const float4*>(rrow + 4 * q);
                s.x += t.x + t.z; s.y += t.y + t.w;
            }
            if (a >= a_lo && a < a_end) {
                float* dst = ring_lane + (a & (RING - 1)) * R2P;
                *reinterpret_cast<float2*>(dst) = s;
                *reinterpret_cast<float2*>(dst + 64) = make_float2(s.y, s.x);
            }
        }
        produced = min(max(a0 + 2, a_lo), a_end);
        __syncwarp();

        if (lane == 0 && g + NSTG < ngroups) {
            fence_proxy_async();
            mbar_expect_tx(&bars[stage], (uint32_t)Gm::STAGE_BYTES);
            twin_load<HINT>(tile, &tmap, &bars[stage], c_in0 / 2, r_in0 + (g + NSTG) * ROWS, b);
        }
        if (++stage == NSTG) { stage = 0; par ^= 1u; }
        if (WPC > 1) asm volatile("bar.sync 1, %0;" ::"r"(32 * WPC) : "memory");
        if (CSYNC) cluster_arrive();
        if (CSYNC == 2) cluster_wait();

        while (K2 < Y1) {
            const int vb = 2 * K2 - HALO;
            if (min(vb + L, p.Mh1) > produced) break;
            float2 lo = make_float2(0.f, 0.f), hi = make_float2(0.f, 0.f);
#pragma unroll
            for (int j = 0; j < L; ++j) {
                const float* rr = ring_lane + ((vb + j) & (RING - 1)) * R2P;
                const float2 l = *reinterpret_cast<const float2*>(rr), hh = *reinterpret_cast<const float2*>(rr + 64);
                lo.x += l.x; lo.y += l.y; hi.x += hh.x; hi.y += hh.y;
            }
            if (store2) {
                twin_st2<HINT>(po2[0], lo);
                twin_st2<HINT>(po2[1], hi);
                twin_st2<HINT>(po2[2], make_float2(lo.y, hi.x));
                twin_st2<HINT>(po2[3], make_float2(hi.y, lo.x));
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) po2[k] += p.o2_rs[k];
            ++K2;
        }
    }
    if (CSYNC == 1 && ngroups > 0) cluster_wait();   // pairs the last arrive
}

// Dynamic shared memory of `w` warps' worth of `smem` bytes each, padded so that at most ctas_per_sm warps fit on an
// SM when ctas_per_sm > 0 (228 KB of shared memory per SM, 1 KB of it reserved per CTA).
static size_t twin_smem(size_t smem, int ctas_per_sm, int w) {
    smem = (smem + 127) / 128 * 128 * w;
    if (ctas_per_sm > 0) {
        const size_t pad = (size_t)(228 * 1024 / (ctas_per_sm / w) - 1024);
        if (pad > smem) smem = pad;
    }
    return smem;
}

// Launches kern over (ceil(nstrip / w), batch, nseg) CTAs of w warps, as clusters of `cluster` CTAs along x.
template <typename K>
static int twin_launch(K kern, const WPairParams& p0, const CUtensorMap& tmap, int nstrip, int64_t B, size_t smem,
                       int w, int cluster, cudaStream_t st) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess && cluster > 8) e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return (int)e;
    const int gx = (nstrip + w - 1) / w;
    if (gx % cluster) return -1;
    WPairParams p = p0;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cluster; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    for (int64_t b0 = 0; b0 < B; b0 += 65535) {
        p.batch0 = (int)b0;
        const int nb = (int)((B - b0) < 65535 ? (B - b0) : 65535);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(gx, nb, p.nseg);
        cfg.blockDim = dim3(32 * w, 1, 1);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = st;
        cfg.attrs = &attr;
        cfg.numAttrs = 1;
        cudaLaunchKernelEx(&cfg, kern, p, tmap);
        e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

}  // namespace wtb

// Launches the twin of fwd2d_wpair_kernel<8, nstg, *> for levels 1-2 described by lv[0], lv[1] (the wt_level layout
// of wt_dwt_fwd).  ctas_per_sm > 0 pads the dynamic shared memory so that at most that many CTAs fit on an SM.
// hint and wpc select HINT and WPC of wpair_twin_kernel (ctas_per_sm then counts warps).  cluster > 1 launches
// one-warp CTAs as clusters of that many adjacent strips, kept in step by the kernel's split cluster barrier
// (csync = 1) or by the same barrier not split (csync = 2).  Returns 0, -1 when the real kernel would decline these
// shapes or the strip count is not a multiple of the cluster size, or the CUDA error code.
extern "C" int wpair_twin_fwd(int nstg, int ctas_per_sm, int hint, int wpc, int cluster, int csync, const float* x,
                              int64_t B, int H, int W, int64_t x_bs, int64_t x_rs, const wt_level* lv, int mode,
                              void* stream) {
    using namespace wtb;
    WPairParams p;
    CUtensorMap tmap;
    int nstrip = 0;
    Taps<float> taps;
    memset(&taps, 0, sizeof(taps));
    const cudaStream_t st = (cudaStream_t)stream;
    auto run = [&](auto kern, size_t smem, bool ok, int w) -> int {
        if (!ok) return -1;
        return twin_launch(kern, p, tmap, nstrip, B, twin_smem(smem, ctas_per_sm, w), w, w > 1 ? 1 : cluster, st);
    };
    if (nstg == 3)
        return run(wpair_twin_kernel<8, 3, 0>, (size_t)WPairGeom<8, 3>::SMEM,
                   wpair_plan<8, 3>(x, B, H, W, x_bs, x_rs, lv[0], lv[1], mode, taps, p, tmap, nstrip), 1);
    const bool ok = wpair_plan<8, 2>(x, B, H, W, x_bs, x_rs, lv[0], lv[1], mode, taps, p, tmap, nstrip);
    const size_t smem = (size_t)WPairGeom<8, 2>::SMEM;
    if (wpc == 2) return run(wpair_twin_kernel<8, 2, 0, 2>, smem, ok, 2);
    if (wpc == 3) return run(wpair_twin_kernel<8, 2, 0, 3>, smem, ok, 3);
    if (wpc == 6) return run(wpair_twin_kernel<8, 2, 0, 6>, smem, ok, 6);
    if (cluster > 1 && csync == 1) return run(wpair_twin_kernel<8, 2, 0, 1, 1>, smem, ok, 1);
    if (cluster > 1 && csync == 2) return run(wpair_twin_kernel<8, 2, 0, 1, 2>, smem, ok, 1);
    switch (hint) {
        case 1: return run(wpair_twin_kernel<8, 2, 1>, smem, ok, 1);
        case 2: return run(wpair_twin_kernel<8, 2, 2>, smem, ok, 1);
        case 3: return run(wpair_twin_kernel<8, 2, 3>, smem, ok, 1);
        default: return run(wpair_twin_kernel<8, 2, 0>, smem, ok, 1);
    }
}

// Launches the real fwd2d_wpair_kernel<8, *, *> on the same shapes (var as the library's WPAIR_VAR: 0 = <8, 2, 12>,
// the db4 default; 1 = <8, 2, 15>; 3 = <8, 3, 12>) with taps dlo / dhi, as clusters of `cluster` strips at at most
// ctas_per_sm CTAs per SM (0: as many as fit), so that it can be timed at the twin's settings.  Returns as
// wpair_twin_fwd.
extern "C" int wpair_kernel_fwd(int var, int ctas_per_sm, int cluster, const float* x, int64_t B, int H, int W,
                                int64_t x_bs, int64_t x_rs, const wt_level* lv, int mode, const double* dlo,
                                const double* dhi, void* stream) {
    using namespace wtb;
    WPairParams p;
    CUtensorMap tmap;
    int nstrip = 0;
    Taps<float> taps;
    for (int k = 0; k < 8; ++k) { taps.lo[k] = (float)dlo[k]; taps.hi[k] = (float)dhi[k]; }
    const cudaStream_t st = (cudaStream_t)stream;
    if (var == 3) {
        if (!wpair_plan<8, 3>(x, B, H, W, x_bs, x_rs, lv[0], lv[1], mode, taps, p, tmap, nstrip)) return -1;
        return twin_launch(fwd2d_wpair_kernel<8, 3, 12>, p, tmap, nstrip, B,
                           twin_smem((size_t)WPairGeom<8, 3>::SMEM, ctas_per_sm, 1), 1, cluster, st);
    }
    if (!wpair_plan<8, 2>(x, B, H, W, x_bs, x_rs, lv[0], lv[1], mode, taps, p, tmap, nstrip)) return -1;
    const size_t smem = twin_smem((size_t)WPairGeom<8, 2>::SMEM, ctas_per_sm, 1);
    if (var == 1) return twin_launch(fwd2d_wpair_kernel<8, 2, 15>, p, tmap, nstrip, B, smem, 1, cluster, st);
    return twin_launch(fwd2d_wpair_kernel<8, 2, 12>, p, tmap, nstrip, B, smem, 1, cluster, st);
}
