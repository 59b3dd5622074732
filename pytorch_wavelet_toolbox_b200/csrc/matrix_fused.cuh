// matrix_fused.cuh -- several analysis levels of the boundary-filter matrix FWT in ONE kernel (float32, and float64
// with NO_DMMA; the float64 default is matrix_dmma.cuh).
//
// The reference applies one sparse operator per level (torch.sparse.mm, src/ptwt/matmul_transform.py:
// 409-425), so every approximation vector makes a round trip through memory: 2x the compulsory traffic
// for a 12-level transform.  Here a CTA takes a chunk of the signal through up to MAXK levels in shared
// memory: only the detail coefficients and the last approximation leave the SM.
//
//   * a CTA owns TK outputs of the last fused level and, going backwards, the sample ranges of the
//     finer levels they depend on (halo L/2 - 1 left, L/2 right per level);
//   * samples are kept de-interleaved (even / odd polyphase arrays): output i reads samples
//     2i - (L/2-1) .. 2i + L/2, i.e. CONTIGUOUS runs of both arrays, so that two adjacent outputs per
//     thread need a handful of conflict-free 128-bit shared loads;
//   * the orthogonalised boundary rows (dense blocks) are evaluated by the CTAs at the two ends; the
//     round-off sized cross-corner entries the QR leaves behind are not reachable from a chunk, so the
//     host only selects this kernel when they are below 1e-13 (float64) -- otherwise the per-level
//     kernels, which keep them, run instead.
#pragma once

#include "common.cuh"

namespace wtb {

constexpr int MATF_MAXK = 8;

template <typename T>
struct MatFusedParams {
    const T* x;                  // [batch, n0]
    int64_t x_stride;
    T* hi[MATF_MAXK];            // detail of fused level j (0-based), [batch, n_j / 2]
    int64_t hi_stride[MATF_MAXK];
    T* lo;                       // approximation of the last fused level
    int64_t lo_stride;
    int k;                       // fused levels
    int n[MATF_MAXK + 1];        // n[0] = input length, n[j] = n[j-1] / 2
    int nb_top[MATF_MAXK], nb_bot[MATF_MAXK], w_left[MATF_MAXK], w_right[MATF_MAXK];
    const T* lo_left[MATF_MAXK];
    const T* lo_right[MATF_MAXK];
    const T* hi_left[MATF_MAXK];
    const T* hi_right[MATF_MAXK];
    int tk;                      // outputs of the last fused level per chunk
    int cpc;                     // consecutive chunks of one row a CTA streams through
    int cap0;                    // capacity (samples) of the level-0 staging arrays
    T flo[16], fhi[16];          // taps in window order: out[i] = sum_k f[k] a[2i - (L/2-1) + k]
    int vec;                     // matrix_dmma.cuh (polyphase kernel): bit j = hi[j] rows 16-byte aligned, bit 15 = lo
};

template <typename T> struct Vec2Of;
template <> struct Vec2Of<double> { using type = double2; };
template <> struct Vec2Of<float> { using type = float2; };

template <typename T, int L, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) mat_fwd_fused_kernel(const __grid_constant__ MatFusedParams<T> p) {
    using V2 = typename Vec2Of<T>::type;
    constexpr int HL = L / 2 - 1, HR = L / 2;
    constexpr int DELTA = HL & 1;                 // parity of the first sample of an even output's window
    constexpr int PQ = ((HL + 1) / 2) & 1;        // parity of the first polyphase index (ranges start at multiples of 4)
    constexpr int NE = (L + 2 + DELTA + 1) / 2;   // polyphase entries covering the window of an output pair
    constexpr int NEV = (NE + PQ + 1) / 2 * 2;    // rounded to whole 2-element vectors

    extern __shared__ __align__(128) unsigned char smem_raw[];
    T* bufA = reinterpret_cast<T*>(smem_raw);     // even | odd arrays of the current level input
    const int capA = p.cap0 / 2 + 8;              // entries per polyphase array (level 0)
    T* bufB = bufA + 2 * capA;                    // even | odd arrays of the next level
    // interleaved samples of the NEXT chunk, filled by cp.async (16-byte aligned destination)
    T* raw = reinterpret_cast<T*>((reinterpret_cast<uintptr_t>(bufB + 2 * (p.cap0 / 4 + 16)) + 15) & ~uintptr_t(15));

    const int tid = threadIdx.x;
    const int b = blockIdx.y;
    const int K = p.k;
    const T* __restrict__ xb = p.x + (int64_t)b * p.x_stride;

    // A CTA streams `cpc` consecutive chunks of one row: while chunk c is taken through the K levels, the samples of
    // chunk c + 1 travel into `raw` with cp.async.
    // ranges: rlo[j], rhi[j] = level-j indices this CTA computes (j >= 1) / stages (j = 0) for one chunk; two sets in
    // shared memory (current chunk / prefetched chunk).  In registers the run-time level index costs a local array.
    __shared__ int s_r[2][2][MATF_MAXK + 1];
    const int nchunks = (p.n[K] + p.tk - 1) / p.tk;
    const int c_first = blockIdx.x * p.cpc, c_last = min(c_first + p.cpc, nchunks);
    if (c_first >= nchunks) return;
    auto ranges = [&](int chunk, int set) {
        int lo_j = chunk * p.tk, hi_j = min(lo_j + p.tk, p.n[K]);
        s_r[set][0][K] = lo_j; s_r[set][1][K] = hi_j;
        for (int j = K; j >= 1; --j) {
            const int half = p.n[j];                  // outputs of level j
            int lo = 2 * lo_j - HL, hi = 2 * (hi_j - 1) + HR + 1;
            if (lo_j < p.nb_top[j - 1]) lo = 0, hi = max(hi, p.w_left[j - 1]);
            if (hi_j > half - p.nb_bot[j - 1]) hi = p.n[j - 1], lo = min(lo, p.n[j - 1] - p.w_right[j - 1]);
            lo = max(lo, 0) & ~3;                     // multiple of 4: polyphase index starts even
            hi = min(hi, p.n[j - 1]);
            s_r[set][0][j - 1] = lo_j = lo;
            s_r[set][1][j - 1] = hi_j = hi;
        }
    };
    // asynchronous copy of samples [s0, s1) of the row into raw[0 ..): 16-byte pieces, element-sized tail
    auto prefetch = [&](int s0, int s1) {
        constexpr int VE = 16 / (int)sizeof(T);
        const int cnt = s1 - s0;
        const int nv = ((uintptr_t)(xb + s0) & 15) ? 0 : cnt / VE;   // float rows with a stride of 2 (mod 4) samples
        for (int q = tid; q < nv; q += NT) {
            const unsigned dst = (unsigned)__cvta_generic_to_shared(raw + VE * q);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(xb + s0 + VE * q) : "memory");
        }
        for (int q = nv * VE + tid; q < cnt; q += NT) {
            const unsigned dst = (unsigned)__cvta_generic_to_shared(raw + q);
            if (sizeof(T) == 8)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(xb + s0 + q) : "memory");
            else
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(xb + s0 + q) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    if (tid == 0) ranges(c_first, 0);
    __syncthreads();
    prefetch(s_r[0][0][0], s_r[0][1][0]);

    int set = 0;
    for (int chunk = c_first; chunk < c_last; ++chunk, set ^= 1) {
    const int* rlo = s_r[set][0];
    const int* rhi = s_r[set][1];
    if (tid == 0 && chunk + 1 < c_last) ranges(chunk + 1, set ^ 1);
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();                                  // raw holds this chunk; the next chunk's ranges are visible

    // de-interleave the staged samples: raw -> even | odd polyphase arrays
    {
        const int cnt = rhi[0] - rlo[0];
        T* ev = bufA;
        T* od = bufA + capA;
        for (int q = tid; 2 * q < cnt; q += NT) {
            if (2 * q + 1 < cnt) {
                const V2 v = *reinterpret_cast<const V2*>(raw + 2 * q);
                ev[q] = v.x; od[q] = v.y;
            } else {
                ev[q] = raw[2 * q]; od[q] = T(0);
            }
        }
    }
    __syncthreads();                                  // raw is free again
    if (chunk + 1 < c_last) prefetch(s_r[set ^ 1][0][0], s_r[set ^ 1][1][0]);

    T* cur = bufA;
    int cur_cap = capA;
    T* nxt = bufB;
#pragma unroll 1
    for (int j = 1; j <= K; ++j) {
        const int half = p.n[j];
        const int nprev = p.n[j - 1];
        const int in0 = rlo[j - 1];               // sample index of polyphase entry 0
        const int nxt_cap = ((rhi[j] - rlo[j]) / 2 + 9) & ~1;   // even: the odd array stays 16-byte aligned
        const T* ev = cur;
        const T* od = cur + cur_cap;
        T* nev = nxt;
        T* nod = nxt + nxt_cap;
        const int own0 = (chunk * p.tk) << (K - j), own1 = min(((chunk + 1) * p.tk) << (K - j), half);
        T* __restrict__ hib = p.hi[j - 1] + (int64_t)b * p.hi_stride[j - 1];
        T* __restrict__ lob = p.lo + (int64_t)b * p.lo_stride;
        const int nbt = p.nb_top[j - 1], nbb = p.nb_bot[j - 1];
        const int npairs = (rhi[j] - rlo[j] + 1) / 2;
        const bool vec_ok = !((uintptr_t)hib & (2 * sizeof(T) - 1)) && !(p.hi_stride[j - 1] & 1) &&
                            (j < K || (!((uintptr_t)lob & (2 * sizeof(T) - 1)) && !(p.lo_stride & 1)));
        for (int pr = tid; pr < npairs; pr += NT) {
            const int i = rlo[j] + 2 * pr;        // even output index
            T alo[2] = {T(0), T(0)}, ahi[2] = {T(0), T(0)};
            const int q0 = ((2 * i - HL - in0) >> 1) - PQ;           // even polyphase index of the first load
            const bool interior = (i >= nbt) && (i + 1 < half - nbb) && (q0 >= 0);
            if (interior) {
                // window of the pair: samples 2i - HL .. 2i + 2 + HR
                T e[NEV], o[NEV];
#pragma unroll
                for (int v = 0; v < NEV / 2; ++v) {
                    const V2 a = *reinterpret_cast<const V2*>(ev + q0 + 2 * v);
                    const V2 c = *reinterpret_cast<const V2*>(od + q0 + 2 * v);
                    e[2 * v] = a.x; e[2 * v + 1] = a.y; o[2 * v] = c.x; o[2 * v + 1] = c.y;
                }
#pragma unroll
                for (int r = 0; r < 2; ++r) {
#pragma unroll
                    for (int k = 0; k < L; ++k) {
                        const int d = 2 * r + k + DELTA + 2 * PQ;    // offset from sample in0 + 2 q0
                        const T s = (d & 1) ? o[d >> 1] : e[d >> 1];
                        alo[r] = fma(p.flo[k], s, alo[r]);
                        ahi[r] = fma(p.fhi[k], s, ahi[r]);
                    }
                }
            } else {
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int ii = i + r;
                    if (ii >= half) continue;
                    auto sample = [&](int s) -> T {
                        const int d = s - in0;
                        return (d & 1) ? od[d >> 1] : ev[d >> 1];
                    };
                    if (ii < nbt || ii >= half - nbb) {
                        const int rr = ii < nbt ? ii : nbt + (ii - (half - nbb));
                        const bool top = ii < nbt;
                        // dense boundary row: all block loads are issued up front (fixed trip count)
                        const int w = top ? p.w_left[j - 1] : p.w_right[j - 1];
                        const int s0 = top ? 0 : nprev - w;
                        const T* __restrict__ bl_ = (top ? p.lo_left[j - 1] : p.lo_right[j - 1]) + rr * w;
                        const T* __restrict__ bh_ = (top ? p.hi_left[j - 1] : p.hi_right[j - 1]) + rr * w;
                        T cl[16], ch[16];
#pragma unroll
                        for (int c = 0; c < 16; ++c) {
                            cl[c] = c < w ? __ldg(bl_ + c) : T(0);
                            ch[c] = c < w ? __ldg(bh_ + c) : T(0);
                        }
#pragma unroll
                        for (int c = 0; c < 16; ++c) {
                            if (c < w) {
                                const T sv = sample(s0 + c);
                                alo[r] = fma(cl[c], sv, alo[r]);
                                ahi[r] = fma(ch[c], sv, ahi[r]);
                            }
                        }
                        for (int c = 16; c < w; ++c) {   // wider blocks than any orthogonal wavelet <= 16 taps produces
                            const T sv = sample(s0 + c);
                            alo[r] = fma(__ldg(bl_ + c), sv, alo[r]);
                            ahi[r] = fma(__ldg(bh_ + c), sv, ahi[r]);
                        }
                    } else {
                        for (int k = 0; k < L; ++k) {
                            const int s = 2 * ii - HL + k;
                            if (s < 0 || s >= nprev) continue;
                            const T v = sample(s);
                            alo[r] = fma(p.flo[k], v, alo[r]);
                            ahi[r] = fma(p.fhi[k], v, ahi[r]);
                        }
                    }
                }
            }
            // approximation -> next level (de-interleaved), detail -> HBM (owned range only)
            const int rel = (i - rlo[j]) >> 1;
            if (j < K) { nev[rel] = alo[0]; nod[rel] = alo[1]; }
            if (i >= own0 && i + 1 < own1 && vec_ok) {
                // i is even and the rows are 16-byte aligned: one 128-bit (f64) / 64-bit (f32) store per band
                V2 hv; hv.x = ahi[0]; hv.y = ahi[1];
                *reinterpret_cast<V2*>(hib + i) = hv;
                if (j == K) { V2 lv; lv.x = alo[0]; lv.y = alo[1]; *reinterpret_cast<V2*>(lob + i) = lv; }
            } else {
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int ii = i + r;
                    if (ii >= own0 && ii < own1) {
                        hib[ii] = ahi[r];
                        if (j == K) lob[ii] = alo[r];
                    }
                }
            }
        }
        __syncthreads();
        T* t = const_cast<T*>(cur); cur = nxt; nxt = t;
        cur_cap = nxt_cap;
    }
    }   // chunks of this CTA
}


// Host: fill the levels of one analysis group (level indices l .. l+k-1 of the caller's arrays) for either cascade
// launcher, launch_mat_fwd_fused below or launch_mat_fwd_dmma2 (matrix_dmma.cuh).  false = the group is not one
// cascade (odd or trimmed lengths inside it, or corner blocks that meet).
template <typename T>
static bool fill_mat_fused_levels(MatFusedParams<T>& p, int L, int k, const int64_t* n, const int32_t* nbt,
                                  const int32_t* nbb, const int32_t* wl, const int32_t* wr,
                                  const T* const* blk_ptrs /* 4 per level */, const T* x, int64_t xs, void* const* hi_out,
                                  const int64_t* hi_stride, T* lo_out, int64_t lo_stride, const Taps<T>& taps) {
    memset(&p, 0, sizeof(p));
    p.x = x; p.x_stride = xs; p.k = k;
    p.n[0] = (int)n[0];
    for (int j = 0; j < k; ++j) {
        if (n[j] & 1) return false;
        p.n[j + 1] = (int)(n[j] / 2);
        if (j + 1 < k && n[j + 1] != n[j] / 2) return false;
        p.hi[j] = (T*)hi_out[j]; p.hi_stride[j] = hi_stride[j];
        p.nb_top[j] = nbt[j]; p.nb_bot[j] = nbb[j]; p.w_left[j] = wl[j]; p.w_right[j] = wr[j];
        p.lo_left[j] = blk_ptrs[4 * j]; p.lo_right[j] = blk_ptrs[4 * j + 1];
        p.hi_left[j] = blk_ptrs[4 * j + 2]; p.hi_right[j] = blk_ptrs[4 * j + 3];
        if (nbt[j] + nbb[j] > p.n[j + 1]) return false;
    }
    p.lo = lo_out; p.lo_stride = lo_stride;
    for (int q = 0; q < L; ++q) { p.flo[q] = taps.lo[L - 1 - q]; p.fhi[q] = taps.hi[L - 1 - q]; }
    return true;
}

// Host: launch one fused group of k levels.
template <typename T>
static bool launch_mat_fwd_fused(int L, int k, const int64_t* n, const int32_t* nbt, const int32_t* nbb, const int32_t* wl,
                                 const int32_t* wr, const T* const* blk_ptrs /* 4 per level */, const T* x, int64_t xs,
                                 int64_t batch, void* const* hi_out, const int64_t* hi_stride, T* lo_out, int64_t lo_stride,
                                 const Taps<T>& taps, cudaStream_t st, cudaError_t* err) {
    *err = cudaSuccess;
    if ((L & 1) || L < 2 || L > 16 || k < 2 || k > MATF_MAXK || batch > 65535) return false;
    if (((uintptr_t)x & 15) || (xs & 1) || n[0] >= (int64_t(1) << 30)) return false;
    MatFusedParams<T> p;
    if (!fill_mat_fused_levels(p, L, k, n, nbt, nbb, wl, wr, blk_ptrs, x, xs, hi_out, hi_stride, lo_out, lo_stride, taps))
        return false;
    const int nk = p.n[k];
    int chunk0 = sizeof(T) == 8 ? 2048 : 4096;                    // level-0 samples per chunk
    if (knob_is_set(K_MATF_CHUNK)) { const int v = (int)knob_val(K_MATF_CHUNK, 0); if (v >= 64 && v <= 16384) chunk0 = v; }
    if (n[0] <= 8192 && n[0] > chunk0) chunk0 = (int)n[0];        // short rows: the whole row is one chunk
    int tk = chunk0 >> k;
    if (tk < 4) tk = 4;
    tk = (tk + 3) & ~3;
    if (tk > nk) tk = (nk + 3) & ~3;
    p.tk = tk;
    int cap0 = (tk << k) + ((L + 6) << k) + 64;
    if (cap0 > p.n[0] + 16) cap0 = (p.n[0] + 16 + 3) & ~3;
    cap0 = (cap0 + 3) & ~3;
    p.cap0 = cap0;
    const size_t smem = (size_t)(2 * (cap0 / 2 + 8) + 2 * (cap0 / 4 + 16) + cap0) * sizeof(T) + 16;
    if (smem > 200 * 1024) return false;
    const int nchunks = (nk + tk - 1) / tk;
    int cpc = (int)knob_val(K_MATF_CPC, 8);
    if (cpc < 1) cpc = 1;
    while (cpc > 1 && (int64_t)((nchunks + cpc - 1) / cpc) * batch < 4 * sm_count()) cpc /= 2;   // keep the machine full
    p.cpc = cpc;
    dim3 grid((nchunks + cpc - 1) / cpc, (unsigned)batch);
    // CTA shape: 128 threads for small chunks (more CTAs per SM: the staging loads of one overlap the cascade of the
    // others), 256 for large ones.  MATF_NT / MATF_MINB override.
    int nt = chunk0 <= 2048 ? 128 : 256;
    if (knob_is_set(K_MATF_NT)) nt = knob_val(K_MATF_NT, 256) == 128 ? 128 : 256;
    const int minb = (int)knob_val(K_MATF_MINB, 1);
#define WTB_MF_LAUNCH(LL, NTT, MB)                                                                              \
    {                                                                                                           \
        cudaError_t e = ensure_dyn_smem(mat_fwd_fused_kernel<T, LL, NTT, MB>, smem > 200 * 1024 ? smem : 200 * 1024); \
        if (e != cudaSuccess) { *err = e; return true; }                                                        \
        mat_fwd_fused_kernel<T, LL, NTT, MB><<<grid, NTT, smem, st>>>(p);                                       \
    }
#define WTB_MF(LL)                                                                                              \
    case LL: {                                                                                                  \
        if (nt == 128) { if (minb > 1) WTB_MF_LAUNCH(LL, 128, 6) else WTB_MF_LAUNCH(LL, 128, 1) }                  \
        else { if (minb > 1) WTB_MF_LAUNCH(LL, 256, 3) else WTB_MF_LAUNCH(LL, 256, 1) }                            \
        break;                                                                                                  \
    }
    switch (L) {
        WTB_MF(2) WTB_MF(4) WTB_MF(6) WTB_MF(8) WTB_MF(10) WTB_MF(12) WTB_MF(14) WTB_MF(16)
        default: return false;
    }
#undef WTB_MF_LAUNCH
#undef WTB_MF
    *err = cudaGetLastError();
    return true;
}

}  // namespace wtb
