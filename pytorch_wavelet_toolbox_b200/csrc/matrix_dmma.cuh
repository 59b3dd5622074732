// matrix_dmma.cuh -- the boundary-filter matrix FWT (float64) on the FP64 TENSOR CORES.
//
// north_star: "tensor cores are used only for the MatrixWavedec path where the boundary-filter sparse matmul is
// reformulated as a banded dense contraction".  The level operator A_n of the reference
// (torch.sparse.mm(A_level, .), src/ptwt/matmul_transform.py:409-425) is block-Toeplitz away from its corner blocks:
// every output pair (lo[i], hi[i]) is the same L-tap window sliding by two samples.  Four consecutive outputs of both
// bands (8 rows) read one window of L + 6 samples, so a tile of 8 such groups is the dense product
//
//     D[8 x 8] = A[8 x (L+6)] * B[(L+6) x 8],   A[(band, s)][u] = f_band[u - 2 s],   B[u][g] = x[2 i0 + 8 g - HL + u]
//
// evaluated with mma.sync.aligned.m8n8k4.f64 (DMMA, the FP64 tensor-core instruction of sm_90; wgmma has no f64
// kind): about (L+6)/4 instructions of 256 FMAs for 64 outputs.  60 % of those FMAs multiply structural zeros of A --
// the price of the dense form -- but the scalar kernel is bound by instruction issue, not by the FP64 pipe, and the
// DMMA form needs ~0.3 warp instructions per output instead of 1.5.
//
// Everything around the contraction is the streaming cascade of matrix_fused.cuh: a CTA takes consecutive chunks of one
// row through K levels, level inputs live in shared memory (interleaved, as the B fragment wants them), the next chunk
// arrives by cp.async meanwhile, details go to HBM, the corner blocks (dense orthogonalised boundary rows) are applied
// by scalar code in the CTAs at the two ends.
#pragma once

#include "matrix_fused.cuh"

namespace wtb {

__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, const double a, const double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d0), "+d"(d1)
                 : "d"(a), "d"(b));
}

template <int L, int NT, bool PERM>
__global__ void __launch_bounds__(NT) mat_fwd_dmma_kernel(const __grid_constant__ MatFusedParams<double> p) {
    constexpr int HL = L / 2 - 1, HR = L / 2;
    // The contraction index u (window sample of a group of 4 outputs) is split as u = E * k + e: lane k of a fragment
    // column holds E CONSECUTIVE samples (E even, window start shifted by SH to an even sample), so the B fragments of
    // one tile are E / 2 aligned 128-bit shared loads per lane (conflict-free for E = 6) instead of one 64-bit load per
    // k-step with 4-way bank conflicts; the A fragment is permuted the same way.
    // PERM = false: u = 4 e + k (E = ceil((L + 6) / 4) k-steps, one 64-bit load each, 4-way conflicts).
    constexpr int SH = PERM ? (HL & 1) : 0;
    constexpr int E = PERM ? ((L + 6 + SH + 3) / 4 + 1) / 2 * 2 : (L + 6 + 3) / 4;
    constexpr int KS = PERM ? E : 1;              // stride of the lane index k in the window
    constexpr int ES = PERM ? 1 : 4;              // stride of the k-step e in the window
    constexpr int NW = NT / 32;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* raw0 = reinterpret_cast<double*>(smem_raw);   // level-0 samples of the current / next chunk (two buffers)
    double* raw1 = raw0 + p.cap0;
    double* levA = raw1 + p.cap0;                          // approximations, alternating
    double* levB = levA + (p.cap0 / 2 + 16);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.y;
    const int K = p.k;
    const double* __restrict__ xb = p.x + (int64_t)b * p.x_stride;

    __shared__ int s_r[2][2][MATF_MAXK + 1];
    const int nchunks = (p.n[K] + p.tk - 1) / p.tk;
    const int c_first = blockIdx.x * p.cpc, c_last = min(c_first + p.cpc, nchunks);
    if (c_first >= nchunks) return;
    auto ranges = [&](int chunk, int set) {
        int lo_j = chunk * p.tk, hi_j = min(lo_j + p.tk, p.n[K]);
        s_r[set][0][K] = lo_j; s_r[set][1][K] = hi_j;
        for (int j = K; j >= 1; --j) {
            const int half = p.n[j];
            int lo = 2 * lo_j - HL, hi = 2 * (hi_j - 1) + HR + 1;
            if (lo_j < p.nb_top[j - 1]) lo = 0, hi = max(hi, p.w_left[j - 1]);
            if (hi_j > half - p.nb_bot[j - 1]) hi = p.n[j - 1], lo = min(lo, p.n[j - 1] - p.w_right[j - 1]);
            lo = max(lo, 0) & ~3;
            hi = min(hi, p.n[j - 1]);
            s_r[set][0][j - 1] = lo_j = lo;
            s_r[set][1][j - 1] = hi_j = hi;
        }
    };
    auto prefetch = [&](double* dst, int s0, int s1) {
        const int cnt = s1 - s0, nv = cnt / 2;
        for (int q = tid; q < nv; q += NT) {
            const unsigned d = (unsigned)__cvta_generic_to_shared(dst + 2 * q);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(xb + s0 + 2 * q) : "memory");
        }
        if ((cnt & 1) && tid == 0) {
            const unsigned d = (unsigned)__cvta_generic_to_shared(dst + cnt - 1);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(xb + s1 - 1) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    // A fragment (row-major 8 x 4 per k-step e): this lane holds A[m = lane / 4][u = E * (lane % 4) + e],
    // row m = 4 * band + s  ->  f_band[u - SH - 2 s]
    double afrag[E];
    {
        const int m = lane >> 2, band = m >> 2, s = m & 3;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const int kk = KS * (lane & 3) + ES * e - SH - 2 * s;
            afrag[e] = (kk >= 0 && kk < L) ? (band ? p.fhi[kk] : p.flo[kk]) : 0.0;
        }
    }
    const int frag_n = lane >> 2, frag_k = lane & 3;      // B fragment: B[k = lane % 4][n = lane / 4]
    const int out_band = lane >> 4, out_s = (lane >> 2) & 3;
    const int out_g0 = 2 * (lane & 3);                     // D fragment: columns (groups) 2 (lane % 4), + 1

    if (tid == 0) ranges(c_first, 0);
    __syncthreads();
    prefetch(raw0, s_r[0][0][0], s_r[0][1][0]);

    int set = 0;
    for (int chunk = c_first; chunk < c_last; ++chunk, set ^= 1) {
        const int* rlo = s_r[set][0];
        const int* rhi = s_r[set][1];
        double* in = set ? raw1 : raw0;
        if (tid == 0 && chunk + 1 < c_last) ranges(chunk + 1, set ^ 1);
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();                              // this chunk's samples landed; the next chunk's ranges are visible
        if (chunk + 1 < c_last) prefetch(set ? raw0 : raw1, s_r[set ^ 1][0][0], s_r[set ^ 1][1][0]);

        double* nxt = levA;
#pragma unroll 1
        for (int j = 1; j <= K; ++j) {
            const int half = p.n[j], nprev = p.n[j - 1];
            const int in0 = rlo[j - 1], in_cnt = rhi[j - 1] - rlo[j - 1];
            const int o0 = rlo[j], o1 = rhi[j];
            const int own0 = (chunk * p.tk) << (K - j), own1 = min(((chunk + 1) * p.tk) << (K - j), half);
            const int nbt = p.nb_top[j - 1], nbb = p.nb_bot[j - 1];
            double* __restrict__ hib = p.hi[j - 1] + (int64_t)b * p.hi_stride[j - 1];
            double* __restrict__ lob = p.lo + (int64_t)b * p.lo_stride;
            const bool last = j == K;

            // ---- interior outputs: tiles of 32 output positions x 2 bands, one warp per tile ----------------------
            const int ntiles = (o1 - o0 + 31) / 32;
            const int lo_all = max(nbt, o0), hi_all = min(half - nbb, o1);
            // Tiles [t_lo, t_hi) are "fast": all 32 outputs are interior ones of this chunk and every sample of their
            // windows is staged (the conditions are linear in the tile index, so the range is computed once per level).
            int t_lo, t_hi;
            {
                const int need0 = max(lo_all - o0, (HL + SH + in0 + 1) / 2 - o0);          // first admissible i0 - o0
                t_lo = need0 > 0 ? (need0 + 31) / 32 : 0;
                const int lim_out = (hi_all - o0) / 32;                                     // i0 + 32 <= hi_all
                const int lim_in = in_cnt - 56 - 4 * E + HL + SH + in0 - 2 * o0;            // 2 (i0 - o0) <= lim_in
                t_hi = min(lim_out, lim_in >= 0 ? lim_in / 64 + 1 : 0);
                t_hi = max(min(t_hi, ntiles), t_lo);
            }
            auto generic_tile = [&](const int t) {
                const int i0 = o0 + 32 * t;
                const int rel0 = 2 * i0 + 8 * frag_n - HL - SH + KS * frag_k - in0;
                double c0 = 0.0, c1 = 0.0;
                const int ia = i0 + 4 * out_g0 + out_s, ib = ia + 4;
                // samples clamped into the staged range (only outputs that the corner-block code below overwrites, or
                // that lie beyond o1, can touch the clamp), stores checked one by one
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const int rel = min(max(rel0 + ES * e, 0), in_cnt - 1);
                    dmma_m8n8k4(c0, c1, afrag[e], in[rel]);
                }
                if (out_band == 0) {
                    if (!last) {
                        if (ia < o1) nxt[ia - o0] = c0;
                        if (ib < o1) nxt[ib - o0] = c1;
                    } else {
                        if (ia >= own0 && ia < own1 && ia >= nbt && ia < half - nbb) lob[ia] = c0;
                        if (ib >= own0 && ib < own1 && ib >= nbt && ib < half - nbb) lob[ib] = c1;
                    }
                } else {
                    if (ia >= own0 && ia < own1 && ia >= nbt && ia < half - nbb) hib[ia] = c0;
                    if (ib >= own0 && ib < own1 && ib >= nbt && ib < half - nbb) hib[ib] = c1;
                }
            };
            for (int t = warp; t < t_lo; t += NW) generic_tile(t);
            for (int t = t_hi + warp; t < ntiles; t += NW) generic_tile(t);
            {
                // fast tiles: running pointers, no range checks besides the owned range of the global stores
                const int tf = t_lo + warp;
                int ia = o0 + 32 * tf + 4 * out_g0 + out_s;
                const double* src = in + (2 * (o0 + 32 * tf) + 8 * frag_n - HL - SH + KS * frag_k - in0);
                double* dsm = nxt + (ia - o0);
                double* dgl = (out_band ? hib : lob) + ia;
                const bool to_smem = out_band == 0 && !last;
                for (int t = tf; t < t_hi; t += NW) {
                    double c0 = 0.0, c1 = 0.0;
                    if constexpr (PERM) {
#pragma unroll
                        for (int e = 0; e < E; e += 2) {
                            const double2 v = *reinterpret_cast<const double2*>(src + e);
                            dmma_m8n8k4(c0, c1, afrag[e], v.x);
                            dmma_m8n8k4(c0, c1, afrag[e + 1], v.y);
                        }
                    } else {
                        double v[E];
#pragma unroll
                        for (int e = 0; e < E; ++e) v[e] = src[4 * e];
#pragma unroll
                        for (int e = 0; e < E; ++e) dmma_m8n8k4(c0, c1, afrag[e], v[e]);
                    }
                    if (to_smem) {
                        dsm[0] = c0; dsm[4] = c1;
                    } else {
                        if (ia >= own0 && ia < own1) dgl[0] = c0;
                        if (ia + 4 >= own0 && ia + 4 < own1) dgl[4] = c1;
                    }
                    src += 64 * NW; dsm += 32 * NW; dgl += 32 * NW; ia += 32 * NW;
                }
            }
            __syncthreads();
            // ---- corner blocks: the dense orthogonalised boundary rows (the CTAs at the two ends of the row) -------
            if (o0 < nbt || o1 > half - nbb) {
                // outputs [o0, min(o1, nbt)) and [max(o0, half - nbb), o1), both bands
                const int nt_ = max(min(o1, nbt) - o0, 0);
                const int b0 = max(o0, half - nbb), nb_ = max(o1 - b0, 0);
                for (int q = tid; q < 2 * (nt_ + nb_); q += NT) {
                    const int band = q & 1, r = q >> 1;
                    const int ii = r < nt_ ? o0 + r : b0 + (r - nt_);
                    const bool top = ii < nbt;
                    const int rr = top ? ii : nbt + (ii - (half - nbb));
                    const int w = top ? p.w_left[j - 1] : p.w_right[j - 1];
                    const int s0 = top ? 0 : nprev - w;
                    const double* __restrict__ blk = (top ? (band ? p.hi_left[j - 1] : p.lo_left[j - 1])
                                                          : (band ? p.hi_right[j - 1] : p.lo_right[j - 1])) + rr * w;
                    double acc = 0.0;
                    for (int c = 0; c < w; ++c) acc = fma(__ldg(blk + c), in[s0 + c - in0], acc);
                    if (band == 0) {
                        if (!last) nxt[ii - o0] = acc;
                        else if (ii >= own0 && ii < own1) lob[ii] = acc;
                    } else if (ii >= own0 && ii < own1) {
                        hib[ii] = acc;
                    }
                }
                __syncthreads();
            }
            in = nxt;
            nxt = (nxt == levA) ? levB : levA;
        }
    }
}

// Host: launch one fused group of k levels on the FP64 tensor cores; false = not applicable (caller falls back).
static bool launch_mat_fwd_dmma(int L, int k, const int64_t* n, const int32_t* nbt, const int32_t* nbb, const int32_t* wl,
                                const int32_t* wr, const double* const* blk_ptrs, const double* x, int64_t xs, int64_t batch,
                                void* const* hi_out, const int64_t* hi_stride, double* lo_out, int64_t lo_stride,
                                const Taps<double>& taps, cudaStream_t st, cudaError_t* err) {
    *err = cudaSuccess;
    if ((L & 1) || L < 2 || L > 16 || k < 1 || k > MATF_MAXK || batch > 65535) return false;
    if (((uintptr_t)x & 15) || (xs & 1) || n[0] >= (int64_t(1) << 30)) return false;
    MatFusedParams<double> p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.x_stride = xs; p.k = k;
    p.n[0] = (int)n[0];
    for (int j = 0; j < k; ++j) {
        if (n[j] & 1) return false;
        p.n[j + 1] = (int)(n[j] / 2);
        if (j + 1 < k && n[j + 1] != n[j] / 2) return false;
        p.hi[j] = (double*)hi_out[j]; p.hi_stride[j] = hi_stride[j];
        p.nb_top[j] = nbt[j]; p.nb_bot[j] = nbb[j]; p.w_left[j] = wl[j]; p.w_right[j] = wr[j];
        p.lo_left[j] = blk_ptrs[4 * j]; p.lo_right[j] = blk_ptrs[4 * j + 1];
        p.hi_left[j] = blk_ptrs[4 * j + 2]; p.hi_right[j] = blk_ptrs[4 * j + 3];
        if (nbt[j] + nbb[j] > p.n[j + 1]) return false;
    }
    p.lo = lo_out; p.lo_stride = lo_stride;
    for (int q = 0; q < L; ++q) { p.flo[q] = taps.lo[L - 1 - q]; p.fhi[q] = taps.hi[L - 1 - q]; }
    const int nk = p.n[k];
    int chunk0 = 2048;
    if (knob_is_set(K_MATF_CHUNK)) { const int v = (int)knob_val(K_MATF_CHUNK, 0); if (v >= 64 && v <= 16384) chunk0 = v; }
    if (n[0] <= 8192 && n[0] > chunk0) chunk0 = (int)n[0];
    int tk = chunk0 >> k;
    if (tk < 4) tk = 4;
    tk = (tk + 3) & ~3;
    if (tk > nk) tk = (nk + 3) & ~3;
    p.tk = tk;
    int cap0 = (tk << k) + ((L + 6) << k) + 64;
    if (cap0 > p.n[0] + 16) cap0 = (p.n[0] + 16 + 3) & ~3;
    cap0 = (cap0 + 3) & ~3;
    p.cap0 = cap0;
    const size_t smem = (size_t)(2 * cap0 + (cap0 / 2 + 16) + (cap0 / 4 + 16)) * sizeof(double);
    if (smem > 200 * 1024) return false;
    const int nchunks = (nk + tk - 1) / tk;
    int cpc = (int)knob_val(K_MATF_CPC, 8);
    if (cpc < 1) cpc = 1;
    const int64_t min_ctas = knob_val(K_MATF_MINCTAS, 4 * sm_count());
    while (cpc > 1 && (int64_t)((nchunks + cpc - 1) / cpc) * batch < min_ctas) cpc /= 2;
    p.cpc = cpc;
    dim3 grid((nchunks + cpc - 1) / cpc, (unsigned)batch);
    const int nt = knob_val(K_MATF_NT, 128) == 256 ? 256 : 128;
    const bool perm = knob_on(K_DMMA_PERM);
#define WTB_MD_LAUNCH(LL, NTT, PP)                                                                     \
    {                                                                                                  \
        cudaError_t e = ensure_dyn_smem(mat_fwd_dmma_kernel<LL, NTT, PP>, 200 * 1024);                 \
        if (e != cudaSuccess) { *err = e; return true; }                                               \
        mat_fwd_dmma_kernel<LL, NTT, PP><<<grid, NTT, smem, st>>>(p);                                  \
    }
#define WTB_MD(LL)                                                                                     \
    case LL:                                                                                           \
        if (nt == 128) { if (perm) WTB_MD_LAUNCH(LL, 128, true) else WTB_MD_LAUNCH(LL, 128, false) }      \
        else { if (perm) WTB_MD_LAUNCH(LL, 256, true) else WTB_MD_LAUNCH(LL, 256, false) }                \
        break;
    switch (L) {
        WTB_MD(2) WTB_MD(4) WTB_MD(6) WTB_MD(8) WTB_MD(10) WTB_MD(12) WTB_MD(14) WTB_MD(16)
        default: return false;
    }
#undef WTB_MD
#undef WTB_MD_LAUNCH
    *err = cudaGetLastError();
    return true;
}


// ==========================================================================================
// The analysis cascade again, laid out like the synthesis kernel below (conflict-free polyphase operand loads, which
// the kernel above lacks): one chunk per CTA, every level input kept as two POLYPHASE arrays
// (even samples | odd samples, the odd array two doubles further in the bank pattern), the DATA in the A operand and
// the polyphase FILTER matrix in the B operand:
//
//     D[8 groups x (2 bands x 4 outputs)] = A[8 x 4 KS] * B[4 KS x 8],
//         A[g][u = (phase, v)] = x_phase[i0 + 4 g + v - C_phase],   B[u][(band, s)] = f_band[2 (v - s) + (phase ^ b)]
//
// so that the A fragment of a k-step is one conflict-free 64-bit shared load per lane and the D fragment of a lane is
// an output PAIR of one band: the approximation pair goes to the next level's even / odd arrays (two conflict-free
// 64-bit stores), the detail pair to HBM as one 128-bit store (a quarter-warp writes 128 contiguous bytes).
// ==========================================================================================
template <int L, int NT>
__global__ void __launch_bounds__(NT) mat_fwd_dmma2_kernel(const __grid_constant__ MatFusedParams<double> p) {
    constexpr int H = L / 2, HL = H - 1, HR = H;
    constexpr int B1 = HL & 1, AA = HL >> 1;
    constexpr int CE = AA, CO = AA + B1;          // x[2 i - HL + m]: even phase starts at i - CE, odd phase at i - CO
    constexpr int KS = (H + 4) / 2;               // k-steps: H + 3 window positions of each phase, padded to even
    constexpr int OFFO = B1 ? 3 : 2;              // odd array: two doubles further in the bank pattern (CO - CE = B1)
    constexpr int NW = NT / 32;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int h0 = p.cap0 / 2 + 8, hA = p.cap0 / 4 + 8, hB = p.cap0 / 8 + 8;   // capacity of one phase array
    double* buf0 = reinterpret_cast<double*>(smem_raw);
    double* bufA = buf0 + 2 * h0 + 4;
    double* bufB = bufA + 2 * hA + 4;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.y;
    const int K = p.k;
    const int chunk = blockIdx.x;
    const double* __restrict__ xb = p.x + (int64_t)b * p.x_stride;

    __shared__ int s_lo[MATF_MAXK + 1], s_hi[MATF_MAXK + 1];
    if (tid == 0) {
        int lo_j = chunk * p.tk, hi_j = min(lo_j + p.tk, p.n[K]);
        s_lo[K] = lo_j; s_hi[K] = hi_j;
        for (int j = K; j >= 1; --j) {
            const int half = p.n[j];
            int lo = 2 * lo_j - HL, hi = 2 * (hi_j - 1) + HR + 1;
            if (lo_j < p.nb_top[j - 1]) lo = 0, hi = max(hi, p.w_left[j - 1]);
            if (hi_j > half - p.nb_bot[j - 1]) hi = p.n[j - 1], lo = min(lo, p.n[j - 1] - p.w_right[j - 1]);
            lo = max(lo, 0) & ~3;
            hi = min(hi, p.n[j - 1]);
            s_lo[j - 1] = lo_j = lo;
            s_hi[j - 1] = hi_j = hi;
        }
    }
    __syncthreads();

    // level-0 samples -> polyphase arrays (8-byte cp.async: thread parity = phase, NT is even)
    {
        const int s0 = s_lo[0], cnt = s_hi[0] - s0;
        double* dst = (tid & 1) ? buf0 + h0 + OFFO : buf0;
        for (int q = tid; q < cnt; q += NT) {
            const unsigned d = (unsigned)__cvta_generic_to_shared(dst + (q >> 1));
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(xb + s0 + q) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }

    // B fragment (the polyphase filter matrix): lane holds B[k = lane % 4][n = lane / 4] of k-step e
    double bfrag[KS];
    {
        const int nn = lane >> 2, k = lane & 3, band = nn >> 2, s = nn & 3, par = k & 1;
#pragma unroll
        for (int e = 0; e < KS; ++e) {
            const int w = 2 * e + (k >> 1) - s;
            const int tap = 2 * w + (par ^ B1);
            bfrag[e] = (w >= 0 && w < H) ? (band ? p.fhi[tap] : p.flo[tap]) : 0.0;
        }
    }
    const int a_par = lane & 1;
    const int a_off = 4 * (lane >> 2) + ((lane & 3) >> 1) - (a_par ? CO : CE);
    const int out_band = (lane & 3) >> 1;
    const int out_off = 4 * (lane >> 2) + 2 * (lane & 1);  // D fragment: outputs i0 + out_off, + 1 of band out_band

    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();

    double* in = buf0;
    int hin = h0;
    double* nxt = bufA;
    int hnx = hA;
#pragma unroll 1
    for (int j = 1; j <= K; ++j) {
        const int half = p.n[j], nprev = p.n[j - 1];
        const int in0 = s_lo[j - 1], in_cnt = s_hi[j - 1] - in0;
        const int cnt_e = (in_cnt + 1) >> 1, cnt_o = in_cnt >> 1, q0 = in0 >> 1;
        const int o0 = s_lo[j], o1 = s_hi[j];
        const int own0 = (chunk * p.tk) << (K - j), own1 = min(((chunk + 1) * p.tk) << (K - j), half);
        const int nbt = p.nb_top[j - 1], nbb = p.nb_bot[j - 1];
        double* __restrict__ hib = p.hi[j - 1] + (int64_t)b * p.hi_stride[j - 1];
        double* __restrict__ lob = p.lo + (int64_t)b * p.lo_stride;
        const bool last = j == K;
        const bool vec_st = out_band ? ((p.vec >> (j - 1)) & 1) : ((p.vec >> 15) & 1);
        const double* xe = in;
        const double* xo = in + hin + OFFO;
        double* nxe = nxt;
        double* nxo = nxt + hnx + OFFO;
        double* __restrict__ gout = out_band ? hib : lob;

        const int ntiles = (o1 - o0 + 31) >> 5;
        const int lo_all = max(nbt, o0), hi_all = min(half - nbb, o1);
        int t_lo, t_hi;
        {
            const int need0 = max(lo_all - o0, q0 + CO - o0);
            t_lo = need0 > 0 ? (need0 + 31) >> 5 : 0;
            const int lim_in = cnt_o - 28 - 2 * KS + CE + q0 - o0;
            t_hi = min((hi_all - o0) >> 5, lim_in >= 0 ? (lim_in >> 5) + 1 : 0);
            t_hi = max(min(t_hi, ntiles), 0);
            t_lo = min(t_lo, t_hi);
        }
        const double* band = a_par ? xo : xe;
        const int cnt_p = a_par ? cnt_o : cnt_e;
        auto generic_tile = [&](const int t) {
            const int i0 = o0 + 32 * t;
            const int rel0 = i0 + a_off - q0;
            double d0 = 0.0, d1 = 0.0;
            // samples clamped into the staged range: only outputs that the corner-block code below overwrites, or that
            // lie beyond o1, can see a clamped value
#pragma unroll
            for (int e = 0; e < KS; ++e) {
                const int rel = min(max(rel0 + 2 * e, 0), cnt_p - 1);
                dmma_m8n8k4(d0, d1, band[rel], bfrag[e]);
            }
            const int ia = i0 + out_off;
            if (out_band == 0 && !last) {
                if (ia < o1) nxe[(ia - o0) >> 1] = d0;
                if (ia + 1 < o1) nxo[(ia - o0) >> 1] = d1;
            } else {
                if (ia >= own0 && ia < own1 && ia >= nbt && ia < half - nbb) gout[ia] = d0;
                if (ia + 1 >= own0 && ia + 1 < own1 && ia + 1 >= nbt && ia + 1 < half - nbb) gout[ia + 1] = d1;
            }
        };
        for (int t = warp; t < t_lo; t += NW) generic_tile(t);
        for (int t = t_hi + warp; t < ntiles; t += NW) generic_tile(t);
        {
            const int tf = t_lo + warp;
            int ia = o0 + 32 * tf + out_off;
            const double* src = band + (o0 + 32 * tf + a_off - q0);
            double* de = nxe + ((ia - o0) >> 1);
            double* dod = nxo + ((ia - o0) >> 1);
            double* dgl = gout + ia;
            const bool to_smem = out_band == 0 && !last;
            for (int t = tf; t < t_hi; t += NW) {
                double v[KS];
#pragma unroll
                for (int e = 0; e < KS; ++e) v[e] = src[2 * e];
                double d0 = 0.0, d1 = 0.0;
#pragma unroll
                for (int e = 0; e < KS; ++e) dmma_m8n8k4(d0, d1, v[e], bfrag[e]);
                if (to_smem) {
                    *de = d0; *dod = d1;
                } else if (ia >= own0 && ia + 1 < own1) {
                    if (vec_st) {
                        *reinterpret_cast<double2*>(dgl) = make_double2(d0, d1);
                    } else {
                        dgl[0] = d0; dgl[1] = d1;
                    }
                } else if (ia >= own0 && ia < own1) {
                    dgl[0] = d0;
                }
                src += 32 * NW; de += 16 * NW; dod += 16 * NW; dgl += 32 * NW; ia += 32 * NW;
            }
        }
        __syncthreads();
        // ---- corner blocks: the dense orthogonalised boundary rows (the CTAs at the two ends of the row) -------
        if (o0 < nbt || o1 > half - nbb) {
            const int nt_ = max(min(o1, nbt) - o0, 0);
            const int b0 = max(o0, half - nbb), nb_ = max(o1 - b0, 0);
            for (int q = tid; q < 2 * (nt_ + nb_); q += NT) {
                const int bnd = q & 1, r = q >> 1;
                const int ii = r < nt_ ? o0 + r : b0 + (r - nt_);
                const bool top = ii < nbt;
                const int rr = top ? ii : nbt + (ii - (half - nbb));
                const int w = top ? p.w_left[j - 1] : p.w_right[j - 1];
                const int s0 = (top ? 0 : nprev - w) - in0;
                const double* __restrict__ blk = (top ? (bnd ? p.hi_left[j - 1] : p.lo_left[j - 1])
                                                      : (bnd ? p.hi_right[j - 1] : p.lo_right[j - 1])) + rr * w;
                double acc = 0.0;
                for (int c = 0; c < w; ++c) {
                    const int pos = s0 + c;
                    acc = fma(__ldg(blk + c), ((pos & 1) ? xo : xe)[pos >> 1], acc);
                }
                if (bnd == 0) {
                    if (!last) ((((ii - o0) & 1) ? nxo : nxe))[(ii - o0) >> 1] = acc;
                    else if (ii >= own0 && ii < own1) lob[ii] = acc;
                } else if (ii >= own0 && ii < own1) {
                    hib[ii] = acc;
                }
            }
            __syncthreads();
        }
        in = nxt; hin = hnx;
        if (nxt == bufA) { nxt = bufB; hnx = hB; } else { nxt = bufA; hnx = hA; }
    }
}

// Host: the polyphase analysis cascade; false = not applicable (caller falls back to the streaming kernel).
static bool launch_mat_fwd_dmma2(int L, int k, const int64_t* n, const int32_t* nbt, const int32_t* nbb, const int32_t* wl,
                                 const int32_t* wr, const double* const* blk_ptrs, const double* x, int64_t xs, int64_t batch,
                                 void* const* hi_out, const int64_t* hi_stride, double* lo_out, int64_t lo_stride,
                                 const Taps<double>& taps, cudaStream_t st, cudaError_t* err) {
    *err = cudaSuccess;
    if ((L & 1) || L < 2 || L > 16 || k < 1 || k > MATF_MAXK || batch > 65535) return false;
    if (n[0] >= (int64_t(1) << 30)) return false;
    MatFusedParams<double> p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.x_stride = xs; p.k = k;
    p.n[0] = (int)n[0];
    int vec = 0;
    if (!((uintptr_t)lo_out & 15) && !(lo_stride & 1)) vec |= 1 << 15;
    for (int j = 0; j < k; ++j) {
        if (n[j] & 1) return false;
        p.n[j + 1] = (int)(n[j] / 2);
        if (j + 1 < k && n[j + 1] != n[j] / 2) return false;
        p.hi[j] = (double*)hi_out[j]; p.hi_stride[j] = hi_stride[j];
        if (!((uintptr_t)hi_out[j] & 15) && !(hi_stride[j] & 1)) vec |= 1 << j;
        p.nb_top[j] = nbt[j]; p.nb_bot[j] = nbb[j]; p.w_left[j] = wl[j]; p.w_right[j] = wr[j];
        p.lo_left[j] = blk_ptrs[4 * j]; p.lo_right[j] = blk_ptrs[4 * j + 1];
        p.hi_left[j] = blk_ptrs[4 * j + 2]; p.hi_right[j] = blk_ptrs[4 * j + 3];
        if (nbt[j] + nbb[j] > p.n[j + 1]) return false;
    }
    p.vec = vec;
    p.lo = lo_out; p.lo_stride = lo_stride;
    for (int q = 0; q < L; ++q) { p.flo[q] = taps.lo[L - 1 - q]; p.fhi[q] = taps.hi[L - 1 - q]; }
    const int nk = p.n[k];
    int chunk0 = 2048;
    if (knob_is_set(K_MATF_CHUNK)) { const int v = (int)knob_val(K_MATF_CHUNK, 0); if (v >= 64 && v <= 16384) chunk0 = v; }
    if (n[0] <= 8192 && n[0] > chunk0 && k > 2) chunk0 = (int)n[0];   // deep cascades of short rows: one CTA per row
    int tk = chunk0 >> k;
    if (tk < 4) tk = 4;
    tk = (tk + 3) & ~3;
    if (tk > nk) tk = (nk + 3) & ~3;
    p.tk = tk;
    int cap0 = (tk << k) + ((L + 6) << k) + 64;
    if (cap0 > p.n[0] + 16) cap0 = p.n[0] + 16;
    cap0 = (cap0 + 31) & ~31;
    p.cap0 = cap0;
    const size_t smem = (size_t)((cap0 + 16 + 4) + (cap0 / 2 + 16 + 4) + (cap0 / 4 + 16 + 4)) * sizeof(double);
    if (smem > 200 * 1024) return false;
    const int nchunks = (nk + tk - 1) / tk;
    p.cpc = 1;
    dim3 grid((unsigned)nchunks, (unsigned)batch);
    const int nt = knob_val(K_MATF_NT, 128) == 256 ? 256 : 128;
#define WTB_MD2_LAUNCH(LL, NTT)                                                                        \
    {                                                                                                  \
        cudaError_t e = ensure_dyn_smem(mat_fwd_dmma2_kernel<LL, NTT>, 200 * 1024);                    \
        if (e != cudaSuccess) { *err = e; return true; }                                               \
        mat_fwd_dmma2_kernel<LL, NTT><<<grid, NTT, smem, st>>>(p);                                     \
    }
#define WTB_MD2(LL)                                                                                    \
    case LL:                                                                                           \
        if (nt == 128) WTB_MD2_LAUNCH(LL, 128) else WTB_MD2_LAUNCH(LL, 256)                            \
        break;
    switch (L) {
        WTB_MD2(2) WTB_MD2(4) WTB_MD2(6) WTB_MD2(8) WTB_MD2(10) WTB_MD2(12) WTB_MD2(14) WTB_MD2(16)
        default: return false;
    }
#undef WTB_MD2
#undef WTB_MD2_LAUNCH
    *err = cudaGetLastError();
    return true;
}

// ==========================================================================================
// MatrixWaverec on the FP64 tensor cores: the synthesis cascade (coarse to fine) of K levels in one launch.
//
// Reference: MatrixWaverec.__call__, src/ptwt/matmul_transform.py:664-761 (torch.sparse.mm(S_level, [lo; hi])).
// Away from the corner blocks every output sample is y[t] = sum_i rec_lo[t + L/2 - 1 - 2 i] lo[i] + rec_hi[..] hi[i].
// Eight consecutive outputs t0 .. t0 + 7 read one window of W = 2 floor(L/4) + 4 coefficients of each band, so a tile
// of 8 such groups is the dense product
//
//     D[8 groups x 8 samples] = A[8 x 2W] * B[2W x 8],   A[g][u] = c_{u & 1}[t0/2 + 4 g - C + (u >> 1)],
//                                                        B[u][s] = rec_{u & 1}[s + L/2 - 1 + 2 C - 2 (u >> 1)]
//
// with the DATA in the A operand and the FILTER in the B operand: the D fragment of lane q is then the output pair
// (t0 + 2 q, t0 + 2 q + 1), one fully coalesced 128-bit store per tile, and the A fragment of k-step e is one 64-bit
// shared load per lane which is bank-conflict free because the detail band is staged two doubles behind the
// approximation band.  W / 2 DMMAs + W / 2 loads + 1 store per 64 outputs (L = 12: 0.17 warp instructions per sample).
//
// The cascade around it is that of mat_inv_fused_kernel (matrix_fused.cuh): a CTA owns a chunk of the finest output,
// stages every detail range and the coarsest approximation range by cp.async (one commit group per level, so the
// coarse levels start while the fine details are still in flight), keeps every intermediate approximation in shared
// memory, and the CTAs at the two ends apply the dense corner rows by scalar code.
// ==========================================================================================
__device__ __forceinline__ void cp_async_wait_dyn(int pending) {
    switch (pending) {
        case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
        case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
        case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
        case 3: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
        case 4: asm volatile("cp.async.wait_group 4;" ::: "memory"); break;
        case 5: asm volatile("cp.async.wait_group 5;" ::: "memory"); break;
        case 6: asm volatile("cp.async.wait_group 6;" ::: "memory"); break;
        default: asm volatile("cp.async.wait_group 7;" ::: "memory"); break;
    }
}

template <int L, int NT>
__global__ void __launch_bounds__(NT) mat_inv_dmma_kernel(const __grid_constant__ MatInvFusedParams<double> p) {
    constexpr int H = L / 2;
    constexpr int C = H / 2;                      // the window of a group of 8 outputs starts at t0 / 2 - C
    constexpr int KS = C + 2;                     // k-steps: 2 coefficients x 2 bands each
    constexpr int W = 2 * KS;                     // coefficients of one band in the window
    constexpr int NW = NT / 32;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* bufA = reinterpret_cast<double*>(smem_raw);
    double* bufB = bufA + p.cap;
    double* shi = bufB + p.cap + 2;               // + 2 doubles: see the bank note above

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.y;
    const int K = p.k;
    if ((int64_t)blockIdx.x * p.chunk >= p.keep0) return;

    // level-j coefficients [s_ra[j], s_rb[j]) are needed (j >= 1); [s_ra[0], s_rb[0]) = samples this CTA writes
    __shared__ int s_ra[MATF_MAXK + 1], s_rb[MATF_MAXK + 1], s_hoff[MATF_MAXK + 1];
    if (tid == 0) {
        int ra = blockIdx.x * p.chunk, rb = min(ra + p.chunk, p.n[0]), ho = 0;
        s_ra[0] = ra; s_rb[0] = rb; s_hoff[0] = 0;
        for (int j = 1; j <= K; ++j) {
            const int nout = p.n[j - 1], N = nout / 2;
            int ia = (ra - H + 1) >> 1;                                 // ceil((a - L/2) / 2)
            int ib = (rb - 1 + H - 1) >> 1;                             // floor((b - 1 + L/2 - 1) / 2)
            if (ra < p.w_left[j - 1]) { ia = 0; ib = max(ib, p.nb_top[j - 1] - 1); }
            if (rb > nout - p.w_right[j - 1]) { ib = N - 1; ia = min(ia, N - p.nb_bot[j - 1]); }
            ra = max(ia, 0) & ~3;
            rb = min(ib + 1, N);
            ho += (rb - ra + 3) & ~3;
            s_ra[j] = ra; s_rb[j] = rb; s_hoff[j] = ho;
        }
    }
    __syncthreads();

    auto stage = [&](double* dst, const double* __restrict__ src, const int cnt, const bool vec) {
        if (vec) {
            const int nv = cnt >> 1;
            for (int q = tid; q < nv; q += NT) {
                const unsigned d = (unsigned)__cvta_generic_to_shared(dst + 2 * q);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src + 2 * q) : "memory");
            }
            if ((cnt & 1) && tid == 0) {
                const unsigned d = (unsigned)__cvta_generic_to_shared(dst + cnt - 1);
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(src + cnt - 1) : "memory");
            }
        } else {
            for (int q = tid; q < cnt; q += NT) {
                const unsigned d = (unsigned)__cvta_generic_to_shared(dst + q);
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(src + q) : "memory");
            }
        }
    };
    // commit group K - j holds what level j needs beyond the coarser levels (coarsest first)
    for (int j = K; j >= 1; --j) {
        if (j == K)
            stage(bufA, p.lo + (int64_t)b * p.lo_stride + s_ra[K], s_rb[K] - s_ra[K], (p.vec >> 15) & 1);
        stage(shi + s_hoff[j - 1], p.hi[j - 1] + (int64_t)b * p.hi_stride[j - 1] + s_ra[j], s_rb[j] - s_ra[j],
              (p.vec >> (j - 1)) & 1);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }

    // B fragment (the filter): lane holds B[k = lane % 4][n = s = lane / 4] of k-step e, u = 4 e + k
    double bfrag[KS];
    {
        const int s = lane >> 2, k = lane & 3;
#pragma unroll
        for (int e = 0; e < KS; ++e) {
            const int w = 2 * e + (k >> 1);
            const int kk = s + H - 1 + 2 * C - 2 * w;
            bfrag[e] = (kk >= 0 && kk < L) ? ((k & 1) ? p.rhi[kk] : p.rlo[kk]) : 0.0;
        }
    }
    // A fragment (the data): lane holds A[m = g = lane / 4][k = lane % 4]: band k & 1, coefficient 4 g + (k >> 1) + 2 e
    const int a_off = 4 * (lane >> 2) + ((lane & 3) >> 1) - C;
    const bool a_hi = lane & 1;
    const bool vec_y = (p.vec >> 14) & 1;

    double* cur = bufA;
    double* nxt = bufB;
#pragma unroll 1
    for (int j = K; j >= 1; --j) {
        const int nout = p.n[j - 1], N = nout / 2;
        const int a = s_ra[j - 1], bnd = s_rb[j - 1];
        const int c0 = s_ra[j], cnt = s_rb[j] - c0;
        const double* sl = cur;
        const double* sh = shi + s_hoff[j - 1];
        const int nbt = p.nb_top[j - 1], nbb = p.nb_bot[j - 1], wl = p.w_left[j - 1], wr = p.w_right[j - 1];
        double* __restrict__ yb = p.y + (int64_t)b * p.y_stride;
        const bool last = j == 1;
        const int lim = last ? min(bnd, p.keep0) : bnd;
        // outputs [a, s_top) and [s_bot, bnd) touch boundary coefficients or corner rows: scalar code below
        const int s_top = min(max(max(wl, 2 * nbt + H), a), bnd);
        const int s_bot = max(min(min(nout - wr, 2 * (N - nbb) - H), bnd), s_top);

        cp_async_wait_dyn(j - 1);
        __syncthreads();

        // ---- interior: tiles of 64 outputs, one warp per tile -------------------------------------------------------
        const int tl_first = (s_top - a) >> 6, tl_end = (s_bot - a + 63) >> 6;
        int f_lo, f_hi;
        {
            // tile t (t0 = a + 64 t) is fast when all 64 outputs are interior ones of this CTA and its whole window is staged
            const int need = max(s_top - a, 2 * (c0 + C) - a);
            f_lo = need > 0 ? (need + 63) >> 6 : 0;
            const int lim_in = 2 * (cnt + c0 + C - W - 28) - a;               // t0 - a <= lim_in
            f_hi = min((s_bot - a) >> 6, lim_in >= 0 ? (lim_in >> 6) + 1 : 0);
            f_lo = min(max(f_lo, tl_first), tl_end);
            f_hi = min(max(f_hi, f_lo), tl_end);
        }
        const double* band = a_hi ? sh : sl;
        auto generic_tile = [&](const int t) {
            const int t0 = a + 64 * t;
            const int rel0 = (t0 >> 1) + a_off - c0;
            double d0 = 0.0, d1 = 0.0;
            // coefficients clamped into the staged range: only outputs outside [s_top, s_bot) can see a clamped value
#pragma unroll
            for (int e = 0; e < KS; ++e) {
                const int rel = min(max(rel0 + 2 * e, 0), cnt - 1);
                dmma_m8n8k4(d0, d1, band[rel], bfrag[e]);
            }
            const int ta = t0 + 2 * lane;
            if (!last) {
                if (ta >= s_top && ta < s_bot) nxt[ta - a] = d0;
                if (ta + 1 >= s_top && ta + 1 < s_bot) nxt[ta + 1 - a] = d1;
            } else {
                if (ta >= s_top && ta < s_bot && ta < lim) yb[ta] = d0;
                if (ta + 1 >= s_top && ta + 1 < s_bot && ta + 1 < lim) yb[ta + 1] = d1;
            }
        };
        for (int t = tl_first + warp; t < f_lo; t += NW) generic_tile(t);
        for (int t = f_hi + warp; t < tl_end; t += NW) generic_tile(t);
        {
            const int tf = f_lo + warp;
            const double* src = band + (((a + 64 * tf) >> 1) + a_off - c0);
            double* dsm = nxt + 64 * tf + 2 * lane;
            double* dgl = yb + a + 64 * tf + 2 * lane;
            for (int t = tf; t < f_hi; t += NW) {
                double v[KS];
#pragma unroll
                for (int e = 0; e < KS; ++e) v[e] = src[2 * e];
                double d0 = 0.0, d1 = 0.0;
#pragma unroll
                for (int e = 0; e < KS; ++e) dmma_m8n8k4(d0, d1, v[e], bfrag[e]);
                if (!last) {
                    *reinterpret_cast<double2*>(dsm) = make_double2(d0, d1);
                } else if (vec_y) {
                    *reinterpret_cast<double2*>(dgl) = make_double2(d0, d1);
                } else {
                    dgl[0] = d0; dgl[1] = d1;
                }
                src += 32 * NW; dsm += 64 * NW; dgl += 64 * NW;
            }
        }
        // ---- the two ends of the row: clipped windows and the dense corner rows -------------------------------------
        {
            const int ntop = s_top - a, nbot = bnd - s_bot;
            for (int q = tid; q < ntop + nbot; q += NT) {
                const int t = q < ntop ? a + q : s_bot + (q - ntop);
                double acc = 0.0;
                int i0 = (t - H + 1) >> 1, i1 = (t + H - 1) >> 1;
                i0 = max(i0, nbt);
                i1 = min(i1, N - nbb - 1);
                for (int i = i0; i <= i1; ++i) {
                    const int kk = t + H - 1 - 2 * i;
                    acc = fma(p.rlo[kk], sl[i - c0], acc);
                    acc = fma(p.rhi[kk], sh[i - c0], acc);
                }
                if (t < wl) {
                    // top boundary rows only: the bottom rows' entries in the left corner are the dropped cross-corner
                    // round-off (same host-side criterion as the analysis kernels)
                    for (int r = 0; r < nbt; ++r) {
                        acc = fma(__ldg(p.lo_left[j - 1] + r * wl + t), sl[r - c0], acc);
                        acc = fma(__ldg(p.hi_left[j - 1] + r * wl + t), sh[r - c0], acc);
                    }
                }
                if (t >= nout - wr) {
                    const int c = t - (nout - wr);
                    for (int r = nbt; r < nbt + nbb; ++r) {
                        const int i = N - nbb + (r - nbt);
                        acc = fma(__ldg(p.lo_right[j - 1] + r * wr + c), sl[i - c0], acc);
                        acc = fma(__ldg(p.hi_right[j - 1] + r * wr + c), sh[i - c0], acc);
                    }
                }
                if (!last) nxt[t - a] = acc;
                else if (t < lim) yb[t] = acc;
            }
        }
        double* tswap = cur; cur = nxt; nxt = tswap;
    }
}

// ------------------------------------------------------------------------------------------
// The same cascade, streaming ROWS: a CTA keeps its chunk index and walks p.rows batch rows.  The coefficient ranges
// and tile ranges depend on the chunk only, so they are computed once; the next row's details and coarsest
// approximation arrive by TMA bulk copies (cp.async.bulk, one mbarrier per level and buffer set) while the current row
// is synthesised, which removes the per-thread staging loops and the per-level range arithmetic of the kernel above.
// Needs 16-byte aligned rows and even band lengths (bulk copies move multiples of 16 bytes).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void md_mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void md_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void md_mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "MD_WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra MD_DONE;\n\t"
        "bra MD_WAIT_LOOP;\n\t"
        "MD_DONE:\n\t"
        "}" ::"r"((uint32_t)__cvta_generic_to_shared(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void md_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     (uint32_t)__cvta_generic_to_shared(dst)),
                 "l"(src), "r"(bytes), "r"((uint32_t)__cvta_generic_to_shared(bar))
                 : "memory");
}

enum { MDI_A = 0, MDI_BND, MDI_C0, MDI_CNT, MDI_STOP, MDI_SBOT, MDI_TL0, MDI_TL1, MDI_FLO, MDI_FHI, MDI_N };

template <int L, int NT>
__global__ void __launch_bounds__(NT) mat_inv_dmma_rows_kernel(const __grid_constant__ MatInvFusedParams<double> p) {
    constexpr int H = L / 2;
    constexpr int C = H / 2;
    constexpr int KS = C + 2;
    constexpr int W = 2 * KS;
    constexpr int NW = NT / 32;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* bufA = reinterpret_cast<double*>(smem_raw);
    double* bufB = bufA + p.cap;
    double* lost = bufB + p.cap;                  // [2][cap_lo]  coarsest approximation of the current / next row
    double* hist = lost + 2 * p.cap_lo + 2;       // [2][hi_cap]  details, two doubles behind (bank note above)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = p.k;
    if ((int64_t)blockIdx.x * p.chunk >= p.keep0) return;
    const int row0 = blockIdx.y * p.rows;
    const int nrows = min(p.rows, p.batch - row0);

    __shared__ int s_info[MATF_MAXK][MDI_N];
    __shared__ int s_hoff[MATF_MAXK + 1];
    __shared__ __align__(8) uint64_t s_bar[2][MATF_MAXK];
    if (tid == 0) {
        int ra = blockIdx.x * p.chunk, rb = min(ra + p.chunk, p.n[0]), ho = 0;
        s_hoff[0] = 0;
        for (int j = 1; j <= K; ++j) {
            const int nout = p.n[j - 1], N = nout / 2;
            const int nbt = p.nb_top[j - 1], nbb = p.nb_bot[j - 1], wl = p.w_left[j - 1], wr = p.w_right[j - 1];
            const int a = ra, bnd = rb;
            int ia = (a - H + 1) >> 1;
            int ib = (bnd - 1 + H - 1) >> 1;
            if (a < wl) { ia = 0; ib = max(ib, nbt - 1); }
            if (bnd > nout - wr) { ib = N - 1; ia = min(ia, N - nbb); }
            ra = max(ia, 0) & ~3;
            rb = min((ib + 2) & ~1, N);                                 // even count: bulk copies move 16-byte units
            const int c0 = ra, cnt = rb - ra;
            ho += (cnt + 3) & ~3;
            s_hoff[j] = ho;
            const int s_top = min(max(max(wl, 2 * nbt + H), a), bnd);
            const int s_bot = max(min(min(nout - wr, 2 * (N - nbb) - H), bnd), s_top);
            const int tl_first = (s_top - a) >> 6, tl_end = (s_bot - a + 63) >> 6;
            const int need = max(s_top - a, 2 * (c0 + C) - a);
            int f_lo = need > 0 ? (need + 63) >> 6 : 0;
            const int lim_in = 2 * (cnt + c0 + C - W - 28) - a;
            int f_hi = min((s_bot - a) >> 6, lim_in >= 0 ? (lim_in >> 6) + 1 : 0);
            f_lo = min(max(f_lo, tl_first), tl_end);
            f_hi = min(max(f_hi, f_lo), tl_end);
            int* o = s_info[j - 1];
            o[MDI_A] = a; o[MDI_BND] = bnd; o[MDI_C0] = c0; o[MDI_CNT] = cnt; o[MDI_STOP] = s_top; o[MDI_SBOT] = s_bot;
            o[MDI_TL0] = tl_first; o[MDI_TL1] = tl_end; o[MDI_FLO] = f_lo; o[MDI_FHI] = f_hi;
        }
        for (int q = 0; q < 2 * MATF_MAXK; ++q) md_mbar_init(&s_bar[0][0] + q, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto issue = [&](const int row, const int set) {                  // one thread
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic reads of this set precede the refill
        for (int j = K; j >= 1; --j) {
            const int c0 = s_info[j - 1][MDI_C0], cnt = s_info[j - 1][MDI_CNT];
            uint64_t* bar = &s_bar[set][j - 1];
            md_mbar_expect_tx(bar, (uint32_t)cnt * 8u * (j == K ? 2u : 1u));
            if (j == K) md_bulk_g2s(lost + set * p.cap_lo, p.lo + (int64_t)row * p.lo_stride + c0, (uint32_t)cnt * 8u, bar);
            md_bulk_g2s(hist + set * p.hi_cap + s_hoff[j - 1], p.hi[j - 1] + (int64_t)row * p.hi_stride[j - 1] + c0,
                        (uint32_t)cnt * 8u, bar);
        }
    };
    if (tid == 0) issue(row0, 0);

    double bfrag[KS];
    {
        const int s = lane >> 2, k = lane & 3;
#pragma unroll
        for (int e = 0; e < KS; ++e) {
            const int w = 2 * e + (k >> 1);
            const int kk = s + H - 1 + 2 * C - 2 * w;
            bfrag[e] = (kk >= 0 && kk < L) ? ((k & 1) ? p.rhi[kk] : p.rlo[kk]) : 0.0;
        }
    }
    const int a_off = 4 * (lane >> 2) + ((lane & 3) >> 1) - C;
    const bool a_hi = lane & 1;
    const bool vec_y = (p.vec >> 14) & 1;

#pragma unroll 1
    for (int r = 0; r < nrows; ++r) {
        const int set = r & 1;
        const uint32_t par = (r >> 1) & 1;
        if (tid == 0 && r + 1 < nrows) issue(row0 + r + 1, set ^ 1);
        double* __restrict__ yb = p.y + (int64_t)(row0 + r) * p.y_stride;
        const double* cur = lost + set * p.cap_lo;
        double* nxt = bufA;
#pragma unroll 1
        for (int j = K; j >= 1; --j) {
            const int* o = s_info[j - 1];
            const int a = o[MDI_A], bnd = o[MDI_BND], c0 = o[MDI_C0], cnt = o[MDI_CNT];
            const int s_top = o[MDI_STOP], s_bot = o[MDI_SBOT];
            const int tl_first = o[MDI_TL0], tl_end = o[MDI_TL1], f_lo = o[MDI_FLO], f_hi = o[MDI_FHI];
            const double* sl = cur;
            const double* sh = hist + set * p.hi_cap + s_hoff[j - 1];
            const bool last = j == 1;
            const int lim = last ? min(bnd, p.keep0) : bnd;

            md_mbar_wait(&s_bar[set][j - 1], par);
            __syncthreads();                       // the coarser level's samples are complete

            const double* band = a_hi ? sh : sl;
            auto generic_tile = [&](const int t) {
                const int t0 = a + 64 * t;
                const int rel0 = (t0 >> 1) + a_off - c0;
                double d0 = 0.0, d1 = 0.0;
#pragma unroll
                for (int e = 0; e < KS; ++e) {
                    const int rel = min(max(rel0 + 2 * e, 0), cnt - 1);
                    dmma_m8n8k4(d0, d1, band[rel], bfrag[e]);
                }
                const int ta = t0 + 2 * lane;
                if (!last) {
                    if (ta >= s_top && ta < s_bot) nxt[ta - a] = d0;
                    if (ta + 1 >= s_top && ta + 1 < s_bot) nxt[ta + 1 - a] = d1;
                } else {
                    if (ta >= s_top && ta < s_bot && ta < lim) yb[ta] = d0;
                    if (ta + 1 >= s_top && ta + 1 < s_bot && ta + 1 < lim) yb[ta + 1] = d1;
                }
            };
            for (int t = tl_first + warp; t < f_lo; t += NW) generic_tile(t);
            for (int t = f_hi + warp; t < tl_end; t += NW) generic_tile(t);
            {
                const int tf = f_lo + warp;
                const double* src = band + (((a + 64 * tf) >> 1) + a_off - c0);
                if (!last) {
                    double* dsm = nxt + 64 * tf + 2 * lane;
                    for (int t = tf; t < f_hi; t += NW) {
                        double v[KS];
#pragma unroll
                        for (int e = 0; e < KS; ++e) v[e] = src[2 * e];
                        double d0 = 0.0, d1 = 0.0;
#pragma unroll
                        for (int e = 0; e < KS; ++e) dmma_m8n8k4(d0, d1, v[e], bfrag[e]);
                        *reinterpret_cast<double2*>(dsm) = make_double2(d0, d1);
                        src += 32 * NW; dsm += 64 * NW;
                    }
                } else {
                    double* dgl = yb + a + 64 * tf + 2 * lane;
                    for (int t = tf; t < f_hi; t += NW) {
                        double v[KS];
#pragma unroll
                        for (int e = 0; e < KS; ++e) v[e] = src[2 * e];
                        double d0 = 0.0, d1 = 0.0;
#pragma unroll
                        for (int e = 0; e < KS; ++e) dmma_m8n8k4(d0, d1, v[e], bfrag[e]);
                        if (vec_y) {
                            *reinterpret_cast<double2*>(dgl) = make_double2(d0, d1);
                        } else {
                            dgl[0] = d0; dgl[1] = d1;
                        }
                        src += 32 * NW; dgl += 64 * NW;
                    }
                }
            }
            const int ntop = s_top - a, nbot = bnd - s_bot;
            if (ntop + nbot > 0) {
                const int nout = p.n[j - 1], N = nout / 2;
                const int nbt = p.nb_top[j - 1], nbb = p.nb_bot[j - 1], wl = p.w_left[j - 1], wr = p.w_right[j - 1];
                for (int q = tid; q < ntop + nbot; q += NT) {
                    const int t = q < ntop ? a + q : s_bot + (q - ntop);
                    double acc = 0.0;
                    int i0 = (t - H + 1) >> 1, i1 = (t + H - 1) >> 1;
                    i0 = max(i0, nbt);
                    i1 = min(i1, N - nbb - 1);
                    for (int i = i0; i <= i1; ++i) {
                        const int kk = t + H - 1 - 2 * i;
                        acc = fma(p.rlo[kk], sl[i - c0], acc);
                        acc = fma(p.rhi[kk], sh[i - c0], acc);
                    }
                    if (t < wl) {
                        for (int rr = 0; rr < nbt; ++rr) {
                            acc = fma(__ldg(p.lo_left[j - 1] + rr * wl + t), sl[rr - c0], acc);
                            acc = fma(__ldg(p.hi_left[j - 1] + rr * wl + t), sh[rr - c0], acc);
                        }
                    }
                    if (t >= nout - wr) {
                        const int c = t - (nout - wr);
                        for (int rr = nbt; rr < nbt + nbb; ++rr) {
                            const int i = N - nbb + (rr - nbt);
                            acc = fma(__ldg(p.lo_right[j - 1] + rr * wr + c), sl[i - c0], acc);
                            acc = fma(__ldg(p.hi_right[j - 1] + rr * wr + c), sh[i - c0], acc);
                        }
                    }
                    if (!last) nxt[t - a] = acc;
                    else if (t < lim) yb[t] = acc;
                }
            }
            cur = nxt;
            nxt = (nxt == bufA) ? bufB : bufA;
        }
        __syncthreads();                           // this row's buffers are free: the next refill may start
    }
}

// Host: one fused synthesis group on the FP64 tensor cores.  Arrays are indexed by fused level j-1 (0 = finest).
static bool launch_mat_inv_dmma(int L, int k, const int64_t* n, int64_t keep0, const int32_t* nbt, const int32_t* nbb,
                                const int32_t* wl, const int32_t* wr, const double* const* blk_ptrs /* 4 per level */,
                                const double* lo, int64_t lo_stride, const void* const* hi_in, const int64_t* hi_stride,
                                int64_t batch, double* y, int64_t y_stride, const double* rlo, const double* rhi,
                                cudaStream_t st, cudaError_t* err) {
    *err = cudaSuccess;
    if ((L & 1) || L < 2 || L > 16 || k < 1 || k > MATF_MAXK || batch > 65535) return false;
    if (n[0] >= (int64_t(1) << 30)) return false;
    MatInvFusedParams<double> p;
    memset(&p, 0, sizeof(p));
    p.lo = lo; p.lo_stride = lo_stride; p.y = y; p.y_stride = y_stride; p.k = k;
    p.keep0 = (int)keep0;
    int vec = 0;
    if (!((uintptr_t)lo & 15) && !(lo_stride & 1)) vec |= 1 << 15;
    if (!((uintptr_t)y & 15) && !(y_stride & 1)) vec |= 1 << 14;
    for (int j = 0; j < k; ++j) {
        if (n[j] & 1) return false;
        if (j + 1 < k && n[j + 1] != n[j] / 2) return false;       // no trimming inside a group
        p.n[j] = (int)n[j];
        p.hi[j] = (const double*)hi_in[j]; p.hi_stride[j] = hi_stride[j];
        if (!((uintptr_t)hi_in[j] & 15) && !(hi_stride[j] & 1)) vec |= 1 << j;
        p.nb_top[j] = nbt[j]; p.nb_bot[j] = nbb[j]; p.w_left[j] = wl[j]; p.w_right[j] = wr[j];
        p.lo_left[j] = blk_ptrs[4 * j]; p.lo_right[j] = blk_ptrs[4 * j + 1];
        p.hi_left[j] = blk_ptrs[4 * j + 2]; p.hi_right[j] = blk_ptrs[4 * j + 3];
        if (nbt[j] + nbb[j] > n[j] / 2) return false;
    }
    p.vec = vec;
    for (int q = 0; q < L; ++q) { p.rlo[q] = rlo[q]; p.rhi[q] = rhi[q]; }
    int chunk = 2048;
    if (knob_is_set(K_MATI_CHUNK)) { const int v = (int)knob_val(K_MATI_CHUNK, 0); if (v >= 64 && v <= 16384) chunk = v; }
    if (!knob_is_set(K_MATI_CHUNK)) {
        // short rows: smaller chunks until the launch has MATI_MINCTAS CTAs
        const int64_t min_ctas = knob_val(K_MATI_MINCTAS, 0);
        while (chunk > 256 && ((p.n[0] + chunk - 1) / chunk) * batch < min_ctas) chunk /= 2;
    }
    if (chunk > p.n[0] && p.n[0] <= 8192) chunk = p.n[0];
    chunk = (chunk + 63) / 64 * 64;
    if (chunk > p.n[0]) chunk = (p.n[0] + 63) / 64 * 64;
    p.chunk = chunk;
    // per level the range grows by at most L/2 + 4 coefficients (halo + alignment) + the corner rows
    int cap = 0, hcap = 0, len = chunk;
    for (int j = 0; j < k; ++j) {
        len = len / 2 + L / 2 + 8 + nbt[j] + nbb[j] + std::max(wl[j], wr[j]);
        if (len > p.n[j] / 2 + 4) len = p.n[j] / 2 + 4;
        len = (len + 3) & ~3;
        cap = std::max(cap, len);
        hcap += len;
    }
    p.cap = cap; p.hi_cap = hcap;
    const int nt = knob_val(K_MATI_NT, 128) == 256 ? 256 : 128;
    const unsigned nchunks = (unsigned)((keep0 + chunk - 1) / chunk);
    // row-streaming kernel (TMA bulk staging): every source row 16-byte aligned, every band length even
    bool rows_ok = (vec & (1 << 15)) != 0;
    for (int j = 0; j < k; ++j) rows_ok = rows_ok && ((vec >> j) & 1) && !(n[j] & 3);
    // WTB200_MATI_ROWS: > 0 = upper bound (lowered until two full waves of CTAs remain), < 0 = exactly that many,
    // 0 = the chunk-per-CTA kernel
    int rows = (int)knob_val(K_MATI_ROWS, 0);
    const bool forced = rows < 0;
    if (forced) rows = -rows;
    if (rows > 64) rows = 64;
    if (!forced)
        while (rows > 1 && (int64_t)nchunks * ((batch + rows - 1) / rows) < 8 * sm_count()) rows /= 2;
    p.rows = rows; p.batch = (int)batch; p.cap_lo = len;           // len = capacity of the coarsest range
    const size_t smem_rows = (size_t)(2 * cap + 2 * len + 2 * hcap + 4) * sizeof(double);
    if (rows_ok && rows >= 1 && smem_rows <= 200 * 1024 && batch < (int64_t(1) << 31)) {
        dim3 grid(nchunks, (unsigned)((batch + rows - 1) / rows));
        if (grid.y <= 65535) {
#define WTB_MIR_LAUNCH(LL, NTT)                                                                        \
    {                                                                                                  \
        cudaError_t e = ensure_dyn_smem(mat_inv_dmma_rows_kernel<LL, NTT>, 200 * 1024);                \
        if (e != cudaSuccess) { *err = e; return true; }                                               \
        mat_inv_dmma_rows_kernel<LL, NTT><<<grid, NTT, smem_rows, st>>>(p);                            \
    }
#define WTB_MIR(LL)                                                                                    \
    case LL:                                                                                           \
        if (nt == 128) WTB_MIR_LAUNCH(LL, 128) else WTB_MIR_LAUNCH(LL, 256)                            \
        break;
            switch (L) {
                WTB_MIR(2) WTB_MIR(4) WTB_MIR(6) WTB_MIR(8) WTB_MIR(10) WTB_MIR(12) WTB_MIR(14) WTB_MIR(16)
                default: return false;
            }
#undef WTB_MIR
#undef WTB_MIR_LAUNCH
            *err = cudaGetLastError();
            return true;
        }
    }
    const size_t smem = (size_t)(2 * cap + hcap + 4) * sizeof(double);
    if (smem > 200 * 1024) return false;
    dim3 grid(nchunks, (unsigned)batch);
#define WTB_MID_LAUNCH(LL, NTT)                                                                        \
    {                                                                                                  \
        cudaError_t e = ensure_dyn_smem(mat_inv_dmma_kernel<LL, NTT>, 200 * 1024);                     \
        if (e != cudaSuccess) { *err = e; return true; }                                               \
        mat_inv_dmma_kernel<LL, NTT><<<grid, NTT, smem, st>>>(p);                                      \
    }
#define WTB_MID(LL)                                                                                    \
    case LL:                                                                                           \
        if (nt == 128) WTB_MID_LAUNCH(LL, 128) else WTB_MID_LAUNCH(LL, 256)                            \
        break;
    switch (L) {
        WTB_MID(2) WTB_MID(4) WTB_MID(6) WTB_MID(8) WTB_MID(10) WTB_MID(12) WTB_MID(14) WTB_MID(16)
        default: return false;
    }
#undef WTB_MID
#undef WTB_MID_LAUNCH
    *err = cudaGetLastError();
    return true;
}

}  // namespace wtb
