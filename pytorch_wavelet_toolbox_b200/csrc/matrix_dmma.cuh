// matrix_dmma.cuh -- the boundary-filter matrix FWT (float64) on the FP64 TENSOR CORES.
//
// north_star: "tensor cores are used only for the MatrixWavedec path where the boundary-filter sparse matmul is
// reformulated as a banded dense contraction".  The level operator A_n of the reference
// (torch.sparse.mm(A_level, .), src/ptwt/matmul_transform.py:409-425) is block-Toeplitz away from its corner blocks:
// every output pair (lo[i], hi[i]) is the same L-tap window sliding by two samples, and the synthesis operator has
// the same structure.  So a tile of consecutive outputs is a small dense product of a window of the input (A operand)
// and a matrix of filter taps (B operand, registers), evaluated with mma.sync.aligned.m8n8k4.f64 (DMMA, the FP64
// tensor-core instruction of sm_90; wgmma has no f64 kind).  Part of the filter matrix is structural zeros -- the
// price of the dense form.
//
// Two kernels, each taking a group of levels through shared memory in one launch, so that only the details and the
// last approximation of a group (analysis) or its finest output (synthesis) reach HBM:
//   mat_fwd_dmma2_kernel  MatrixWavedec, the polyphase analysis cascade
//   mat_inv_dmma_kernel   MatrixWaverec, the synthesis cascade
// The corner blocks (dense orthogonalised boundary rows) are applied by scalar code in the CTAs at the two ends of a
// row.
#pragma once

#include "matrix_fused.cuh"

namespace wtb {

__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, const double a, const double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d0), "+d"(d1)
                 : "d"(a), "d"(b));
}

// ==========================================================================================
// MatrixWavedec on the FP64 tensor cores: the analysis cascade of K levels in one launch, laid out like the synthesis
// kernel below: one chunk per CTA, every level input kept as two POLYPHASE arrays
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

// Host: the polyphase analysis cascade; false = not applicable (the caller runs mat_fwd_fused_kernel or the per-level
// kernels instead).
static bool launch_mat_fwd_dmma2(int L, int k, const int64_t* n, const int32_t* nbt, const int32_t* nbb, const int32_t* wl,
                                 const int32_t* wr, const double* const* blk_ptrs, const double* x, int64_t xs, int64_t batch,
                                 void* const* hi_out, const int64_t* hi_stride, double* lo_out, int64_t lo_stride,
                                 const Taps<double>& taps, cudaStream_t st, cudaError_t* err) {
    *err = cudaSuccess;
    if ((L & 1) || L < 2 || L > 16 || k < 1 || k > MATF_MAXK || batch > 65535) return false;
    if (n[0] >= (int64_t(1) << 30)) return false;
    MatFusedParams<double> p;
    if (!fill_mat_fused_levels(p, L, k, n, nbt, nbb, wl, wr, blk_ptrs, x, xs, hi_out, hi_stride, lo_out, lo_stride, taps))
        return false;
    int vec = 0;
    if (!((uintptr_t)lo_out & 15) && !(lo_stride & 1)) vec |= 1 << 15;
    for (int j = 0; j < k; ++j)
        if (!((uintptr_t)hi_out[j] & 15) && !(hi_stride[j] & 1)) vec |= 1 << j;
    p.vec = vec;
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
// The cascade around it: a CTA owns a chunk of the finest output, stages every detail range and the coarsest
// approximation range by cp.async (one commit group per level, so the coarse levels start while the fine details are
// still in flight), keeps every intermediate approximation in shared memory, and the CTAs at the two ends apply the
// dense corner rows by scalar code.
// ==========================================================================================
template <typename T>
struct MatInvFusedParams {
    const T* lo;                 // approximation entering the coarsest fused level, [batch, n[K-1]/2]
    int64_t lo_stride;
    const T* hi[MATF_MAXK];      // hi[j-1]: detail of fused level j (j = 1 finest), [batch, n[j-1]/2]
    int64_t hi_stride[MATF_MAXK];
    T* y;                        // [batch, keep0]
    int64_t y_stride;
    int k;
    int n[MATF_MAXK];            // n[j-1] = operator size of fused level j (its output length before trimming)
    int keep0;                   // samples of the finest output that are stored (n[0] or n[0] - 1)
    int nb_top[MATF_MAXK], nb_bot[MATF_MAXK], w_left[MATF_MAXK], w_right[MATF_MAXK];
    const T* lo_left[MATF_MAXK];
    const T* lo_right[MATF_MAXK];
    const T* hi_left[MATF_MAXK];
    const T* hi_right[MATF_MAXK];
    int chunk;                   // finest-level samples per CTA (multiple of 64)
    int cap;                     // capacity of one approximation buffer
    int hi_cap;                  // capacity of the detail staging area
    T rlo[16], rhi[16];          // rec_lo / rec_hi, un-flipped
    int vec;                     // bit j-1 = hi[j-1] rows 16-byte aligned, bit 14 = y, bit 15 = lo
};

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
    const size_t smem = (size_t)(2 * cap + hcap + 4) * sizeof(double);
    if (smem > 200 * 1024) return false;
    dim3 grid((unsigned)((keep0 + chunk - 1) / chunk), (unsigned)batch);
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
