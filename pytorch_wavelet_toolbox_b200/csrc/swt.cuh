// swt.cuh -- the stationary (undecimated, "a trous") wavelet transform, ptwt.swt / ptwt.iswt.
//
// The reference runs one level as  _circular_pad -> conv1d(dilation 2^(j-1), 2 output channels) -> split
// (src/ptwt/stationary_transform.py:96-106) and the inverse as  stack -> _circular_pad -> conv_transpose1d ->
// mean  (:139-151), so every intermediate approximation makes a round trip through memory plus a padded copy.
// Here a group of levels runs in ONE launch with the intermediate approximations in shared memory: analysis
// reads the group's input once and writes only the details and the group's last approximation; synthesis
// reads the group's input approximation and details and writes only its finest reconstruction.
//
// Closed form of one level j, dilation d = 2^(j-1), hl = L/2 - 1, indices mod n (the periodic extension):
//   analysis   c_k[i] = sum_m f_k[m] a[i + d (m - hl)]          swt: f_k = dec_k[::-1]; adjoint of iswt: 0.5 rec_k
//   synthesis  y[i]   = sum_m g_lo[m] a[i + d (hl - m)] + g_hi[m] c[i + d (hl - m)]
//                                                               iswt: g = 0.5 rec; adjoint of swt: g = dec[::-1]
// The two forms are each other's adjoint, so the same kernels serve the backward passes.
//
// Tiling.  When D = 2^t divides both n and the group's first dilation, the signal seen as M = n / D rows of D
// samples (sample s = row * D + column) splits into D independent periodic columns, and every level of the
// group is a dilated stencil along the rows.  A CTA holds a tile of R consecutive columns:
//   * "full" tiles hold all M rows: no halo, row indices wrap inside the tile (short signals, deep levels);
//   * "halo" tiles own C rows and stage (L-1) * d0 * (2^K - 1) more rows around them, wrapped periodically at
//     the signal ends; each level shrinks the valid range by its own reach (long signals, shallow levels).
// With D = R the tile is a contiguous chunk of the signal.  Levels whose pad the reference wraps in several
// non-periodic rounds (_circular_pad with a pad longer than n) run one per launch through a host-built table of
// source indices (swt_level_*_kernel), as do levels whose halo would not fit a tile.
//
// 2-D (swt2, one axis of one level per launch).  The pass along the contiguous axis is the 1-D case on rows of W
// samples.  The pass along the other axis treats each dense H x W plane as ONE periodic signal of n = H W samples at
// dilation b = d W: a shift by d W modulo H W moves d rows modulo H and keeps the column, so the signal seen as rows
// of D = gcd(n, b) = W gcd(H, d) samples splits into independent periodic columns exactly as above.  D need not be a
// power of two then; a tile's R columns are a power of two that divides it.  That pass filters the two bands of the
// contiguous-axis pass (lo_W, hi_W) in one launch: items [batch, 2 batch) of the launch are the second band set.
#pragma once

#include <numeric>

#include "common.cuh"

namespace wtb {

constexpr int SWT_THREADS = 512;
constexpr int SWT_MAXK = 32;                       // levels per fused launch
constexpr int SWT_FWD_BUF_BYTES = 48 * 1024;       // per tile buffer: analysis stages 2, synthesis 3
constexpr int SWT_INV_BUF_BYTES = 32 * 1024;
// outputs per thread along the rows in the unrolled path (float64: 2, so that L = 16 needs no spills)
template <typename T>
constexpr int swt_q() { return sizeof(T) == 8 ? 2 : 4; }

template <typename T>
struct SwtTileParams {
    const T* a;                // group input approximation [batch, n]
    int64_t a_bs;
    T* out;                    // group output approximation (analysis) / reconstruction (synthesis)
    int64_t out_bs;
    T* det[SWT_MAXK];          // detail of group level k (k = 0 finest), batch stride det_bs
    int64_t det_bs;
    int64_t batch;
    // second band set (sets == 2, K == 1 only): items [batch, 2 batch) read a2 and write out2 / det2
    const T* a2;
    T* out2;
    T* det2;
    int64_t a2_bs, out2_bs, det2_bs;
    int sets;
    int64_t D, M;              // the signal as M rows of D samples
    int64_t d0;                // dilation of level k = 0 in rows; level k has d0 << k
    int64_t C;                 // rows a CTA owns; C == M: whole columns, no halo
    int K, R, lgR, L;
    T f0[WT_MAX_FILT_LEN];     // analysis: f_lo; synthesis: g_lo
    T f1[WT_MAX_FILT_LEN];     // analysis: f_hi; synthesis: g_hi
};

// Tile geometry shared by both directions.  hl_reach / hr_reach: rows one level of dilation 1 reads to the
// left / right of its output.
struct SwtTile {
    int64_t i0, c0;            // first owned row, first column
    int HLr, rows, own_hi;     // left halo rows, staged rows, owned rows end (tile-local)
    bool full;
};

template <typename T>
__device__ __forceinline__ SwtTile swt_tile(const SwtTileParams<T>& p, int hl_reach, int hr_reach) {
    SwtTile t;
    t.full = p.C == p.M;
    const int64_t ntile = t.full ? 1 : (p.M + p.C - 1) / p.C;
    t.i0 = (blockIdx.x % ntile) * p.C;
    t.c0 = (int64_t)(blockIdx.x / ntile) << p.lgR;
    const int64_t span = ((int64_t(1) << p.K) - 1) * p.d0;
    t.HLr = t.full ? 0 : (int)(span * hl_reach);
    t.rows = t.full ? (int)p.M : (int)(p.C + span * (hl_reach + hr_reach));
    t.own_hi = t.HLr + (int)min(p.C, p.M - t.i0);
    return t;
}

// Stage rows [r_lo, r_hi) of a [batch, n] band into a tile buffer (tile row r <-> signal row i0 - HLr + r).
template <typename T>
__device__ __forceinline__ void swt_stage(T* buf, const T* src, const SwtTileParams<T>& p, const SwtTile& t,
                                          int r_lo, int r_hi) {
    const int lo = r_lo << p.lgR, hi = r_hi << p.lgR;
    for (int u = lo + threadIdx.x; u < hi; u += SWT_THREADS) {
        int64_t g = t.i0 - t.HLr + (u >> p.lgR);
        if (g < 0) g += p.M;                 // halo tiles exist only when the halo is shorter than the signal
        else if (g >= p.M) g -= p.M;
        buf[u] = src[g * p.D + t.c0 + (u & (p.R - 1))];
    }
}

// Tile row that holds row r: a full tile wraps mod M, a halo tile needs no wrapping (the halo covers the reach).
__device__ __forceinline__ int swt_wrap(int64_t r, int64_t M, bool full) {
    if (full) {
        r %= M;
        if (r < 0) r += M;
    }
    return (int)r;
}

// The same for |r - [0, M)| < M (the unrolled paths only run where the reach is shorter than M).
__device__ __forceinline__ int swt_wrap1(int r, int M, bool full) {
    if (full) {
        if (r < 0) r += M;
        else if (r >= M) r -= M;
    }
    return r;
}

// Analysis: levels k = 0..K-1 of one tile; A holds the staged input.
template <typename T, int LT>
__global__ void __launch_bounds__(SWT_THREADS, 1) swt_fwd_kernel(const __grid_constant__ SwtTileParams<T> p) {
    constexpr int SWT_Q = swt_q<T>();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int L = LT > 0 ? LT : p.L;
    const int hl = L / 2 - 1;
    const SwtTile t = swt_tile(p, hl, L / 2);
    const int cnt = t.rows << p.lgR;
    for (int64_t bb = blockIdx.y; bb < p.batch * p.sets; bb += gridDim.y) {
        const bool s2 = bb >= p.batch;
        const int64_t b = s2 ? bb - p.batch : bb;
        T* A = reinterpret_cast<T*>(smem_raw);
        T* B = A + cnt;
        swt_stage(A, s2 ? p.a2 + b * p.a2_bs : p.a + b * p.a_bs, p, t, 0, t.rows);
        __syncthreads();
        int lo = 0, hi = t.rows;
        for (int k = 0; k < p.K; ++k) {
            const int64_t dk = p.d0 << k;
            const int olo = t.full ? 0 : lo + (int)(dk * hl);
            const int ohi = t.full ? hi : hi - (int)(dk * (L / 2));
            const bool last = k == p.K - 1;
            T* det = s2 ? p.det2 + b * p.det2_bs : p.det[k] + b * p.det_bs;
            T* out = s2 ? p.out2 + b * p.out2_bs : p.out + b * p.out_bs;
            auto emit = [&](int row, int col, T vlo, T vhi) {
                if (!last) B[(row << p.lgR) + col] = vlo;
                if (row >= t.HLr && row < t.own_hi) {
                    const int64_t g = (t.i0 + row - t.HLr) * p.D + t.c0 + col;
                    det[g] = vhi;
                    if (last) out[g] = vlo;
                }
            };
            const int nrows = ohi - olo;
            // unrolled path: SWT_Q outputs dk rows apart per thread share L + SWT_Q - 1 staged samples
            const bool unrolled = LT > 0 && dk * SWT_Q <= nrows && (!t.full || dk * (L + SWT_Q) <= p.M);
            if (unrolled) {
                constexpr int NV = (LT > 0 ? LT : 2) + SWT_Q - 1;
                const int S = (int)dk;
                const int lanes = S << p.lgR;                 // S and R are powers of two
                const int nblk = (nrows + SWT_Q * S - 1) / (SWT_Q * S);
                for (int u = threadIdx.x; u < nblk * lanes; u += SWT_THREADS) {
                    const int blk = u / lanes, w = u - blk * lanes;
                    const int row0 = olo + blk * SWT_Q * S + (w >> p.lgR), col = w & (p.R - 1);
                    T v[NV];
#pragma unroll
                    for (int e = 0; e < NV; ++e) {
                        const int r = row0 + (e - hl) * S;
                        v[e] = (t.full || r < hi) ? A[(swt_wrap1(r, (int)p.M, t.full) << p.lgR) + col] : T(0);
                    }
#pragma unroll
                    for (int q = 0; q < SWT_Q; ++q) {
                        T alo = T(0), ahi = T(0);
#pragma unroll
                        for (int m = 0; m < (LT > 0 ? LT : 2); ++m) {
                            alo = fma(p.f0[m], v[q + m], alo);
                            ahi = fma(p.f1[m], v[q + m], ahi);
                        }
                        if (row0 + q * S < ohi) emit(row0 + q * S, col, alo, ahi);
                    }
                }
            } else {
                for (int u = threadIdx.x; u < nrows << p.lgR; u += SWT_THREADS) {
                    const int row = olo + (u >> p.lgR), col = u & (p.R - 1);
                    T alo = T(0), ahi = T(0);
                    for (int m = 0; m < L; ++m) {
                        const T v = A[(swt_wrap(row + (int64_t)(m - hl) * dk, p.M, t.full) << p.lgR) + col];
                        alo = fma(p.f0[m], v, alo);
                        ahi = fma(p.f1[m], v, ahi);
                    }
                    emit(row, col, alo, ahi);
                }
            }
            __syncthreads();
            T* tmp = A; A = B; B = tmp;
            lo = olo; hi = ohi;
        }
    }
}

// Synthesis: levels k = K-1 down to 0 of one tile; A holds the staged approximation, Dt the level's detail.
template <typename T, int LT>
__global__ void __launch_bounds__(SWT_THREADS, 1) swt_inv_kernel(const __grid_constant__ SwtTileParams<T> p) {
    constexpr int SWT_Q = swt_q<T>();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int L = LT > 0 ? LT : p.L;
    const int hl = L / 2 - 1;
    const SwtTile t = swt_tile(p, L / 2, hl);
    const int cnt = t.rows << p.lgR;
    for (int64_t bb = blockIdx.y; bb < p.batch * p.sets; bb += gridDim.y) {
        const bool s2 = bb >= p.batch;
        const int64_t b = s2 ? bb - p.batch : bb;
        T* A = reinterpret_cast<T*>(smem_raw);
        T* B = A + cnt;
        T* Dt = B + cnt;
        swt_stage(A, s2 ? p.a2 + b * p.a2_bs : p.a + b * p.a_bs, p, t, 0, t.rows);
        int lo = 0, hi = t.rows;
        for (int k = p.K - 1; k >= 0; --k) {
            const int64_t dk = p.d0 << k;
            swt_stage(Dt, s2 ? p.det2 + b * p.det2_bs : p.det[k] + b * p.det_bs, p, t, lo, hi);
            __syncthreads();
            const int olo = t.full ? 0 : lo + (int)(dk * (L / 2));
            const int ohi = t.full ? hi : hi - (int)(dk * hl);
            const bool last = k == 0;
            T* out = s2 ? p.out2 + b * p.out2_bs : p.out + b * p.out_bs;
            auto emit = [&](int row, int col, T v) {
                if (!last) B[(row << p.lgR) + col] = v;
                else if (row >= t.HLr && row < t.own_hi) out[(t.i0 + row - t.HLr) * p.D + t.c0 + col] = v;
            };
            const int nrows = ohi - olo;
            const bool unrolled = LT > 0 && dk * SWT_Q <= nrows && (!t.full || dk * (L + SWT_Q) <= p.M);
            if (unrolled) {
                constexpr int NV = (LT > 0 ? LT : 2) + SWT_Q - 1;
                const int S = (int)dk;
                const int lanes = S << p.lgR;
                const int nblk = (nrows + SWT_Q * S - 1) / (SWT_Q * S);
                for (int u = threadIdx.x; u < nblk * lanes; u += SWT_THREADS) {
                    const int blk = u / lanes, w = u - blk * lanes;
                    const int row0 = olo + blk * SWT_Q * S + (w >> p.lgR), col = w & (p.R - 1);
                    // v[e] = row0 + (e - L/2) * S: output q, tap m reads e = q - m + L - 1
                    T va[NV], vd[NV];
#pragma unroll
                    for (int e = 0; e < NV; ++e) {
                        const int r = row0 + (e - (LT > 0 ? LT : 2) / 2) * S;
                        const bool ok = t.full || r < hi;
                        const int s = (swt_wrap1(r, (int)p.M, t.full) << p.lgR) + col;
                        va[e] = ok ? A[s] : T(0);
                        vd[e] = ok ? Dt[s] : T(0);
                    }
#pragma unroll
                    for (int q = 0; q < SWT_Q; ++q) {
                        T alo = T(0), ahi = T(0);
#pragma unroll
                        for (int m = 0; m < (LT > 0 ? LT : 2); ++m) {
                            alo = fma(p.f0[m], va[q - m + NV - SWT_Q], alo);
                            ahi = fma(p.f1[m], vd[q - m + NV - SWT_Q], ahi);
                        }
                        if (row0 + q * S < ohi) emit(row0 + q * S, col, alo + ahi);
                    }
                }
            } else {
                for (int u = threadIdx.x; u < nrows << p.lgR; u += SWT_THREADS) {
                    const int row = olo + (u >> p.lgR), col = u & (p.R - 1);
                    T alo = T(0), ahi = T(0);
                    for (int m = 0; m < L; ++m) {
                        const int s = (swt_wrap(row + (int64_t)(hl - m) * dk, p.M, t.full) << p.lgR) + col;
                        alo = fma(p.f0[m], A[s], alo);
                        ahi = fma(p.f1[m], Dt[s], ahi);
                    }
                    emit(row, col, alo + ahi);
                }
            }
            __syncthreads();
            T* tmp = A; A = B; B = tmp;
            lo = olo; hi = ohi;
        }
    }
}

// One level straight from global memory, for the levels a tile cannot take.  tab == NULL: periodic extension
// with dilation d.  Otherwise a CSR table built on the host: int32 rowptr[n + 1], then at element offset
// 2 * ((n + 2) / 2) the (source index, tap) pairs of every output -- the reference's multi-round circular pad
// (or the transpose of it, for the adjoint).
template <typename T>
struct SwtLevelParams {
    const T* a0;               // analysis: the input; synthesis: approximation
    const T* a1;               // synthesis: detail
    int64_t a0_bs, a1_bs;
    T* o0;                     // analysis: low band (approximation); synthesis: the reconstruction
    T* o1;                     // analysis: detail
    int64_t o0_bs, o1_bs;
    int64_t batch, n, d;
    const int32_t* tab;
    int L;
    T f0[WT_MAX_FILT_LEN], f1[WT_MAX_FILT_LEN];
};

template <typename T, bool SYN>
__global__ void __launch_bounds__(256) swt_level_kernel(const __grid_constant__ SwtLevelParams<T> p) {
    const int hl = p.L / 2 - 1;
    const int64_t total = p.batch * p.n;
    for (int64_t u = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; u < total; u += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = u / p.n, i = u - b * p.n;
        const T* a0 = p.a0 + b * p.a0_bs;
        const T* a1 = SYN ? p.a1 + b * p.a1_bs : nullptr;
        T s0 = T(0), s1 = T(0);
        if (p.tab) {
            const int2* ent = reinterpret_cast<const int2*>(p.tab + 2 * ((p.n + 2) / 2));
            for (int e = p.tab[i]; e < p.tab[i + 1]; ++e) {
                const int2 ct = ent[e];
                s0 = fma(p.f0[ct.y], a0[ct.x], s0);
                s1 = fma(p.f1[ct.y], SYN ? a1[ct.x] : a0[ct.x], s1);
            }
        } else {
            for (int m = 0; m < p.L; ++m) {
                int64_t s = (i + (SYN ? hl - m : m - hl) * p.d) % p.n;
                if (s < 0) s += p.n;
                s0 = fma(p.f0[m], a0[s], s0);
                s1 = fma(p.f1[m], SYN ? a1[s] : a0[s], s1);
            }
        }
        if (SYN) {
            p.o0[b * p.o0_bs + i] = s0 + s1;
        } else {
            p.o0[b * p.o0_bs + i] = s0;
            p.o1[b * p.o1_bs + i] = s1;
        }
    }
}

// ---- host -----------------------------------------------------------------------------------------------------
// One launch of the plan: levels [j0, j0 + K) as a tile group, or (table / periodic) one level from global memory.
struct SwtStep {
    int j0, K;
    bool tiled;
    int64_t D, d0, C;
    int R, lgR;
};

static inline int swt_log2(int64_t v) {
    int l = 0;
    while ((int64_t(1) << (l + 1)) <= v) ++l;
    return l;
}

// Levels 1..levels, finest first; level j has dilation b0 2^(j-1) (1-D: b0 = 1; the 2-D pass along the slow axis:
// b0 = d W).  A level with a table always runs alone.  Otherwise the group starting at level j sees the signal as rows
// of D = gcd(n, b0 2^(j-1)) samples; it takes whole columns when a tile of at least one 32-byte sector per row holds
// all M = n / D rows, else a halo tile of as many levels as keep the halo within a quarter of the tile.  A tile's
// column count R is a power of two that divides D (for b0 = 1, D is a power of two itself).
static int swt_plan(int es, bool inverse, int levels, int L, int64_t n, const void* const* tables, SwtStep* steps,
                    int64_t b0 = 1) {
    const int64_t cap = (inverse ? SWT_INV_BUF_BYTES : SWT_FWD_BUF_BYTES) / es;
    int ns = 0;
    for (int j = 1; j <= levels;) {
        SwtStep s{};
        s.j0 = j;
        s.K = 1;
        if (tables && tables[j - 1]) {
            steps[ns++] = s;
            ++j;
            continue;
        }
        const int64_t d = b0 << (j - 1);
        const int64_t D = std::gcd(n, d);
        const int64_t Dp = D & -D;             // largest power of two dividing D
        const int64_t M = n / D;
        int kmax = 0;
        while (j + kmax <= levels && kmax < SWT_MAXK && !(tables && tables[j + kmax - 1])) ++kmax;
        const int64_t rmin = std::min<int64_t>(Dp, 32 / es);
        s.D = D;
        s.d0 = d / D;
        if (M * rmin <= cap) {
            s.tiled = true;
            s.K = kmax;
            s.C = M;
            s.lgR = swt_log2(std::min<int64_t>(Dp, cap / M));
        } else {
            const int64_t rows_cap = cap / rmin;
            int K = 0;
            while (K < kmax && s.d0 * (L - 1) * ((int64_t(1) << (K + 1)) - 1) <= rows_cap / 4) ++K;
            if (K > 0) {
                s.tiled = true;
                s.K = K;
                s.C = std::min<int64_t>(rows_cap - s.d0 * (L - 1) * ((int64_t(1) << K) - 1), M);
                s.lgR = swt_log2(rmin);
            }
        }
        s.R = 1 << s.lgR;
        steps[ns++] = s;
        j += s.K;
    }
    return ns;
}

template <typename T, int LT>
static cudaError_t swt_launch_tile(bool inverse, const SwtTileParams<T>& p, size_t smem, cudaStream_t st) {
    const int64_t ntile = (p.M + p.C - 1) / p.C;
    dim3 grid((unsigned)(ntile * (p.D / p.R)), (unsigned)std::min<int64_t>(p.batch * p.sets, 65535));
    const size_t most = (inverse ? 3 * SWT_INV_BUF_BYTES : 2 * SWT_FWD_BUF_BYTES) + 64;
    cudaError_t e;
    if (inverse) {
        e = ensure_dyn_smem(swt_inv_kernel<T, LT>, most);
        if (e == cudaSuccess) swt_inv_kernel<T, LT><<<grid, SWT_THREADS, smem, st>>>(p);
    } else {
        e = ensure_dyn_smem(swt_fwd_kernel<T, LT>, most);
        if (e == cudaSuccess) swt_fwd_kernel<T, LT><<<grid, SWT_THREADS, smem, st>>>(p);
    }
    return e == cudaSuccess ? cudaGetLastError() : e;
}

template <typename T>
static cudaError_t swt_run_tile(bool inverse, const SwtTileParams<T>& p, cudaStream_t st) {
    const int L = p.L, hl = L / 2 - 1;
    const int64_t span = ((int64_t(1) << p.K) - 1) * p.d0;
    const int64_t rows = p.C == p.M ? p.M : p.C + span * (hl + L / 2);
    const size_t smem = (size_t)(inverse ? 3 : 2) * (size_t)(rows << p.lgR) * sizeof(T);
    switch (L) {
        case 2: return swt_launch_tile<T, 2>(inverse, p, smem, st);
        case 4: return swt_launch_tile<T, 4>(inverse, p, smem, st);
        case 6: return swt_launch_tile<T, 6>(inverse, p, smem, st);
        case 8: return swt_launch_tile<T, 8>(inverse, p, smem, st);
        case 10: return swt_launch_tile<T, 10>(inverse, p, smem, st);
        case 12: return swt_launch_tile<T, 12>(inverse, p, smem, st);
        case 14: return swt_launch_tile<T, 14>(inverse, p, smem, st);
        case 16: return swt_launch_tile<T, 16>(inverse, p, smem, st);
        default: return swt_launch_tile<T, 0>(inverse, p, smem, st);
    }
}

template <typename T>
static cudaError_t swt_run_level(bool inverse, const SwtLevelParams<T>& p, cudaStream_t st) {
    const int64_t total = p.batch * p.n;
    const int64_t grid = std::max<int64_t>(1, std::min<int64_t>((total + 255) / 256, (int64_t)sm_count() * 16));
    if (inverse) swt_level_kernel<T, true><<<(unsigned)grid, 256, 0, st>>>(p);
    else swt_level_kernel<T, false><<<(unsigned)grid, 256, 0, st>>>(p);
    return cudaGetLastError();
}

}  // namespace wtb
