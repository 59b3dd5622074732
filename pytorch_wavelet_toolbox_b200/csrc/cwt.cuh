// cwt.cuh -- the continuous wavelet transform, ptwt.cwt, as uniformly partitioned overlap-save in float64.
//
// The reference runs one FFT convolution per scale (src/ptwt/continuous_transform.py:103-137): FFT of the filter,
// FFT of the data whenever the padded length nextpow2(n + K - 1) changes, product, inverse FFT, then a `diff`
// copy, a crop copy and finally a `torch.stack` of all scales.  Written as one FIR per scale s (host side,
// continuous.py) that is
//     y_s[t] = sum_j c_s[j] x[t + D_s - j],     c_s[j] = 0 outside [0, P_s H),  D_s = d_s H + e_s (0 <= e_s < H)
// with the diff, the -sqrt(s) factor and the crop folded into the taps c_s and the delay D_s.
//
// Blocks.  Hop H, FFT size F = 2H.  Data window q is x[(q - 1) H, (q + 1) H) (zero outside [0, n)); its spectrum
// X_q is computed once and shared by every scale.  Filter part p of channel c is c[pH, pH + H) zero-padded to F;
// its spectrum C_{c,p} (scaled by 1/F) is computed once per filter set and cached by the caller.  Output block b
// of channel c, samples t in [bH - e, bH - e + H), is the second half of
//     IFFT( sum_p X_{b + d - p} C_{c,p} )
// so no full-length convolution, diff, crop or stack buffer is ever written.  The output blocks of a channel are
// shifted by e rather than the taps by H - e, so a filter of K + 1 taps needs only ceil((K + 1) / H) parts.  The
// work per output sample is O(P + log F), not O(K); there are nb + 1 output blocks, nb = ceil(n / H).
//
// Channels.  A channel is one complex-wavelet scale (complex output) or a PAIR of real-wavelet scales packed as
// c = c_s1 + i c_s2: the input is real, so the real part of the channel's output is y_s1 and the imaginary part
// y_s2, and one inverse FFT serves two scales.
//
// Adjoint (gradient w.r.t. the data):  xbar = Re sum_c c^H ybar_c with ybar_c = ybar_s1 + i ybar_s2 for a pair.
// With Y_b = FFT([0_H, ybar_c on output block b]):  xbar[rH + i] = Re IFFT( Z_{r+1} + (-1)^k Z_r )[i],
//     Z_q = sum_c sum_p conj(C_{c,p}) Y_{c, q - d_c + p},
// one inverse FFT per data block after the sum over every channel.
//
// FFTs are complex128 in shared memory, two radix-2 stages per pass, with fp64 twiddles from a table the caller
// builds (tw[k] = exp(-2 pi i k / F), k < F / 2); spectra are kept in bit-reversed bin order (see cwt_fft_dif).
#pragma once

#include "common.cuh"

namespace wtb {

constexpr int CWT_THREADS = 256;
constexpr int CWT_MIN_LOG2 = 6;    // F = 64
constexpr int CWT_MAX_LOG2 = 12;   // F = 4096: 64 KB of complex128 per CTA
constexpr int CWT_META = 6;        // per channel: first part, parts P, delay d (blocks), scale s1, s2 (or -1), e

__device__ __forceinline__ double2 cwt_cmul(double2 a, double2 b) {
    return make_double2(fma(a.x, b.x, -a.y * b.y), fma(a.x, b.y, a.y * b.x));
}

__device__ __forceinline__ double2 cwt_cmul_conj(double2 a, double2 b) {   // a * conj(b)
    return make_double2(fma(a.x, b.x, a.y * b.y), fma(a.y, b.x, -a.x * b.y));
}

__device__ __forceinline__ double2 cwt_add(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 cwt_sub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }

// Spectra live in BIT-REVERSED bin order: the forward transforms take their input in natural order (conflict-free
// shared-memory stores) and leave the spectrum bit-reversed (decimation in frequency), the products are bin by bin,
// and the inverse transform takes them in that order and returns natural order (decimation in time).  Both do two
// radix-2 stages per pass over shared memory (one radix-2 stage more when lg is odd), with
// W_m^j = tw[j F / m], tw[k] = exp(-2 pi i k / F).  Both end with a barrier.

// Forward FFT, natural order in, bit-reversed order out.
__device__ void cwt_fft_dif(double2* buf, int lg, const double2* __restrict__ tw) {
    int s = lg - 2;
    for (; s >= 0; s -= 2) {
        // spans 2h then h, h = 2^s: a_m = a0 + m h; (a0, a2) with W_{4h}^j, (a1, a3) with W_{4h}^{j+h}, then
        // (a0, a1) and (a2, a3) with W_{2h}^j
        const int h = 1 << s, sh = lg - 2 - s;
        for (int b = threadIdx.x; b < (1 << (lg - 2)); b += blockDim.x) {
            const int j = b & (h - 1);
            const int a0 = ((b >> s) << (s + 2)) + j;
            const double2 w1 = __ldg(&tw[j << (sh + 1)]), w2 = __ldg(&tw[j << sh]), w3 = __ldg(&tw[(j + h) << sh]);
            const double2 x0 = buf[a0], x1 = buf[a0 + h], x2 = buf[a0 + 2 * h], x3 = buf[a0 + 3 * h];
            const double2 y0 = cwt_add(x0, x2), y2 = cwt_cmul(cwt_sub(x0, x2), w2);
            const double2 y1 = cwt_add(x1, x3), y3 = cwt_cmul(cwt_sub(x1, x3), w3);
            buf[a0] = cwt_add(y0, y1);
            buf[a0 + h] = cwt_cmul(cwt_sub(y0, y1), w1);
            buf[a0 + 2 * h] = cwt_add(y2, y3);
            buf[a0 + 3 * h] = cwt_cmul(cwt_sub(y2, y3), w1);
        }
        __syncthreads();
    }
    if (s == -1) {   // span 1, twiddle 1
        for (int b = threadIdx.x; b < (1 << (lg - 1)); b += blockDim.x) {
            const double2 u = buf[2 * b], v = buf[2 * b + 1];
            buf[2 * b] = cwt_add(u, v);
            buf[2 * b + 1] = cwt_sub(u, v);
        }
        __syncthreads();
    }
}

// Inverse FFT (unnormalised), bit-reversed order in, natural order out.
__device__ void cwt_ifft_dit(double2* buf, int lg, const double2* __restrict__ tw) {
    int s = 0;
    for (; s + 1 < lg; s += 2) {
        // spans h then 2h: (a0, a1) and (a2, a3) with conj W_{2h}^j, then (a0, a2) with conj W_{4h}^j and (a1, a3)
        // with conj W_{4h}^{j+h}
        const int h = 1 << s, sh = lg - 2 - s;
        for (int b = threadIdx.x; b < (1 << (lg - 2)); b += blockDim.x) {
            const int j = b & (h - 1);
            const int a0 = ((b >> s) << (s + 2)) + j;
            double2 w1 = __ldg(&tw[j << (sh + 1)]), w2 = __ldg(&tw[j << sh]), w3 = __ldg(&tw[(j + h) << sh]);
            w1.y = -w1.y; w2.y = -w2.y; w3.y = -w3.y;
            const double2 x0 = buf[a0], x2 = buf[a0 + 2 * h];
            const double2 t1 = cwt_cmul(buf[a0 + h], w1), t3 = cwt_cmul(buf[a0 + 3 * h], w1);
            const double2 y0 = cwt_add(x0, t1), y1 = cwt_sub(x0, t1), y2 = cwt_add(x2, t3), y3 = cwt_sub(x2, t3);
            const double2 t2 = cwt_cmul(y2, w2), t4 = cwt_cmul(y3, w3);
            buf[a0] = cwt_add(y0, t2);
            buf[a0 + 2 * h] = cwt_sub(y0, t2);
            buf[a0 + h] = cwt_add(y1, t4);
            buf[a0 + 3 * h] = cwt_sub(y1, t4);
        }
        __syncthreads();
    }
    if (s < lg) {    // span F / 2, conj W_F^j
        const int h = 1 << s;
        for (int b = threadIdx.x; b < h; b += blockDim.x) {
            double2 w = __ldg(&tw[b]);
            w.y = -w.y;
            const double2 u = buf[b], v = cwt_cmul(buf[b + h], w);
            buf[b] = cwt_add(u, v);
            buf[b + h] = cwt_sub(u, v);
        }
        __syncthreads();
    }
}

// spec[r] = FFT(taps[r] zero-padded to F) / F (bit-reversed bin order), one CTA per filter part r.
__global__ void __launch_bounds__(CWT_THREADS) cwt_filter_spectra_kernel(const double2* __restrict__ taps,
                                                                         const double2* __restrict__ tw,
                                                                         double2* __restrict__ spec, int lg) {
    extern __shared__ double2 cwt_buf[];
    const int F = 1 << lg, H = F >> 1;
    const int64_t r = blockIdx.x;
    for (int i = threadIdx.x; i < F; i += blockDim.x)
        cwt_buf[i] = i < H ? taps[r * H + i] : make_double2(0.0, 0.0);
    __syncthreads();
    cwt_fft_dif(cwt_buf, lg, tw);
    const double sc = 1.0 / F;
    for (int k = threadIdx.x; k < F; k += blockDim.x) {
        const double2 v = cwt_buf[k];
        spec[r * F + k] = make_double2(v.x * sc, v.y * sc);
    }
}

// X[sig][q] = FFT(x[sig][(q - 1) H, (q + 1) H)) (bit-reversed bin order), grid (window q, signal); input widened
// to fp64 on load.
template <typename T>
__global__ void __launch_bounds__(CWT_THREADS) cwt_data_spectra_kernel(const T* __restrict__ x, int64_t xbs,
                                                                       int64_t n, int64_t nq, int lg,
                                                                       const double2* __restrict__ tw,
                                                                       double2* __restrict__ X) {
    extern __shared__ double2 cwt_buf[];
    const int F = 1 << lg, H = F >> 1;
    const int64_t q = blockIdx.x, sig = blockIdx.y, base = (q - 1) * H;
    const T* xs = x + sig * xbs;
    for (int i = threadIdx.x; i < F; i += blockDim.x) {
        const int64_t t = base + i;
        cwt_buf[i] = make_double2(t >= 0 && t < n ? (double)xs[t] : 0.0, 0.0);
    }
    __syncthreads();
    cwt_fft_dif(cwt_buf, lg, tw);
    double2* Xs = X + (sig * nq + q) * F;
    for (int k = threadIdx.x; k < F; k += blockDim.x) Xs[k] = cwt_buf[k];
}

struct CwtParams {
    const int* meta;          // [channels][CWT_META], device
    const double2* spec;      // filter part spectra [parts][F], device
    const double2* tw;        // [F / 2]
    const double2* X;         // forward: data spectra [chunk][nq][F];  adjoint: output spectra [chunk][ch][nq][F]
    void* out;                // forward: coefficients;  adjoint: input gradient (T)
    const void* gy;           // adjoint: output gradient
    int64_t n, nb, nq, channels;   // nq = nb + 1 data windows and output blocks
    int64_t sig0;             // first signal of this chunk
    int64_t o_scale, o_batch; // element strides of the [S, batch, n] coefficients (complex elements if complex)
    int64_t gx_bs;            // adjoint: batch stride of the input gradient
    int lg;
};

// One CTA per (channel, output block, signal), channel fastest so the data spectra are re-read from L2.
template <bool CPLX>
__global__ void __launch_bounds__(CWT_THREADS) cwt_main_kernel(CwtParams p) {
    extern __shared__ double2 cwt_buf[];
    const int F = 1 << p.lg, H = F >> 1;
    const int64_t c = blockIdx.x % p.channels, b = blockIdx.x / p.channels, sig = blockIdx.z;
    const int* m = p.meta + c * CWT_META;
    const int part0 = m[0], P = m[1], d = m[2], s1 = m[3], s2 = m[4], e = m[5];
    const int64_t t0 = b * H - e;
    if (t0 >= p.n) return;                       // the whole CTA: this channel's output ends before the block
    // window q = b + d - pp must lie in [0, nq)
    const int64_t plo = max((int64_t)0, b + d - (p.nq - 1)), phi = min((int64_t)P - 1, b + d);
    const double2* Xs = p.X + (sig * p.nq + b + d) * F;
    const double2* Cs = p.spec + (int64_t)part0 * F;
    for (int k = threadIdx.x; k < F; k += blockDim.x) {
        double2 acc = make_double2(0.0, 0.0);
        for (int64_t pp = plo; pp <= phi; ++pp) {
            const double2 xv = __ldg(&Xs[k - pp * F]), cv = __ldg(&Cs[pp * F + k]);
            acc.x = fma(xv.x, cv.x, fma(-xv.y, cv.y, acc.x));
            acc.y = fma(xv.x, cv.y, fma(xv.y, cv.x, acc.y));
        }
        cwt_buf[k] = acc;
    }
    __syncthreads();
    cwt_ifft_dit(cwt_buf, p.lg, p.tw);
    const int64_t row = p.sig0 + sig;
    const int ilo = (int)max((int64_t)0, -t0), ihi = (int)min((int64_t)H, p.n - t0);
    const int64_t o1 = s1 * p.o_scale + row * p.o_batch + t0, o2 = s2 * p.o_scale + row * p.o_batch + t0;
    for (int i = ilo + threadIdx.x; i < ihi; i += blockDim.x) {
        const double2 v = cwt_buf[H + i];
        if (CPLX) {
            reinterpret_cast<double2*>(p.out)[o1 + i] = v;
        } else {
            double* o = reinterpret_cast<double*>(p.out);
            o[o1 + i] = v.x;
            if (s2 >= 0) o[o2 + i] = v.y;
        }
    }
}

// Adjoint, step 1: Y[sig][c][b] = FFT([0_H, ybar_c[bH - e, bH - e + H)]), grid (channel + block, signal).
template <bool CPLX>
__global__ void __launch_bounds__(CWT_THREADS) cwt_adj_spectra_kernel(CwtParams p, double2* __restrict__ Y) {
    extern __shared__ double2 cwt_buf[];
    const int F = 1 << p.lg, H = F >> 1;
    const int64_t c = blockIdx.x % p.channels, b = blockIdx.x / p.channels, sig = blockIdx.y;
    const int* m = p.meta + c * CWT_META;
    const int s1 = m[3], s2 = m[4], e = m[5];
    const int64_t row = p.sig0 + sig;
    for (int i = threadIdx.x; i < F; i += blockDim.x) {
        const int64_t t = b * H - e + i - H;
        double2 v = make_double2(0.0, 0.0);
        if (i >= H && t >= 0 && t < p.n) {
            if (CPLX) {
                v = reinterpret_cast<const double2*>(p.gy)[s1 * p.o_scale + row * p.o_batch + t];
            } else {
                const double* g = reinterpret_cast<const double*>(p.gy);
                v.x = g[s1 * p.o_scale + row * p.o_batch + t];
                if (s2 >= 0) v.y = g[s2 * p.o_scale + row * p.o_batch + t];
            }
        }
        cwt_buf[i] = v;
    }
    __syncthreads();
    cwt_fft_dif(cwt_buf, p.lg, p.tw);
    double2* Ys = Y + ((sig * p.channels + c) * p.nq + b) * F;
    for (int k = threadIdx.x; k < F; k += blockDim.x) Ys[k] = cwt_buf[k];
}

// Adjoint, step 2: one CTA per (data block r, signal) sums every channel and part, then one inverse FFT.
template <typename T>
__global__ void __launch_bounds__(CWT_THREADS) cwt_adj_main_kernel(CwtParams p) {
    extern __shared__ double2 cwt_buf[];
    const int F = 1 << p.lg, H = F >> 1;
    const int64_t r = blockIdx.x, sig = blockIdx.y;
    const double2* Ysig = p.X + sig * p.channels * p.nq * F;
    for (int k = threadIdx.x; k < F; k += blockDim.x) {
        const double sgn = (k >> (p.lg - 1)) ? -1.0 : 1.0;   // (-1)^(natural bin index): its lowest bit
        double2 acc = make_double2(0.0, 0.0);
        for (int64_t c = 0; c < p.channels; ++c) {
            const int* m = p.meta + c * CWT_META;
            const int part0 = m[0], P = m[1], d = m[2];
            const double2* Yc = Ysig + c * p.nq * F;
            // block b1 = r + 1 - d + pp feeds window r + 1, b0 = b1 - 1 feeds window r
            const int64_t plo = max((int64_t)0, d - r - 1), phi = min((int64_t)P - 1, p.nq - r + d - 1);
            for (int64_t pp = plo; pp <= phi; ++pp) {
                const int64_t b1 = r + 1 - d + pp, b0 = b1 - 1;
                double2 v = make_double2(0.0, 0.0);
                if (b1 < p.nq) v = __ldg(&Yc[b1 * F + k]);
                if (b0 >= 0) {
                    const double2 w = __ldg(&Yc[b0 * F + k]);
                    v.x = fma(sgn, w.x, v.x);
                    v.y = fma(sgn, w.y, v.y);
                }
                const double2 t = cwt_cmul_conj(v, __ldg(&p.spec[((int64_t)part0 + pp) * F + k]));
                acc.x += t.x;
                acc.y += t.y;
            }
        }
        cwt_buf[k] = acc;
    }
    __syncthreads();
    cwt_ifft_dit(cwt_buf, p.lg, p.tw);
    T* gx = reinterpret_cast<T*>(p.out) + (p.sig0 + sig) * p.gx_bs;
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        const int64_t t = r * H + i;
        if (t >= p.n) break;
        gx[t] = (T)cwt_buf[i].x;
    }
}

}  // namespace wtb
