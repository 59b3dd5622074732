// wtb200.cu -- C ABI (include/wtb200.h) and host-side drivers of the H100 wavelet
// filter bank.  Build: see build.py (nvcc -gencode arch=compute_90a,code=sm_90a).
//
// Host drivers here only sequence launches; they never allocate device memory, never
// synchronise, and keep no state besides the launch counter and the thread-local error
// string.

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "common.cuh"
#include "generic_axis.cuh"
#include "matrix_generic.cuh"
#include "axis1d_fast.cuh"
#include "matrix_fused.cuh"
#include "matrix_dmma.cuh"
#include "axis1d_fused.cuh"
#include "tap_grad.cuh"
#include "swt.cuh"
#include "cwt.cuh"

namespace wtb {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

static int cuda_fail(cudaError_t e, const char* what) {
    snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
    return (int)e;
}

}  // namespace wtb
#include "fused2d.cuh"
#include "fused2d_wpair.cuh"
#include "fused2d_fuse2.cuh"
#include "inv2d.cuh"
#include "fwd3d.cuh"
#include "inv3d.cuh"
namespace wtb {

static inline int pad_left(int L) { return (2 * L - 3) / 2; }

static inline int64_t coeff_len(int64_t n, int L) {
    // F.pad by (padl, padl + n%2) then a stride-2 valid convolution with L taps
    // (reference src/ptwt/_util.py:222-228).
    const int64_t padl = pad_left(L);
    const int64_t padded = n + 2 * padl + (n % 2);
    return (padded - L) / 2 + 1;
}

static int grid_for(int64_t total, int block) {
    int64_t g = (total + block - 1) / block;
    const int64_t cap = (int64_t)sm_count() * 64;  // grid-stride beyond this
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

template <typename T>
static void fill_taps(Taps<T>& t, const double* lo, const double* hi, int L, bool flip) {
    for (int k = 0; k < L; ++k) {
        const int s = flip ? L - 1 - k : k;
        t.lo[k] = (T)lo[s];
        t.hi[k] = (T)hi[s];
    }
}

// ---- one single-axis pass over a [o1, o2, n, inner] view -------------------------------
template <typename T>
struct View {
    T* ptr;
    int64_t s_o1, s_o2, s_n;
};

template <typename T>
static cudaError_t launch_axis_fwd(const View<const T>& x, const View<T>& lo, const View<T>& hi,
                                   int64_t o1, int64_t o2, int64_t n, int64_t inner, int mode, int L,
                                   const Taps<T>& taps, cudaStream_t st) {
    AxisFwdParams<T> p;
    p.x = x.ptr; p.lo = lo.ptr; p.hi = hi.ptr;
    p.n = n; p.m = coeff_len(n, L); p.inner = inner; p.o1 = o1; p.o2 = o2;
    p.xs_o1 = x.s_o1; p.xs_o2 = x.s_o2; p.xs_n = x.s_n;
    p.ls_o1 = lo.s_o1; p.ls_o2 = lo.s_o2; p.ls_m = lo.s_n;
    p.hs_o1 = hi.s_o1; p.hs_o2 = hi.s_o2; p.hs_m = hi.s_n;
    p.mode = mode; p.L = L; p.padl = pad_left(L);
    p.taps = taps;
    const int64_t total = o1 * o2 * p.m * inner;
    if (total == 0) return cudaSuccess;
    axis_fwd_kernel<T><<<grid_for(total, 256), 256, 0, st>>>(p);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

template <typename T>
static cudaError_t launch_axis_inv(const View<const T>& lo, const View<const T>& hi, const View<T>& y,
                                   int64_t o1, int64_t o2, int64_t m, int64_t nout, int64_t inner, int L,
                                   const Taps<T>& taps, cudaStream_t st) {
    AxisInvParams<T> p;
    p.lo = lo.ptr; p.hi = hi.ptr; p.y = y.ptr;
    p.m = m; p.nout = nout; p.inner = inner; p.o1 = o1; p.o2 = o2;
    p.ls_o1 = lo.s_o1; p.ls_o2 = lo.s_o2; p.ls_m = lo.s_n;
    p.hs_o1 = hi.s_o1; p.hs_o2 = hi.s_o2; p.hs_m = hi.s_n;
    p.ys_o1 = y.s_o1; p.ys_o2 = y.s_o2; p.ys_n = y.s_n;
    p.L = L; p.padl = pad_left(L);
    p.taps = taps;
    const int64_t total = o1 * o2 * nout * inner;
    if (total == 0) return cudaSuccess;
    axis_inv_kernel<T><<<grid_for(total, 256), 256, 0, st>>>(p);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
}

// Scratch of the general (one launch per axis pass) path, in elements: the per-level temporaries of the LARGEST
// level.  Extents can grow from level to level (an explicit `levels` beyond dwt_max_level on an axis shorter than
// L - 2: n -> floor((n + L - 1) / 2) > n), so every level is walked.
//   analysis, level input [H, W] / [D, H, W] with coefficient extents M*:
//     2-D: 2 * batch * H * Mw                      3-D: 2 * batch * D * H * Mw + 4 * batch * D * Mh * Mw
//   synthesis, level output [OH, OW] / [OD, OH, OW] from coefficient extents M* (upper bounds: the output of a level
//   may be one sample longer than the next finer coefficient extent):
//     2-D: 2 * batch * OH * Mw                     3-D: 4 * batch * OD * Mh * Mw + 2 * batch * OD * OH * Mw
static void generic_scratch_elems(int ndim, int L, int levels, int64_t batch, const int64_t* dims, int inverse,
                                  int64_t* s1, int64_t* s2) {
    *s1 = 0; *s2 = 0;
    if (ndim == 1) return;
    int64_t cur[3] = {1, 1, 1};
    for (int a = 0; a < ndim; ++a) cur[a] = dims[a];
    int64_t best = -1;
    for (int l = 0; l < (levels > 0 ? levels : 1); ++l) {
        int64_t a1 = 0, a2 = 0, c[3] = {1, 1, 1};
        if (!inverse) {
            for (int a = 0; a < ndim; ++a) c[a] = coeff_len(cur[a], L);
            if (ndim == 2) {
                a1 = 2 * batch * cur[0] * c[1];
            } else {
                a1 = 2 * batch * cur[0] * cur[1] * c[2];
                a2 = 4 * batch * cur[0] * c[1] * c[2];
            }
        } else {
            int64_t full[3] = {1, 1, 1};
            for (int a = 0; a < ndim; ++a) { c[a] = coeff_len(cur[a] + (cur[a] & 1), L) + 1; full[a] = cur[a] + 1; }
            if (ndim == 2) {
                a1 = 2 * batch * full[0] * c[1];
            } else {
                a1 = 4 * batch * full[0] * c[1] * c[2];
                a2 = 2 * batch * full[0] * full[1] * c[2];
            }
        }
        if (a1 + a2 > best) { best = a1 + a2; *s1 = a1; *s2 = a2; }
        for (int a = 0; a < ndim; ++a) cur[a] = c[a];
    }
}

// Which kernels run a 2-D or 3-D DWT call: the fused kernels, which run every level and need no workspace, or the
// general path (dwt_fwd_generic / dwt_inv_generic), which needs generic_scratch_elems.  Decided from the call's shapes
// alone, before its first launch, for wt_dwt_workspace_bytes and the transform alike, so the two always agree and a
// fused call never falls through to the general path.  The limits are those of the launchers, computed by the same
// geometry functions.  dims are the input extents of an analysis, the output extents of a synthesis.
enum DwtRoute { ROUTE_GENERAL, ROUTE_FUSED2D, ROUTE_FUSED3D };

static DwtRoute dwt_route(bool inverse, int ndim, int es, int levels, int L, int64_t batch, const int64_t* dims) {
    if (ndim < 2 || (L & 1) || knob_on(K_DISABLE_FUSED)) return ROUTE_GENERAL;
    if (ndim == 2 && (L > 16 || (inverse && es != 4))) return ROUTE_GENERAL;
    if (ndim == 3 && (L > 8 || es != 4 || batch > 65535)) return ROUTE_GENERAL;   // 3-D: the batch is gridDim.z
    // per level: n[] its input (analysis) or output (synthesis) extents, m[] its coefficient extents (coeff_len is
    // exact in both directions for even L)
    int64_t n[3], m[3];
    for (int a = 0; a < ndim; ++a) n[a] = dims[a];
    for (int l = 0; l < levels; ++l) {
        for (int a = 0; a < ndim; ++a) {
            m[a] = coeff_len(n[a], L);
            // 2-D: the strip kernels take level inputs (analysis) or coefficients (synthesis) below 2^30;
            // 3-D: the tile launchers narrow every extent to int
            if (ndim == 2 ? (inverse ? m[a] : n[a]) >= (int64_t(1) << 30) : n[a] >= (int64_t(1) << 31))
                return ROUTE_GENERAL;
        }
        bool fits;
        if (ndim == 2 && !inverse) {
            // the level-pair kernels fall back to the strip kernel, so it has to fit every level; a chunk of the
            // batch may be one image, which gives the most segments
            fits = fwd2d_grid(m[0], m[1], 1, L, fwd2d_strip_width(es)).nseg <= 65535;
        } else if (ndim == 2) {
            fits = inv2d_grid(n[0], n[1], batch, L).nseg <= 65535;
        } else if (!inverse) {
            const int* tile = FWD3D_TILES[fwd3d_tile_shape(m[1], m[2], L)];
            fits = fwd3d_grid(m[0], m[1], m[2], batch, tile[0], tile[1]).fits(batch);
        } else {
            fits = inv3d_grid(n[0], n[1], n[2], batch).fits(batch);
        }
        if (!fits) return ROUTE_GENERAL;
        for (int a = 0; a < ndim; ++a) n[a] = m[a];
    }
    return ndim == 2 ? ROUTE_FUSED2D : ROUTE_FUSED3D;
}

// The kernels of both paths read and write rows of unit stride.
static bool unit_rows(int ndim, const int64_t* strides, const wt_level* lv, int levels) {
    const int a = ndim - 1;
    if (strides[a] != 1) return false;
    for (int l = 0; l < levels; ++l)
        if (lv[l].strides[a] != 1 || lv[l].approx_strides[a] != 1) return false;
    return true;
}

template <typename T>
static int dwt_fwd_generic(int ndim, int mode, int levels, int L, const Taps<T>& taps, const T* x,
                           int64_t batch, const int64_t* dims, const int64_t* xs, int64_t xbs,
                           const wt_level* lv, T* ws, cudaStream_t st) {
    int64_t cur[3];
    int64_t cs[3];
    int64_t cbs = xbs;
    const T* src = x;
    for (int a = 0; a < ndim; ++a) { cur[a] = dims[a]; cs[a] = xs[a]; }
    for (int l = 0; l < levels; ++l) {
        if (ndim == 1 && cs[0] == 1 && !knob_on(K_DISABLE_FUSED)) {
            // group of consecutive levels -> one fused launch (intermediate approximations stay in shared memory;
            // their scratch buffers are left untouched, see the scratch semantics in include/wtb200.h)
            int kmax = 5;
            if (knob_is_set(K_CONVF_K)) { const int v = (int)knob_val(K_CONVF_K, 0); if (v >= 1 && v <= CONVF_MAXK) kmax = v; }
            int k = levels - l < kmax ? levels - l : kmax;
            bool ok = k >= 2;
            int64_t nn[CONVF_MAXK + 1];
            void* hi_ptr[CONVF_MAXK];
            int64_t hi_bs[CONVF_MAXK];
            nn[0] = cur[0];
            for (int j = 0; j < k && ok; ++j) {
                const wt_level& dj = lv[l + j];
                nn[j + 1] = dj.dims[0];
                hi_ptr[j] = dj.details;
                hi_bs[j] = dj.details_batch_stride;
                if (dj.strides[0] != 1 || dj.approx_strides[0] != 1) ok = false;
            }
            if (ok) {
                T flo[16], fhi[16];
                if (L <= 16) for (int q = 0; q < L; ++q) { flo[q] = taps.lo[L - 1 - q]; fhi[q] = taps.hi[L - 1 - q]; }
                const wt_level& dl = lv[l + k - 1];
                cudaError_t e = cudaSuccess;
                if (L <= 16 && launch_conv1d_fused<T>(L, k, nn, mode, src, cbs, batch, hi_ptr, hi_bs, (T*)dl.approx,
                                                      dl.approx_batch_stride, flo, fhi, st, &e)) {
                    g_launches.fetch_add(1, std::memory_order_relaxed);
                    if (e != cudaSuccess) return cuda_fail(e, "conv1d_fused_kernel");
                    src = (const T*)dl.approx; cbs = dl.approx_batch_stride;
                    cur[0] = dl.dims[0]; cs[0] = dl.approx_strides[0];
                    l += k - 1;
                    continue;
                }
            }
        }
        const wt_level& d = lv[l];
        T* det = (T*)d.details;
        T* app = (T*)d.approx;
        // output band k as a view: s_o1 = batch stride; st(k)[a] = element stride of axis a
        auto band = [&](int k) -> View<T> {
            if (k == 0) return View<T>{app, d.approx_batch_stride, 0, 0};
            return View<T>{det + (int64_t)(k - 1) * d.band_stride, d.details_batch_stride, 0, 0};
        };
        auto st_of = [&](int k) -> const int64_t* { return k == 0 ? d.approx_strides : d.strides; };
        cudaError_t e = cudaSuccess;
        if (ndim == 1) {
            View<const T> xv{src, cbs, 0, cs[0]};
            View<T> lo = band(0), hi = band(1);
            lo.s_n = st_of(0)[0]; hi.s_n = st_of(1)[0];
            bool done1 = false;
            if (cs[0] == 1 && lo.s_n == 1 && hi.s_n == 1 && cur[0] < (1 << 30) && L <= 16 && !knob_on(K_DISABLE_FUSED)) {
                Fast1dParams<T> fp;
                memset(&fp, 0, sizeof(fp));
                fp.x = src; fp.lo = lo.ptr; fp.hi = hi.ptr;
                fp.xs = cbs; fp.ls = lo.s_o1; fp.hs = hi.s_o1;
                fp.n = fp.n_in = (int)cur[0]; fp.m = (int)d.dims[0];
                fp.base = -pad_left(L); fp.mode = mode;
                for (int k = 0; k < L; ++k) { fp.flo[k] = taps.lo[L - 1 - k]; fp.fhi[k] = taps.hi[L - 1 - k]; }
                done1 = launch_axis1d_fast<T, false>(fp, L, batch, st, &e);
                if (done1) g_launches.fetch_add(1, std::memory_order_relaxed);
                if (done1 && e != cudaSuccess) return cuda_fail(e, "axis1d_fast_kernel");
            }
            if (!done1) e = launch_axis_fwd<T>(xv, lo, hi, batch, 1, cur[0], 1, mode, L, taps, st);
            if (e != cudaSuccess) return cuda_fail(e, "axis_fwd_kernel");
        } else if (ndim == 2) {
            const int64_t H = cur[0], W = cur[1], Mw = d.dims[1];
            T* tlo = ws;
            T* thi = ws + batch * H * Mw;
            // pass along W (last axis): [batch, H, W] -> t{lo,hi} [batch, H, Mw]
            {
                View<const T> xv{src, cbs, cs[0], 1};
                View<T> lo{tlo, H * Mw, Mw, 1}, hi{thi, H * Mw, Mw, 1};
                e = launch_axis_fwd<T>(xv, lo, hi, batch, H, W, 1, mode, L, taps, st);
                if (e != cudaSuccess) return cuda_fail(e, "axis_fwd_kernel(W)");
            }
            // pass along H: t_lo -> (k=0, k=2), t_hi -> (k=1, k=3)
            for (int w = 0; w < 2; ++w) {
                View<const T> xv{w ? thi : tlo, H * Mw, 0, Mw};
                View<T> lo = band(w), hi = band(2 + w);
                lo.s_n = st_of(w)[0]; hi.s_n = st_of(2 + w)[0];
                e = launch_axis_fwd<T>(xv, lo, hi, batch, 1, H, Mw, mode, L, taps, st);
                if (e != cudaSuccess) return cuda_fail(e, "axis_fwd_kernel(H)");
            }
        } else {
            const int64_t D = cur[0], H = cur[1], W = cur[2];
            const int64_t Mh = d.dims[1], Mw = d.dims[2];
            const int64_t n1 = batch * D * H * Mw;
            T* t1[2] = {ws, ws + n1};
            const int64_t n2 = batch * D * Mh * Mw;
            T* t2base = ws + 2 * n1;
            // W pass: view [batch*?]: o1 = batch, o2 = D*H needs uniform stride -> do per (batch, D) x H rows
            // input [batch, D, H, W]: o1 = batch (stride cbs), o2 = D (stride cs[0]) with rows H folded
            // into n-major is not possible in one view, so fold (D, H) when contiguous, else loop D.
            if (cs[0] == H * cs[1]) {
                View<const T> xv{src, cbs, cs[1], 1};
                View<T> lo{t1[0], D * H * Mw, Mw, 1}, hi{t1[1], D * H * Mw, Mw, 1};
                e = launch_axis_fwd<T>(xv, lo, hi, batch, D * H, W, 1, mode, L, taps, st);
                if (e != cudaSuccess) return cuda_fail(e, "axis_fwd_kernel(W)");
            } else {
                for (int64_t z = 0; z < D; ++z) {
                    View<const T> xv{src + z * cs[0], cbs, cs[1], 1};
                    View<T> lo{t1[0] + z * H * Mw, D * H * Mw, Mw, 1}, hi{t1[1] + z * H * Mw, D * H * Mw, Mw, 1};
                    e = launch_axis_fwd<T>(xv, lo, hi, batch, H, W, 1, mode, L, taps, st);
                    if (e != cudaSuccess) return cuda_fail(e, "axis_fwd_kernel(W)");
                }
            }
            // H pass: t1[w] [batch*D, H, Mw] -> t2[h][w] [batch*D, Mh, Mw]
            for (int w = 0; w < 2; ++w) {
                View<const T> xv{t1[w], H * Mw, 0, Mw};
                View<T> lo{t2base + (0 * 2 + w) * n2, Mh * Mw, 0, Mw};
                View<T> hi{t2base + (1 * 2 + w) * n2, Mh * Mw, 0, Mw};
                e = launch_axis_fwd<T>(xv, lo, hi, batch * D, 1, H, Mw, mode, L, taps, st);
                if (e != cudaSuccess) return cuda_fail(e, "axis_fwd_kernel(H)");
            }
            // D pass: t2[h][w] [batch, D, Mh*Mw] -> bands k = 4 d + 2 h + w, inner = Mh*Mw needs the
            // output plane to be dense: out stride[0] == Mh * stride[1] and stride[1] == Mw ... general
            // case: treat inner = Mw rows and o2 = Mh.
            for (int hw = 0; hw < 4; ++hw) {
                View<const T> xv{t2base + hw * n2, D * Mh * Mw, Mw, Mh * Mw};
                View<T> lo = band(hw), hi = band(4 + hw);
                lo.s_o2 = st_of(hw)[1]; hi.s_o2 = st_of(4 + hw)[1];
                lo.s_n = st_of(hw)[0]; hi.s_n = st_of(4 + hw)[0];
                e = launch_axis_fwd<T>(xv, lo, hi, batch, Mh, D, Mw, mode, L, taps, st);
                if (e != cudaSuccess) return cuda_fail(e, "axis_fwd_kernel(D)");
            }
        }
        src = app; cbs = d.approx_batch_stride;
        for (int a = 0; a < ndim; ++a) { cur[a] = d.dims[a]; cs[a] = d.approx_strides[a]; }
    }
    return 0;
}

template <typename T>
static int dwt_inv_generic(int ndim, int levels, int L, const Taps<T>& taps, T* y, int64_t batch,
                           const int64_t* out_dims, const int64_t* ys, int64_t ybs, const wt_level* lv,
                           T* ws, cudaStream_t st) {
    for (int l = levels - 1; l >= 0; --l) {
        const wt_level& d = lv[l];
        const T* det = (const T*)d.details;
        const T* app = (const T*)d.approx;
        auto band = [&](int k) -> View<const T> {
            if (k == 0) return View<const T>{app, d.approx_batch_stride, 0, 0};
            return View<const T>{det + (int64_t)(k - 1) * d.band_stride, d.details_batch_stride, 0, 0};
        };
        auto st_of = [&](int k) -> const int64_t* { return k == 0 ? d.approx_strides : d.strides; };
        // destination of this level's reconstruction
        T* dst; int64_t dbs; int64_t ds[3]; int64_t dd[3];
        if (l > 0) {
            dst = (T*)lv[l - 1].approx; dbs = lv[l - 1].approx_batch_stride;
            for (int a = 0; a < ndim; ++a) { ds[a] = lv[l - 1].approx_strides[a]; dd[a] = lv[l - 1].dims[a]; }
        } else {
            dst = y; dbs = ybs;
            for (int a = 0; a < ndim; ++a) { ds[a] = ys[a]; dd[a] = out_dims[a]; }
        }
        cudaError_t e = cudaSuccess;
        if (ndim == 1) {
            View<const T> lo = band(0), hi = band(1);
            lo.s_n = st_of(0)[0]; hi.s_n = st_of(1)[0];
            View<T> yv{dst, dbs, 0, ds[0]};
            bool done1 = false;
            if (lo.s_n == 1 && hi.s_n == 1 && ds[0] == 1 && d.dims[0] < (1 << 29) && L <= 16 && !knob_on(K_DISABLE_FUSED)) {
                Fast1dInvParams<T> fp;
                memset(&fp, 0, sizeof(fp));
                fp.lo = lo.ptr; fp.hi = hi.ptr; fp.y = dst;
                fp.ls = lo.s_o1; fp.hs = hi.s_o1; fp.ys = dbs;
                fp.m = (int)d.dims[0]; fp.nout = (int)dd[0];
                for (int k = 0; k < L; ++k) { fp.rlo[k] = taps.lo[k]; fp.rhi[k] = taps.hi[k]; }
                done1 = launch_axis1d_inv_fast<T>(fp, L, batch, st, &e);
                if (done1) g_launches.fetch_add(1, std::memory_order_relaxed);
                if (done1 && e != cudaSuccess) return cuda_fail(e, "axis1d_inv_fast_kernel");
            }
            if (!done1) e = launch_axis_inv<T>(lo, hi, yv, batch, 1, d.dims[0], dd[0], 1, L, taps, st);
            if (e != cudaSuccess) return cuda_fail(e, "axis_inv_kernel");
        } else if (ndim == 2) {
            const int64_t Mh = d.dims[0], Mw = d.dims[1], OH = dd[0], OW = dd[1];
            T* t[2] = {ws, ws + batch * OH * Mw};
            // along H: (k=0,k=2) -> t_lo ; (k=1,k=3) -> t_hi    [batch, OH, Mw]
            for (int w = 0; w < 2; ++w) {
                View<const T> lo = band(w), hi = band(2 + w);
                lo.s_n = st_of(w)[0]; hi.s_n = st_of(2 + w)[0];
                View<T> yv{t[w], OH * Mw, 0, Mw};
                e = launch_axis_inv<T>(lo, hi, yv, batch, 1, Mh, OH, Mw, L, taps, st);
                if (e != cudaSuccess) return cuda_fail(e, "axis_inv_kernel(H)");
            }
            // along W
            View<const T> lo{t[0], OH * Mw, Mw, 1}, hi{t[1], OH * Mw, Mw, 1};
            View<T> yv{dst, dbs, ds[0], 1};
            e = launch_axis_inv<T>(lo, hi, yv, batch, OH, Mw, OW, 1, L, taps, st);
            if (e != cudaSuccess) return cuda_fail(e, "axis_inv_kernel(W)");
        } else {
            const int64_t Md = d.dims[0], Mh = d.dims[1], Mw = d.dims[2];
            const int64_t OD = dd[0], OH = dd[1], OW = dd[2];
            const int64_t n1 = batch * OD * Mh * Mw;
            T* t1 = ws;                 // 4 arrays [batch, OD, Mh, Mw]
            T* t2 = ws + 4 * n1;        // 2 arrays [batch, OD, OH, Mw]
            const int64_t n2 = batch * OD * OH * Mw;
            for (int hw = 0; hw < 4; ++hw) {
                View<const T> lo = band(hw), hi = band(4 + hw);
                lo.s_o2 = st_of(hw)[1]; hi.s_o2 = st_of(4 + hw)[1];
                lo.s_n = st_of(hw)[0]; hi.s_n = st_of(4 + hw)[0];
                View<T> yv{t1 + hw * n1, OD * Mh * Mw, Mw, Mh * Mw};
                e = launch_axis_inv<T>(lo, hi, yv, batch, Mh, Md, OD, Mw, L, taps, st);
                if (e != cudaSuccess) return cuda_fail(e, "axis_inv_kernel(D)");
            }
            for (int w = 0; w < 2; ++w) {
                View<const T> lo{t1 + (0 * 2 + w) * n1, Mh * Mw, 0, Mw}, hi{t1 + (1 * 2 + w) * n1, Mh * Mw, 0, Mw};
                View<T> yv{t2 + w * n2, OH * Mw, 0, Mw};
                e = launch_axis_inv<T>(lo, hi, yv, batch * OD, 1, Mh, OH, Mw, L, taps, st);
                if (e != cudaSuccess) return cuda_fail(e, "axis_inv_kernel(H)");
            }
            if (ds[0] == OH * ds[1]) {
                View<const T> lo{t2, OD * OH * Mw, Mw, 1}, hi{t2 + n2, OD * OH * Mw, Mw, 1};
                View<T> yv{dst, dbs, ds[1], 1};
                e = launch_axis_inv<T>(lo, hi, yv, batch, OD * OH, Mw, OW, 1, L, taps, st);
                if (e != cudaSuccess) return cuda_fail(e, "axis_inv_kernel(W)");
            } else {
                for (int64_t z = 0; z < OD; ++z) {
                    View<const T> lo{t2 + z * OH * Mw, OD * OH * Mw, Mw, 1}, hi{t2 + n2 + z * OH * Mw, OD * OH * Mw, Mw, 1};
                    View<T> yv{dst + z * ds[0], dbs, ds[1], 1};
                    e = launch_axis_inv<T>(lo, hi, yv, batch, OH, Mw, OW, 1, L, taps, st);
                    if (e != cudaSuccess) return cuda_fail(e, "axis_inv_kernel(W)");
                }
            }
        }
    }
    return 0;
}

static int check_common(int ndim, int dtype, int levels, int L, int64_t batch, const int64_t* dims) {
    if (ndim < 1 || ndim > WT_MAX_NDIM) return fail(WT_EINVAL, "ndim must be 1..3, got %d", ndim);
    if (dtype != WT_F32 && dtype != WT_F64) return fail(WT_EINVAL, "dtype must be WT_F32 or WT_F64");
    if (levels < 0) return fail(WT_EINVAL, "levels must be >= 0");
    if (L < 2 || L > WT_MAX_FILT_LEN) return fail(WT_EUNSUPPORTED, "filter length %d outside [2, %d]", L, WT_MAX_FILT_LEN);
    if (batch < 0) return fail(WT_EINVAL, "negative batch");
    if (!dims) return fail(WT_EINVAL, "dims is NULL");
    for (int a = 0; a < ndim; ++a)
        if (dims[a] < 1) return fail(WT_ESHAPE, "extent %d is %lld", a, (long long)dims[a]);
    return 0;
}

template <typename T>
static int dwt_fwd_t(int ndim, int mode, int levels, int L, const double* dlo, const double* dhi,
                     const void* x, int64_t batch, const int64_t* dims, const int64_t* xs, int64_t xbs,
                     const wt_level* lv, void* ws, size_t ws_bytes, cudaStream_t st) {
    Taps<T> taps;
    fill_taps(taps, dlo, dhi, L, false);
    // validate extents against the reference's formula
    int64_t cur[3];
    for (int a = 0; a < ndim; ++a) cur[a] = dims[a];
    for (int l = 0; l < levels; ++l) {
        for (int a = 0; a < ndim; ++a) {
            const int64_t want = coeff_len(cur[a], L);
            if (lv[l].dims[a] != want)
                return fail(WT_ESHAPE, "level %d axis %d: extent %lld, expected %lld", l + 1, a,
                            (long long)lv[l].dims[a], (long long)want);
            cur[a] = want;
        }
        if (!lv[l].details || !lv[l].approx) return fail(WT_EINVAL, "level %d: NULL buffer", l + 1);
    }
    if (ndim > 1 && !unit_rows(ndim, xs, lv, levels)) return fail(WT_EINVAL, "innermost stride must be 1");
    const DwtRoute route = dwt_route(false, ndim, sizeof(T), levels, L, batch, dims);
    if constexpr (sizeof(T) == 4) {
        if (route == ROUTE_FUSED3D) return fused3d_fwd(mode, levels, L, dlo, dhi, (const float*)x, batch, dims, xs, xbs, lv, st);
    }
    if (route == ROUTE_FUSED2D) return fused2d_fwd<T>(mode, levels, L, dlo, dhi, (const T*)x, batch, dims, xs, xbs, lv, st);
    int64_t s1, s2;
    generic_scratch_elems(ndim, L, levels, batch, dims, 0, &s1, &s2);
    if (ndim > 1 && ((size_t)(s1 + s2) * sizeof(T) > ws_bytes || !ws))
        return fail(WT_EWORKSPACE, "workspace: need %zu bytes, have %zu", (size_t)(s1 + s2) * sizeof(T), ws_bytes);
    return dwt_fwd_generic<T>(ndim, mode, levels, L, taps, (const T*)x, batch, dims, xs, xbs, lv, (T*)ws, st);
}

template <typename T>
static int dwt_inv_t(int ndim, int levels, int L, const double* rlo, const double* rhi, void* y,
                     int64_t batch, const int64_t* out_dims, const int64_t* ys, int64_t ybs,
                     const wt_level* lv, void* ws, size_t ws_bytes, cudaStream_t st) {
    Taps<T> taps;
    fill_taps(taps, rlo, rhi, L, false);
    const int padl = pad_left(L);
    for (int l = levels - 1; l >= 0; --l) {
        for (int a = 0; a < ndim; ++a) {
            const int64_t full = 2 * (lv[l].dims[a] - 1) + L - 2 * padl;  // after the symmetric crop
            const int64_t next = l > 0 ? lv[l - 1].dims[a] : out_dims[a];
            if (!(next == full || next == full - 1))
                return fail(WT_ESHAPE, "level %d axis %d: reconstruction has %lld samples, next level expects %lld",
                            l + 1, a, (long long)full, (long long)next);
        }
        if (!lv[l].details || !lv[l].approx) return fail(WT_EINVAL, "level %d: NULL buffer", l + 1);
    }
    if (ndim > 1 && !unit_rows(ndim, ys, lv, levels)) return fail(WT_EINVAL, "innermost stride must be 1");
    const DwtRoute route = dwt_route(true, ndim, sizeof(T), levels, L, batch, out_dims);
    if constexpr (sizeof(T) == 4) {
        if (route == ROUTE_FUSED2D) return fused2d_inv(levels, L, rlo, rhi, (float*)y, batch, out_dims, ys, ybs, lv, st);
        if (route == ROUTE_FUSED3D) return fused3d_inv(levels, L, rlo, rhi, (float*)y, batch, out_dims, ys, ybs, lv, st);
    }
    int64_t s1, s2;
    generic_scratch_elems(ndim, L, levels, batch, out_dims, 1, &s1, &s2);
    if (ndim > 1 && ((size_t)(s1 + s2) * sizeof(T) > ws_bytes || !ws))
        return fail(WT_EWORKSPACE, "workspace: need %zu bytes, have %zu", (size_t)(s1 + s2) * sizeof(T), ws_bytes);
    return dwt_inv_generic<T>(ndim, levels, L, taps, (T*)y, batch, out_dims, ys, ybs, lv, (T*)ws, st);
}

// ---- matrix FWT -------------------------------------------------------------------------
template <typename T>
static int matrix_fwd_t(int levels, int L, const double* dlo, const double* dhi, const int64_t* n,
                        const int32_t* padded, int odd_mode, const int32_t* nbt, const int32_t* nbb,
                        const int32_t* wt, const int32_t* wb, const void* blocks, const void* x, int64_t batch,
                        int64_t xs, void* const* hi_out, const int64_t* hi_stride, void* lo_out,
                        int64_t lo_stride, void* scratch, size_t scratch_bytes, int allow_fused, cudaStream_t st) {
    Taps<T> taps;
    fill_taps(taps, dlo, dhi, L, false);
    const size_t need = levels > 1 ? (size_t)2 * batch * (n[0] / 2) * sizeof(T) : 0;
    if (need > scratch_bytes) return fail(WT_EWORKSPACE, "scratch: need %zu bytes, have %zu", need, scratch_bytes);
    const T* blk = (const T*)blocks;
    const T* src = (const T*)x;
    int64_t src_stride = xs;
    T* ping[2] = {(T*)scratch, (T*)scratch + batch * (n[0] / 2)};
    // block pointers of every level (lo_left, lo_right, hi_left, hi_right)
    const T* bptr[4 * 64];
    if (levels > 64) return fail(WT_EUNSUPPORTED, "more than 64 levels");
    {
        const T* q = blk;
        for (int l = 0; l < levels; ++l) {
            const int64_t nb = (int64_t)nbt[l] + nbb[l];
            bptr[4 * l] = q; q += nb * wt[l];
            bptr[4 * l + 1] = q; q += nb * wb[l];
            bptr[4 * l + 2] = q; q += nb * wt[l];
            bptr[4 * l + 3] = q; q += nb * wb[l];
        }
    }
    for (int l = 0; l < levels; ++l) {
        if (n[l] < 2 || (n[l] & 1)) return fail(WT_ESHAPE, "level %d: operator size %lld must be even", l + 1, (long long)n[l]);
        if (allow_fused && !knob_on(K_DISABLE_FUSED)) {
            // group of consecutive unpadded levels -> one fused launch
            int k = 0;
            // float32: 4 levels per launch while a row is cut into chunks, all remaining levels (up to MATF_MAXK) once
            // a whole row fits one chunk.  float64 (DMMA cascade): 2 levels per launch throughout (deeper cascades
            // save traffic but lose more to CTA barriers and thin coarse levels)
            const bool dmma64 = sizeof(T) == 8 && !knob_on(K_NO_DMMA);
            int kmax = n[l] <= 8192 ? (int)knob_val(K_MATF_KCOARSE, dmma64 ? 2 : MATF_MAXK) : (dmma64 ? 2 : 4);
            if (kmax < 1 || kmax > MATF_MAXK) kmax = MATF_MAXK;
            if (knob_is_set(K_MATF_K)) { const int v = (int)knob_val(K_MATF_K, 0); if (v >= 1 && v <= MATF_MAXK) kmax = v; }
            while (l + k < levels && k < kmax && !padded[l + k] && !(n[l + k] & 1) &&
                   (k == 0 || n[l + k] == n[l + k - 1] / 2))
                ++k;
            if (k >= 2) {
                const bool last = (l + k == levels);
                // the scratch half that is not this group's source (groups of even depth would otherwise write the
                // approximation over the buffer they are reading)
                T* lo_dst = last ? (T*)lo_out : (src == ping[0] ? ping[1] : ping[0]);
                const int64_t lo_ds = last ? lo_stride : n[l + k - 1] / 2;
                cudaError_t e = cudaSuccess;
                bool launched = false;
                if constexpr (sizeof(T) == 8) {
                    // float64: the polyphase band contraction on the FP64 tensor cores (matrix_dmma.cuh); the scalar
                    // cascade below where it does not apply
                    if (dmma64)
                        launched = launch_mat_fwd_dmma2(L, k, n + l, nbt + l, nbb + l, wt + l, wb + l,
                                                        (const double* const*)(bptr + 4 * l), (const double*)src, src_stride, batch,
                                                        hi_out + l, hi_stride + l, (double*)lo_dst, lo_ds, taps, st, &e);
                }
                if (launched ||
                    launch_mat_fwd_fused<T>(L, k, n + l, nbt + l, nbb + l, wt + l, wb + l, bptr + 4 * l, src, src_stride, batch,
                                            hi_out + l, hi_stride + l, lo_dst, lo_ds, taps, st, &e)) {
                    g_launches.fetch_add(1, std::memory_order_relaxed);
                    if (e != cudaSuccess) return cuda_fail(e, "mat_fwd_fused_kernel");
                    src = lo_dst; src_stride = lo_ds;
                    // keep blk in step with the per-level path
                    blk = bptr[4 * (l + k - 1) + 3] + ((int64_t)nbt[l + k - 1] + nbb[l + k - 1]) * wb[l + k - 1];
                    l += k - 1;
                    continue;
                }
            }
        }
        MatFwdParams<T> p;
        p.x = src; p.x_stride = src_stride;
        p.batch = batch; p.n = n[l]; p.n_in = n[l] - (padded[l] ? 1 : 0);
        p.hi = (T*)hi_out[l]; p.hi_stride = hi_stride[l];
        const bool last = (l == levels - 1);
        p.lo = last ? (T*)lo_out : (src == ping[0] ? ping[1] : ping[0]);
        p.lo_stride = last ? lo_stride : n[l] / 2;
        p.L = L; p.shift = L / 2 + (L % 2); p.odd_mode = odd_mode;
        p.nb_top = nbt[l]; p.nb_bot = nbb[l]; p.w_left = wt[l]; p.w_right = wb[l];
        const int64_t nb = (int64_t)nbt[l] + nbb[l];
        p.lo_left = blk; blk += nb * wt[l];
        p.lo_right = blk; blk += nb * wb[l];
        p.hi_left = blk; blk += nb * wt[l];
        p.hi_right = blk; blk += nb * wb[l];
        p.taps = taps;
        const int64_t total = batch * (n[l] / 2);
        if (total > 0) {
            bool done1 = false;
            cudaError_t e = cudaSuccess;
            if (n[l] < (1 << 30) && !(L & 1) && L <= 16 && !knob_on(K_DISABLE_FUSED)) {
                Fast1dParams<T> fp;
                memset(&fp, 0, sizeof(fp));
                fp.x = p.x; fp.lo = p.lo; fp.hi = p.hi;
                fp.xs = p.x_stride; fp.ls = p.lo_stride; fp.hs = p.hi_stride;
                fp.n = (int)p.n; fp.n_in = (int)p.n_in; fp.m = (int)(p.n / 2);
                fp.base = p.shift - (L - 1); fp.mode = odd_mode;
                fp.nb_top = p.nb_top; fp.nb_bot = p.nb_bot; fp.w_left = p.w_left; fp.w_right = p.w_right;
                fp.lo_left = p.lo_left; fp.lo_right = p.lo_right; fp.hi_left = p.hi_left; fp.hi_right = p.hi_right;
                for (int k = 0; k < L; ++k) { fp.flo[k] = taps.lo[L - 1 - k]; fp.fhi[k] = taps.hi[L - 1 - k]; }
                done1 = launch_axis1d_fast<T, true>(fp, L, batch, st, &e);
            }
            if (!done1) {
                mat_fwd_kernel<T><<<grid_for(total, 256), 256, 0, st>>>(p);
                e = cudaGetLastError();
            }
            g_launches.fetch_add(1, std::memory_order_relaxed);
            if (e != cudaSuccess) return cuda_fail(e, "mat_fwd_kernel");
        }
        src = p.lo; src_stride = p.lo_stride;
    }
    return 0;
}

template <typename T>
static int matrix_inv_t(int levels, int L, const double* rlo, const double* rhi, const int64_t* n,
                        const int64_t* next_len, const int32_t* nbt, const int32_t* nbb, const int32_t* wt,
                        const int32_t* wb, const void* blocks, const void* lo_in, int64_t lo_stride,
                        const void* const* hi_in, const int64_t* hi_stride, int64_t batch, void* y,
                        int64_t ys, void* scratch, size_t scratch_bytes, int allow_fused, cudaStream_t st) {
    Taps<T> taps;
    fill_taps(taps, rlo, rhi, L, true);  // rows of S^T carry the flipped rec filters
    const size_t need = levels > 1 ? (size_t)2 * batch * n[0] * sizeof(T) : 0;
    if (need > scratch_bytes) return fail(WT_EWORKSPACE, "scratch: need %zu bytes, have %zu", need, scratch_bytes);
    // block offsets per level
    int64_t off[64];
    if (levels > 64) return fail(WT_EUNSUPPORTED, "more than 64 levels");
    int64_t o = 0;
    for (int l = 0; l < levels; ++l) {
        off[l] = o;
        o += 2 * ((int64_t)nbt[l] + nbb[l]) * ((int64_t)wt[l] + wb[l]);
    }
    const T* src = (const T*)lo_in;
    int64_t src_stride = lo_stride;
    T* ping[2] = {(T*)scratch, (T*)scratch + batch * n[0]};
    int pp = 0;  // scratch half the next intermediate result goes to
    const T* bptr[4 * 64];
    for (int l = 0; l < levels; ++l) {
        const T* q = (const T*)blocks + off[l];
        const int64_t nb = (int64_t)nbt[l] + nbb[l];
        bptr[4 * l] = q; q += nb * wt[l];
        bptr[4 * l + 1] = q; q += nb * wb[l];
        bptr[4 * l + 2] = q; q += nb * wt[l];
        bptr[4 * l + 3] = q;
    }
    // float64: groups of levels run as one synthesis cascade on the FP64 tensor cores (matrix_dmma.cuh).  float32 (and
    // float64 with NO_DMMA) runs the register-blocked per-level kernels, which neither stage in shared memory nor
    // synchronise per level.
    const bool dmma = sizeof(T) == 8 && !knob_on(K_NO_DMMA);
    for (int l = levels - 1; l >= 0; --l) {
        if (dmma && allow_fused && !knob_on(K_DISABLE_FUSED)) {
            // group of levels l, l-1, ..., l-k+1 whose intermediate results are not trimmed -> one launch, 2 levels
            // per launch -- deeper cascades save HBM traffic but lose more to barriers and thin coarse levels.
            // WTB200_MATI_K sets the number of levels per launch.
            int kmax = 2;
            if (knob_is_set(K_MATI_K)) { const int v = (int)knob_val(K_MATI_K, 0); if (v >= 1 && v <= MATF_MAXK) kmax = v; }
            int k = 1;
            const int64_t merge_n = !knob_is_set(K_MATI_K) ? knob_val(K_MATI_MERGE_N, 1024) : 0;
            while (l - k >= 0 && next_len[l - k + 1] == n[l - k + 1] && n[l - k] == 2 * n[l - k + 1] &&
                   (k < kmax || (k < MATF_MAXK && n[l - k] <= merge_n)))
                ++k;
            if (k >= 2) {
                const int lf = l - k + 1;  // finest level of the group
                const bool last = (lf == 0);
                const int64_t keep0 = next_len[lf];
                const int64_t keep4 = (keep0 + 3) & ~int64_t(3);
                T* dst = last ? (T*)y : ping[pp];
                const int64_t dst_stride = last ? ys : (keep4 <= n[0] ? keep4 : keep0);
                cudaError_t e = cudaSuccess;
                bool launched = false;
                if constexpr (sizeof(T) == 8) {
                    if (keep0 == n[lf] || keep0 == n[lf] - 1)
                        launched = launch_mat_inv_dmma(L, k, n + lf, keep0, nbt + lf, nbb + lf, wt + lf, wb + lf,
                                                       (const double* const*)(bptr + 4 * lf), (const double*)src, src_stride,
                                                       hi_in + lf, hi_stride + lf, batch, (double*)dst, dst_stride, rlo, rhi,
                                                       st, &e);
                }
                if (launched) {
                    g_launches.fetch_add(1, std::memory_order_relaxed);
                    if (e != cudaSuccess) return cuda_fail(e, "mat_inv_dmma_kernel");
                    src = dst; src_stride = dst_stride;
                    if (!last) pp ^= 1;
                    l = lf;
                    continue;
                }
            }
        }
        MatInvParams<T> p;
        p.lo = src; p.lo_stride = src_stride;
        p.hi = (const T*)hi_in[l]; p.hi_stride = hi_stride[l];
        p.batch = batch; p.n = n[l]; p.keep = next_len[l];
        if (!(p.keep == p.n || p.keep == p.n - 1))
            return fail(WT_ESHAPE, "level %d: keep %lld of %lld samples", l + 1, (long long)p.keep, (long long)p.n);
        const bool last = (l == 0);
        p.y = last ? (T*)y : ping[pp];
        // intermediate rows start on 16-byte boundaries (vector loads of the next level) when they fit
        const int64_t keep4 = (p.keep + 3) & ~int64_t(3);
        p.y_stride = last ? ys : (keep4 <= n[0] ? keep4 : p.keep);
        p.L = L; p.shift = L / 2 + (L % 2);
        p.nb_top = nbt[l]; p.nb_bot = nbb[l]; p.w_left = wt[l]; p.w_right = wb[l];
        const T* blk = (const T*)blocks + off[l];
        const int64_t nb = (int64_t)nbt[l] + nbb[l];
        p.lo_left = blk; blk += nb * wt[l];
        p.lo_right = blk; blk += nb * wb[l];
        p.hi_left = blk; blk += nb * wt[l];
        p.hi_right = blk;
        p.taps = taps;
        const int64_t total = batch * p.keep;
        if (total > 0) {
            cudaError_t e = cudaSuccess;
            const bool fast = !knob_on(K_DISABLE_FUSED) && launch_mat_inv_fast<T>(p, st, &e);
            if (!fast) {
                mat_inv_kernel<T><<<grid_for(total, 256), 256, 0, st>>>(p);
                e = cudaGetLastError();
            }
            g_launches.fetch_add(1, std::memory_order_relaxed);
            if (e != cudaSuccess) return cuda_fail(e, fast ? "mat_inv_fast_kernel" : "mat_inv_kernel");
        }
        src = p.y; src_stride = p.y_stride;
        if (!last) pp ^= 1;
    }
    return 0;
}

}  // namespace wtb

using namespace wtb;

template <typename T>
static int matrix_axis_t(bool inverse, int L, const double* flo, const double* fhi, int64_t n, int64_t n_in, int64_t keep,
                         int odd_mode, int nbt, int nbb, int wl, int wr, const void* blocks, const void* x, int64_t outer,
                         int64_t inner, int64_t xos, int64_t xas, void* y, int64_t yos, int64_t yas, cudaStream_t st) {
    MatAxisParams<T> p;
    fill_taps(p.taps, flo, fhi, L, inverse);  // synthesis: rows of S^T carry the flipped rec filters
    p.x = (const T*)x; p.y = (T*)y;
    p.outer = outer; p.inner = inner; p.n = n; p.n_in = n_in; p.keep = keep;
    p.x_os = xos; p.x_as = xas; p.y_os = yos; p.y_as = yas;
    p.L = L; p.shift = L / 2 + (L % 2); p.odd_mode = odd_mode;
    p.nb_top = nbt; p.nb_bot = nbb; p.w_left = wl; p.w_right = wr;
    const T* blk = (const T*)blocks;
    const int64_t nb = (int64_t)nbt + nbb;
    p.lo_left = blk; blk += nb * wl;
    p.lo_right = blk; blk += nb * wr;
    p.hi_left = blk; blk += nb * wl;
    p.hi_right = blk;
    const int64_t total = outer * (inverse ? keep : n / 2) * inner;
    if (total <= 0) return 0;
    // contiguous axis: the register-blocked 1-D kernels of MatrixWavedec / MatrixWaverec apply directly
    if (inner == 1 && xas == 1 && yas == 1 && n < (int64_t(1) << 30) && !(L & 1) && L <= 16 && !knob_on(K_DISABLE_FUSED)) {
        cudaError_t e = cudaSuccess;
        bool done = true;
        // the row index rides on gridDim.y: at most 65535 rows per launch
        for (int64_t r0 = 0; r0 < outer && done && e == cudaSuccess; r0 += 65535) {
            const int64_t rows = outer - r0 < 65535 ? outer - r0 : 65535;
            if (inverse) {
                MatInvParams<T> q;
                q.lo = p.x + r0 * xos; q.hi = q.lo + n / 2; q.y = p.y + r0 * yos;
                q.batch = rows; q.n = n; q.keep = keep; q.lo_stride = xos; q.hi_stride = xos; q.y_stride = yos;
                q.L = L; q.shift = p.shift;
                q.nb_top = nbt; q.nb_bot = nbb; q.w_left = wl; q.w_right = wr;
                q.lo_left = p.lo_left; q.lo_right = p.lo_right; q.hi_left = p.hi_left; q.hi_right = p.hi_right;
                q.taps = p.taps;
                done = launch_mat_inv_fast<T>(q, st, &e);
            } else {
                Fast1dParams<T> fp;
                memset(&fp, 0, sizeof(fp));
                fp.x = p.x + r0 * xos; fp.lo = p.y + r0 * yos; fp.hi = fp.lo + n / 2;
                fp.xs = xos; fp.ls = yos; fp.hs = yos;
                fp.n = (int)n; fp.n_in = (int)n_in; fp.m = (int)(n / 2);
                fp.base = p.shift - (L - 1); fp.mode = odd_mode;
                fp.nb_top = nbt; fp.nb_bot = nbb; fp.w_left = wl; fp.w_right = wr;
                fp.lo_left = p.lo_left; fp.lo_right = p.lo_right; fp.hi_left = p.hi_left; fp.hi_right = p.hi_right;
                for (int k = 0; k < L; ++k) { fp.flo[k] = p.taps.lo[L - 1 - k]; fp.fhi[k] = p.taps.hi[L - 1 - k]; }
                done = launch_axis1d_fast<T, true>(fp, L, rows, st, &e);
            }
            if (done) g_launches.fetch_add(1, std::memory_order_relaxed);
            else if (r0 > 0) return fail(WT_EUNSUPPORTED, "row chunk %lld rejected by the fast path", (long long)r0);
        }
        if (done) {
            if (e != cudaSuccess) return cuda_fail(e, inverse ? "mat_inv_fast_kernel" : "axis1d_fast_kernel");
            return 0;
        }
    }
    if (inner > 1 && !knob_on(K_DISABLE_FUSED)) {
        cudaError_t e = cudaSuccess;
        if (launch_mat_axis_blk<T>(p, inverse, st, &e)) {
            g_launches.fetch_add(1, std::memory_order_relaxed);
            if (e != cudaSuccess) return cuda_fail(e, inverse ? "mat_axis_inv_blk_kernel" : "mat_axis_fwd_blk_kernel");
            return 0;
        }
    }
    if (inverse) mat_axis_inv_kernel<T><<<grid_for(total, 256), 256, 0, st>>>(p);
    else mat_axis_fwd_kernel<T><<<grid_for(total, 256), 256, 0, st>>>(p);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, inverse ? "mat_axis_inv_kernel" : "mat_axis_fwd_kernel");
    return 0;
}

static int matrix_axis_check(int dtype, int filt_len, const double* lo, const double* hi, int64_t n, int nbt, int nbb, int wl,
                             int wr, const void* blocks, const void* x, const void* y, int64_t outer, int64_t inner) {
    if (dtype != WT_F32 && dtype != WT_F64) return fail(WT_EINVAL, "dtype must be WT_F32 or WT_F64");
    if (filt_len < 2 || filt_len > WT_MAX_FILT_LEN) return fail(WT_EUNSUPPORTED, "filter length %d", filt_len);
    if (!lo || !hi) return fail(WT_EINVAL, "NULL filter");
    if (n < 2 || (n & 1)) return fail(WT_ESHAPE, "operator size %lld must be even", (long long)n);
    if (outer < 0 || inner < 0) return fail(WT_EINVAL, "negative extent");
    if (nbt < 0 || nbb < 0 || wl < 0 || wr < 0 || (int64_t)nbt + nbb > n / 2 || wl > n || wr > n)
        return fail(WT_EINVAL, "boundary block geometry");
    if (outer * inner > 0 && (!x || !y || (!blocks && nbt + nbb > 0))) return fail(WT_EINVAL, "NULL argument");
    return 0;
}

// ---- stationary transform -------------------------------------------------------------------------------------
static int swt_check(int dtype, int levels, int filt_len, const double* t0, const double* t1, int64_t batch, int64_t n) {
    if (dtype != WT_F32 && dtype != WT_F64) return fail(WT_EINVAL, "dtype must be WT_F32 or WT_F64");
    if (filt_len < 2 || filt_len > WT_MAX_FILT_LEN || (filt_len & 1))
        return fail(WT_EUNSUPPORTED, "filter length %d (even, 2..%d)", filt_len, WT_MAX_FILT_LEN);
    if (levels < 0 || levels > 40) return fail(WT_EINVAL, "levels %d", levels);
    if (batch < 0 || n < 1) return fail(WT_ESHAPE, "batch %lld, n %lld", (long long)batch, (long long)n);
    if (!t0 || !t1) return fail(WT_EINVAL, "NULL filter");
    return 0;
}

// Which buffer receives the approximation leaving step s of ns (in execution order): the last step writes the
// final one, the others alternate between the workspace and that final buffer, so no step reads what it writes.
static inline bool swt_to_workspace(int s, int ns) { return ((ns - 1 - s) & 1) != 0; }

template <typename T>
static int swt_fwd_t(int levels, int L, const double* f_lo, const double* f_hi, const T* x, int64_t batch, int64_t n,
                     int64_t xbs, T* out, int64_t obs, int64_t band, const void* const* tables, T* ws, size_t ws_bytes,
                     cudaStream_t st) {
    SwtStep steps[64];
    const int ns = swt_plan(sizeof(T), false, levels, L, n, tables, steps);
    if (ns > 1 && ws_bytes < (size_t)(batch * n) * sizeof(T)) return fail(WT_EWORKSPACE, "swt workspace too small");
    const T* in = x;
    int64_t in_bs = xbs;
    for (int s = 0; s < ns; ++s) {
        const SwtStep& S = steps[s];
        const bool to_ws = swt_to_workspace(s, ns);
        T* a_out = to_ws ? ws : out;
        const int64_t a_bs = to_ws ? n : obs;
        cudaError_t e;
        if (S.tiled) {
            SwtTileParams<T> p;
            memset(&p, 0, sizeof(p));
            p.a = in; p.a_bs = in_bs; p.out = a_out; p.out_bs = a_bs;
            for (int k = 0; k < S.K; ++k) p.det[k] = out + (int64_t)(levels + 1 - (S.j0 + k)) * band;
            p.det_bs = obs; p.batch = batch; p.sets = 1;
            p.D = S.D; p.M = n / S.D; p.d0 = S.d0; p.C = S.C;
            p.K = S.K; p.R = S.R; p.lgR = S.lgR; p.L = L;
            for (int m = 0; m < L; ++m) { p.f0[m] = (T)f_lo[m]; p.f1[m] = (T)f_hi[m]; }
            e = swt_run_tile<T>(false, p, st);
        } else {
            SwtLevelParams<T> p;
            memset(&p, 0, sizeof(p));
            p.a0 = in; p.a0_bs = in_bs;
            p.o0 = a_out; p.o0_bs = a_bs;
            p.o1 = out + (int64_t)(levels + 1 - S.j0) * band; p.o1_bs = obs;
            p.batch = batch; p.n = n; p.d = int64_t(1) << (S.j0 - 1); p.L = L;
            p.tab = tables ? (const int32_t*)tables[S.j0 - 1] : nullptr;
            for (int m = 0; m < L; ++m) { p.f0[m] = (T)f_lo[m]; p.f1[m] = (T)f_hi[m]; }
            e = swt_run_level<T>(false, p, st);
        }
        g_launches.fetch_add(1, std::memory_order_relaxed);
        if (e != cudaSuccess) return cuda_fail(e, S.tiled ? "swt_fwd_kernel" : "swt_level_kernel");
        in = a_out;
        in_bs = a_bs;
    }
    return 0;
}

template <typename T>
static int swt_inv_t(int levels, int L, const double* g_lo, const double* g_hi, const T* approx, int64_t abs_,
                     const T* det, int64_t dbs, int64_t band, int64_t batch, int64_t n, T* y, int64_t ybs,
                     const void* const* tables, T* ws, size_t ws_bytes, cudaStream_t st) {
    SwtStep steps[64];
    const int ns = swt_plan(sizeof(T), true, levels, L, n, tables, steps);
    if (ns > 1 && ws_bytes < (size_t)(batch * n) * sizeof(T)) return fail(WT_EWORKSPACE, "iswt workspace too small");
    const T* in = approx;
    int64_t in_bs = abs_;
    for (int s = 0; s < ns; ++s) {                       // coarsest group first
        const SwtStep& S = steps[ns - 1 - s];
        const bool to_ws = swt_to_workspace(s, ns);
        T* a_out = to_ws ? ws : y;
        const int64_t a_bs = to_ws ? n : ybs;
        cudaError_t e;
        if (S.tiled) {
            SwtTileParams<T> p;
            memset(&p, 0, sizeof(p));
            p.a = in; p.a_bs = in_bs; p.out = a_out; p.out_bs = a_bs;
            for (int k = 0; k < S.K; ++k) p.det[k] = const_cast<T*>(det) + (int64_t)(levels - (S.j0 + k)) * band;
            p.det_bs = dbs; p.batch = batch; p.sets = 1;
            p.D = S.D; p.M = n / S.D; p.d0 = S.d0; p.C = S.C;
            p.K = S.K; p.R = S.R; p.lgR = S.lgR; p.L = L;
            for (int m = 0; m < L; ++m) { p.f0[m] = (T)g_lo[m]; p.f1[m] = (T)g_hi[m]; }
            e = swt_run_tile<T>(true, p, st);
        } else {
            SwtLevelParams<T> p;
            memset(&p, 0, sizeof(p));
            p.a0 = in; p.a0_bs = in_bs;
            p.a1 = det + (int64_t)(levels - S.j0) * band; p.a1_bs = dbs;
            p.o0 = a_out; p.o0_bs = a_bs;
            p.batch = batch; p.n = n; p.d = int64_t(1) << (S.j0 - 1); p.L = L;
            p.tab = tables ? (const int32_t*)tables[S.j0 - 1] : nullptr;
            for (int m = 0; m < L; ++m) { p.f0[m] = (T)g_lo[m]; p.f1[m] = (T)g_hi[m]; }
            e = swt_run_level<T>(true, p, st);
        }
        g_launches.fetch_add(1, std::memory_order_relaxed);
        if (e != cudaSuccess) return cuda_fail(e, S.tiled ? "swt_inv_kernel" : "swt_level_kernel");
        in = a_out;
        in_bs = a_bs;
    }
    return 0;
}

// One level of one axis of the 2-D transform: the first group of swt_plan(levels = 1) at dilation b, on `sets` (1 or
// 2) band sets.  A tile takes both sets in one launch; the per-level kernel runs one launch per set.  Analysis: in0
// is the input, out0 / out1 the low / high band.  Synthesis: in0 / in1 the low / high band, out0 the result.
template <typename T>
static int swt_pass_t(bool inverse, int L, const double* f0, const double* f1, int64_t b, int sets,
                      const void* const* in0, const int64_t* in0_bs, const void* const* in1, const int64_t* in1_bs,
                      void* const* out0, const int64_t* out0_bs, void* const* out1, const int64_t* out1_bs,
                      int64_t batch, int64_t n, cudaStream_t st) {
    SwtStep steps[64];
    swt_plan(sizeof(T), inverse, 1, L, n, nullptr, steps, b);
    const SwtStep& S = steps[0];
    cudaError_t e = cudaSuccess;
    if (S.tiled) {
        SwtTileParams<T> p;
        memset(&p, 0, sizeof(p));
        p.a = (const T*)in0[0]; p.a_bs = in0_bs[0];
        p.out = (T*)out0[0]; p.out_bs = out0_bs[0];
        p.det[0] = inverse ? (T*)in1[0] : (T*)out1[0];
        p.det_bs = inverse ? in1_bs[0] : out1_bs[0];
        if (sets == 2) {
            p.a2 = (const T*)in0[1]; p.a2_bs = in0_bs[1];
            p.out2 = (T*)out0[1]; p.out2_bs = out0_bs[1];
            p.det2 = inverse ? (T*)in1[1] : (T*)out1[1];
            p.det2_bs = inverse ? in1_bs[1] : out1_bs[1];
        }
        p.batch = batch; p.sets = sets;
        p.D = S.D; p.M = n / S.D; p.d0 = S.d0; p.C = S.C;
        p.K = 1; p.R = S.R; p.lgR = S.lgR; p.L = L;
        for (int m = 0; m < L; ++m) { p.f0[m] = (T)f0[m]; p.f1[m] = (T)f1[m]; }
        e = swt_run_tile<T>(inverse, p, st);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        if (e != cudaSuccess) return cuda_fail(e, inverse ? "swt_inv_kernel" : "swt_fwd_kernel");
        return 0;
    }
    for (int s = 0; s < sets; ++s) {
        SwtLevelParams<T> p;
        memset(&p, 0, sizeof(p));
        p.a0 = (const T*)in0[s]; p.a0_bs = in0_bs[s];
        if (inverse) { p.a1 = (const T*)in1[s]; p.a1_bs = in1_bs[s]; }
        p.o0 = (T*)out0[s]; p.o0_bs = out0_bs[s];
        if (!inverse) { p.o1 = (T*)out1[s]; p.o1_bs = out1_bs[s]; }
        p.batch = batch; p.n = n; p.d = b; p.L = L;
        for (int m = 0; m < L; ++m) { p.f0[m] = (T)f0[m]; p.f1[m] = (T)f1[m]; }
        e = swt_run_level<T>(inverse, p, st);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        if (e != cudaSuccess) return cuda_fail(e, "swt_level_kernel");
    }
    return 0;
}

static const double g_unit_tap = 1.0;   // a non-NULL tap array for wt_swt_pass_plan's argument check

static int swt_pass_check(int dtype, int filt_len, const double* t0, const double* t1, int64_t dilation, int sets,
                          int64_t batch, int64_t n) {
    int rc = swt_check(dtype, 1, filt_len, t0, t1, batch, n);
    if (rc) return rc;
    if (dilation < 1) return fail(WT_EINVAL, "dilation %lld", (long long)dilation);
    if (sets != 1 && sets != 2) return fail(WT_EINVAL, "sets %d (1 or 2)", sets);
    return 0;
}

// ---- continuous transform --------------------------------------------------------------------------------------
// The batch runs in chunks of signals whose spectra fit CWT_WS_BUDGET; one chunk costs two launches.
constexpr size_t CWT_WS_BUDGET = size_t(1) << 29;

static int64_t cwt_blocks(int64_t n, int lg) { return (n + (int64_t(1) << (lg - 1)) - 1) >> (lg - 1); }

static size_t cwt_signal_bytes(int lg, int64_t n, int64_t channels, bool adjoint) {
    const int64_t nb = cwt_blocks(n, lg);
    return (size_t)((adjoint ? channels : 1) * (nb + 1) << lg) * sizeof(double2);
}

static int64_t cwt_chunk(int lg, int64_t batch, int64_t n, int64_t channels, bool adjoint) {
    const size_t per = cwt_signal_bytes(lg, n, channels, adjoint);
    int64_t c = (int64_t)std::max<size_t>(1, CWT_WS_BUDGET / per);
    return std::min<int64_t>(std::min<int64_t>(c, batch), 65535);
}

static int cwt_check(int lg, int64_t channels, int64_t batch, int64_t n) {
    if (lg < CWT_MIN_LOG2 || lg > CWT_MAX_LOG2)
        return fail(WT_EUNSUPPORTED, "cwt FFT size 2^%d (2^%d..2^%d)", lg, CWT_MIN_LOG2, CWT_MAX_LOG2);
    if (channels < 1 || batch < 0 || n < 1)
        return fail(WT_ESHAPE, "cwt channels %lld, batch %lld, n %lld", (long long)channels, (long long)batch,
                    (long long)n);
    if ((cwt_blocks(n, lg) + 1) * channels > INT32_MAX)
        return fail(WT_ESHAPE, "cwt grid too large");
    return 0;
}

template <typename K>
static cudaError_t cwt_prepare(K kern) { return ensure_dyn_smem(kern, sizeof(double2) << CWT_MAX_LOG2); }

template <typename T>
static int cwt_fwd_t(CwtParams p, const T* x, int64_t batch, int64_t xbs, bool cplx, double2* ws, size_t ws_bytes,
                     cudaStream_t st) {
    const int64_t chunk = cwt_chunk(p.lg, batch, p.n, p.channels, false);
    if (ws_bytes < (size_t)chunk * cwt_signal_bytes(p.lg, p.n, p.channels, false))
        return fail(WT_EWORKSPACE, "cwt workspace too small");
    const size_t smem = sizeof(double2) << p.lg;
    cudaError_t e = cwt_prepare(cwt_data_spectra_kernel<T>);
    if (e == cudaSuccess) e = cwt_prepare(cplx ? cwt_main_kernel<true> : cwt_main_kernel<false>);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(cwt)");
    p.X = ws;
    for (int64_t s0 = 0; s0 < batch; s0 += chunk) {
        const int64_t cs = std::min(chunk, batch - s0);
        cwt_data_spectra_kernel<T><<<dim3((unsigned)p.nq, (unsigned)cs), CWT_THREADS, smem, st>>>(
            x + s0 * xbs, xbs, p.n, p.nq, p.lg, p.tw, ws);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) return cuda_fail(e, "cwt_data_spectra_kernel");
        p.sig0 = s0;
        const dim3 grid((unsigned)(p.nq * p.channels), 1, (unsigned)cs);
        if (cplx) cwt_main_kernel<true><<<grid, CWT_THREADS, smem, st>>>(p);
        else cwt_main_kernel<false><<<grid, CWT_THREADS, smem, st>>>(p);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) return cuda_fail(e, "cwt_main_kernel");
    }
    return 0;
}

template <typename T>
static int cwt_adj_t(CwtParams p, int64_t batch, bool cplx, double2* ws, size_t ws_bytes, cudaStream_t st) {
    const int64_t chunk = cwt_chunk(p.lg, batch, p.n, p.channels, true);
    if (ws_bytes < (size_t)chunk * cwt_signal_bytes(p.lg, p.n, p.channels, true))
        return fail(WT_EWORKSPACE, "cwt adjoint workspace too small");
    const size_t smem = sizeof(double2) << p.lg;
    cudaError_t e = cwt_prepare(cplx ? cwt_adj_spectra_kernel<true> : cwt_adj_spectra_kernel<false>);
    if (e == cudaSuccess) e = cwt_prepare(cwt_adj_main_kernel<T>);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(cwt adjoint)");
    p.X = ws;
    for (int64_t s0 = 0; s0 < batch; s0 += chunk) {
        const int64_t cs = std::min(chunk, batch - s0);
        p.sig0 = s0;
        const dim3 g1((unsigned)(p.nq * p.channels), (unsigned)cs);
        if (cplx) cwt_adj_spectra_kernel<true><<<g1, CWT_THREADS, smem, st>>>(p, ws);
        else cwt_adj_spectra_kernel<false><<<g1, CWT_THREADS, smem, st>>>(p, ws);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) return cuda_fail(e, "cwt_adj_spectra_kernel");
        cwt_adj_main_kernel<T><<<dim3((unsigned)p.nb, (unsigned)cs), CWT_THREADS, smem, st>>>(p);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        if ((e = cudaGetLastError()) != cudaSuccess) return cuda_fail(e, "cwt_adj_main_kernel");
    }
    return 0;
}

static CwtParams cwt_params(int lg, int64_t channels, const int32_t* meta, const void* spectra, const void* twiddles,
                            int64_t n, int64_t out_scale_stride, int64_t out_batch_stride) {
    CwtParams p;
    memset(&p, 0, sizeof(p));
    p.meta = meta; p.spec = (const double2*)spectra; p.tw = (const double2*)twiddles;
    p.n = n; p.nb = cwt_blocks(n, lg); p.nq = p.nb + 1; p.channels = channels;
    p.o_scale = out_scale_stride; p.o_batch = out_batch_stride; p.lg = lg;
    return p;
}

extern "C" {

int wt_version(void) { return WT_VERSION; }

size_t wt_cwt_workspace_bytes(int fft_log2, int64_t batch, int64_t n, int64_t channels, int adjoint) {
    if (cwt_check(fft_log2, channels, batch, n) || batch < 1) return 0;
    return (size_t)cwt_chunk(fft_log2, batch, n, channels, adjoint != 0) *
           cwt_signal_bytes(fft_log2, n, channels, adjoint != 0);
}

int wt_cwt_filter_spectra(int fft_log2, int64_t parts, const void* taps, const void* twiddles, void* spectra,
                          void* stream) {
    if (fft_log2 < CWT_MIN_LOG2 || fft_log2 > CWT_MAX_LOG2) return fail(WT_EUNSUPPORTED, "cwt FFT size 2^%d", fft_log2);
    if (parts < 0 || parts > INT32_MAX) return fail(WT_ESHAPE, "cwt filter parts %lld", (long long)parts);
    if (parts == 0) return 0;
    if (!taps || !twiddles || !spectra) return fail(WT_EINVAL, "NULL argument");
    cudaError_t e = cwt_prepare(cwt_filter_spectra_kernel);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(cwt_filter_spectra_kernel)");
    cwt_filter_spectra_kernel<<<(unsigned)parts, CWT_THREADS, sizeof(double2) << fft_log2, (cudaStream_t)stream>>>(
        (const double2*)taps, (const double2*)twiddles, (double2*)spectra, fft_log2);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_fail(e, "cwt_filter_spectra_kernel");
    return 0;
}

int wt_cwt_fwd(int dtype, int fft_log2, int64_t channels, const int32_t* meta, const void* spectra,
               const void* twiddles, int complex_out, const void* x, int64_t batch, int64_t n, int64_t x_batch_stride,
               void* out, int64_t out_scale_stride, int64_t out_batch_stride, void* workspace, size_t workspace_bytes,
               void* stream) {
    if (dtype != WT_F32 && dtype != WT_F64) return fail(WT_EINVAL, "dtype must be WT_F32 or WT_F64");
    int rc = cwt_check(fft_log2, channels, batch, n);
    if (rc) return rc;
    if (batch == 0) return 0;
    if (!meta || !spectra || !twiddles || !x || !out || !workspace) return fail(WT_EINVAL, "NULL argument");
    CwtParams p = cwt_params(fft_log2, channels, meta, spectra, twiddles, n, out_scale_stride, out_batch_stride);
    p.out = out;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return cwt_fwd_t<float>(p, (const float*)x, batch, x_batch_stride, complex_out != 0, (double2*)workspace,
                                workspace_bytes, st);
    return cwt_fwd_t<double>(p, (const double*)x, batch, x_batch_stride, complex_out != 0, (double2*)workspace,
                             workspace_bytes, st);
}

int wt_cwt_adj(int dtype, int fft_log2, int64_t channels, const int32_t* meta, const void* spectra,
               const void* twiddles, int complex_out, const void* gy, int64_t out_scale_stride,
               int64_t out_batch_stride, int64_t batch, int64_t n, void* gx, int64_t gx_batch_stride,
               void* workspace, size_t workspace_bytes, void* stream) {
    if (dtype != WT_F32 && dtype != WT_F64) return fail(WT_EINVAL, "dtype must be WT_F32 or WT_F64");
    int rc = cwt_check(fft_log2, channels, batch, n);
    if (rc) return rc;
    if (batch == 0) return 0;
    if (!meta || !spectra || !twiddles || !gy || !gx || !workspace) return fail(WT_EINVAL, "NULL argument");
    CwtParams p = cwt_params(fft_log2, channels, meta, spectra, twiddles, n, out_scale_stride, out_batch_stride);
    p.gy = gy; p.out = gx; p.gx_bs = gx_batch_stride;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32) return cwt_adj_t<float>(p, batch, complex_out != 0, (double2*)workspace, workspace_bytes, st);
    return cwt_adj_t<double>(p, batch, complex_out != 0, (double2*)workspace, workspace_bytes, st);
}

size_t wt_swt_workspace_bytes(int dtype, int levels, int filt_len, int64_t batch, int64_t n,
                              const void* const* tables, int inverse) {
    if ((dtype != WT_F32 && dtype != WT_F64) || levels < 1 || levels > 40 || filt_len < 2 ||
        filt_len > WT_MAX_FILT_LEN || (filt_len & 1) || batch < 1 || n < 1)
        return 0;
    const int es = dtype == WT_F64 ? 8 : 4;
    SwtStep steps[64];
    return swt_plan(es, inverse != 0, levels, filt_len, n, tables, steps) > 1 ? (size_t)(batch * n) * es : 0;
}

int wt_swt_fwd(int dtype, int levels, int filt_len, const double* f_lo, const double* f_hi, const void* x,
               int64_t batch, int64_t n, int64_t x_batch_stride, void* out, int64_t out_batch_stride,
               int64_t out_band_stride, const void* const* tables, void* workspace, size_t workspace_bytes,
               void* stream) {
    int rc = swt_check(dtype, levels, filt_len, f_lo, f_hi, batch, n);
    if (rc) return rc;
    if (levels == 0 || batch == 0) return 0;
    if (!x || !out) return fail(WT_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return swt_fwd_t<float>(levels, filt_len, f_lo, f_hi, (const float*)x, batch, n, x_batch_stride, (float*)out,
                                out_batch_stride, out_band_stride, tables, (float*)workspace, workspace_bytes, st);
    return swt_fwd_t<double>(levels, filt_len, f_lo, f_hi, (const double*)x, batch, n, x_batch_stride, (double*)out,
                             out_batch_stride, out_band_stride, tables, (double*)workspace, workspace_bytes, st);
}

int wt_swt_inv(int dtype, int levels, int filt_len, const double* g_lo, const double* g_hi, const void* approx,
               int64_t approx_batch_stride, const void* details, int64_t details_batch_stride,
               int64_t details_band_stride, int64_t batch, int64_t n, void* y, int64_t y_batch_stride,
               const void* const* tables, void* workspace, size_t workspace_bytes, void* stream) {
    int rc = swt_check(dtype, levels, filt_len, g_lo, g_hi, batch, n);
    if (rc) return rc;
    if (levels == 0 || batch == 0) return 0;
    if (!approx || !details || !y) return fail(WT_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return swt_inv_t<float>(levels, filt_len, g_lo, g_hi, (const float*)approx, approx_batch_stride,
                                (const float*)details, details_batch_stride, details_band_stride, batch, n, (float*)y,
                                y_batch_stride, tables, (float*)workspace, workspace_bytes, st);
    return swt_inv_t<double>(levels, filt_len, g_lo, g_hi, (const double*)approx, approx_batch_stride,
                             (const double*)details, details_batch_stride, details_band_stride, batch, n, (double*)y,
                             y_batch_stride, tables, (double*)workspace, workspace_bytes, st);
}

int wt_swt_pass_plan(int dtype, int inverse, int filt_len, int64_t n, int64_t dilation, int64_t* tile) {
    int rc = swt_pass_check(dtype, filt_len, &g_unit_tap, &g_unit_tap, dilation, 1, 0, n);
    if (rc) return rc;
    if (!tile) return fail(WT_EINVAL, "NULL argument");
    SwtStep steps[64];
    swt_plan(dtype == WT_F64 ? 8 : 4, inverse != 0, 1, filt_len, n, nullptr, steps, dilation);
    const SwtStep& S = steps[0];
    tile[0] = S.D; tile[1] = S.tiled ? n / S.D : 0; tile[2] = S.C; tile[3] = S.R;
    return S.tiled ? 1 : 0;
}

size_t wt_swt2_workspace_bytes(int dtype, int levels, int64_t batch, int64_t h, int64_t w) {
    if ((dtype != WT_F32 && dtype != WT_F64) || levels < 1 || levels > 40 || batch < 1 || h < 1 || w < 1) return 0;
    const size_t plane = (size_t)(batch * h * w) * (dtype == WT_F64 ? 8 : 4);
    return plane * (levels > 1 ? 3 : 2);
}

int wt_swt_pass_fwd(int dtype, int filt_len, const double* f_lo, const double* f_hi, int64_t dilation, int sets,
                    const void* const* x, const int64_t* x_batch_stride, void* const* lo, const int64_t* lo_batch_stride,
                    void* const* hi, const int64_t* hi_batch_stride, int64_t batch, int64_t n, void* stream) {
    int rc = swt_pass_check(dtype, filt_len, f_lo, f_hi, dilation, sets, batch, n);
    if (rc) return rc;
    if (batch == 0) return 0;
    if (!x || !x_batch_stride || !lo || !lo_batch_stride || !hi || !hi_batch_stride) return fail(WT_EINVAL, "NULL argument");
    for (int s = 0; s < sets; ++s)
        if (!x[s] || !lo[s] || !hi[s]) return fail(WT_EINVAL, "NULL band of set %d", s);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return swt_pass_t<float>(false, filt_len, f_lo, f_hi, dilation, sets, x, x_batch_stride, nullptr, nullptr, lo,
                                 lo_batch_stride, hi, hi_batch_stride, batch, n, st);
    return swt_pass_t<double>(false, filt_len, f_lo, f_hi, dilation, sets, x, x_batch_stride, nullptr, nullptr, lo,
                              lo_batch_stride, hi, hi_batch_stride, batch, n, st);
}

int wt_swt_pass_inv(int dtype, int filt_len, const double* g_lo, const double* g_hi, int64_t dilation, int sets,
                    const void* const* lo, const int64_t* lo_batch_stride, const void* const* hi,
                    const int64_t* hi_batch_stride, void* const* y, const int64_t* y_batch_stride, int64_t batch,
                    int64_t n, void* stream) {
    int rc = swt_pass_check(dtype, filt_len, g_lo, g_hi, dilation, sets, batch, n);
    if (rc) return rc;
    if (batch == 0) return 0;
    if (!lo || !lo_batch_stride || !hi || !hi_batch_stride || !y || !y_batch_stride) return fail(WT_EINVAL, "NULL argument");
    for (int s = 0; s < sets; ++s)
        if (!lo[s] || !hi[s] || !y[s]) return fail(WT_EINVAL, "NULL band of set %d", s);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return swt_pass_t<float>(true, filt_len, g_lo, g_hi, dilation, sets, lo, lo_batch_stride, hi, hi_batch_stride,
                                 y, y_batch_stride, nullptr, nullptr, batch, n, st);
    return swt_pass_t<double>(true, filt_len, g_lo, g_hi, dilation, sets, lo, lo_batch_stride, hi, hi_batch_stride, y,
                              y_batch_stride, nullptr, nullptr, batch, n, st);
}

const char* wt_last_error(void) { return g_err; }

int wt_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) return cuda_fail(e, "cudaGetDeviceProperties");
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return 0;
}

int64_t wt_coeff_len(int64_t n, int filt_len) { return coeff_len(n, filt_len); }

size_t wt_dwt_workspace_bytes(int ndim, int dtype, int levels, int filt_len, int64_t batch, const int64_t* dims,
                              int inverse) {
    if (check_common(ndim, dtype, levels, filt_len, batch, dims) || levels == 0 || batch == 0) return 0;
    inverse &= 1;   // bit 1 is retired (include/wtb200.h)
    const int es = dtype == WT_F64 ? 8 : 4;
    if (dwt_route(inverse, ndim, es, levels, filt_len, batch, dims) != ROUTE_GENERAL) return 0;
    int64_t s1, s2;
    generic_scratch_elems(ndim, filt_len, levels, batch, dims, inverse, &s1, &s2);
    return (size_t)(s1 + s2) * es;
}

int wt_dwt_fwd(int ndim, int dtype, int mode, int levels, int filt_len, const double* dec_lo,
               const double* dec_hi, const void* x, int64_t batch, const int64_t* dims, const int64_t* x_strides,
               int64_t x_batch_stride, const wt_level* levels_desc, void* workspace, size_t workspace_bytes,
               void* stream) {
    int rc = check_common(ndim, dtype, levels, filt_len, batch, dims);
    if (rc) return rc;
    if (mode < WT_MODE_ZERO || mode > WT_MODE_SYMMETRIC) return fail(WT_EINVAL, "unknown boundary mode %d", mode);
    if (!dec_lo || !dec_hi || !x_strides) return fail(WT_EINVAL, "NULL argument");
    if (levels == 0 || batch == 0) return 0;
    if (!x || !levels_desc) return fail(WT_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return dwt_fwd_t<float>(ndim, mode, levels, filt_len, dec_lo, dec_hi, x, batch, dims, x_strides,
                                x_batch_stride, levels_desc, workspace, workspace_bytes, st);
    return dwt_fwd_t<double>(ndim, mode, levels, filt_len, dec_lo, dec_hi, x, batch, dims, x_strides,
                             x_batch_stride, levels_desc, workspace, workspace_bytes, st);
}

int wt_dwt_inv(int ndim, int dtype, int levels, int filt_len, const double* rec_lo, const double* rec_hi,
               void* y, int64_t batch, const int64_t* out_dims, const int64_t* y_strides, int64_t y_batch_stride,
               const wt_level* levels_desc, void* workspace, size_t workspace_bytes, void* stream) {
    int rc = check_common(ndim, dtype, levels, filt_len, batch, out_dims);
    if (rc) return rc;
    if (!rec_lo || !rec_hi || !y_strides) return fail(WT_EINVAL, "NULL argument");
    if (levels == 0 || batch == 0) return 0;
    if (!y || !levels_desc) return fail(WT_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return dwt_inv_t<float>(ndim, levels, filt_len, rec_lo, rec_hi, y, batch, out_dims, y_strides,
                                y_batch_stride, levels_desc, workspace, workspace_bytes, st);
    return dwt_inv_t<double>(ndim, levels, filt_len, rec_lo, rec_hi, y, batch, out_dims, y_strides,
                             y_batch_stride, levels_desc, workspace, workspace_bytes, st);
}

int wt_matrix_fwd(int dtype, int levels, int filt_len, const double* dec_lo, const double* dec_hi,
                  const int64_t* n, const int32_t* padded, int odd_mode, const int32_t* nb_top,
                  const int32_t* nb_bot, const int32_t* w_left, const int32_t* w_right, const void* blocks,
                  const void* x, int64_t batch, int64_t x_stride, void* const* hi_out, const int64_t* hi_stride,
                  void* lo_out, int64_t lo_stride, void* scratch, size_t scratch_bytes, int allow_fused, void* stream) {
    if (dtype != WT_F32 && dtype != WT_F64) return fail(WT_EINVAL, "dtype must be WT_F32 or WT_F64");
    if (levels < 1) return fail(WT_EINVAL, "levels must be >= 1");
    if (filt_len < 2 || filt_len > WT_MAX_FILT_LEN) return fail(WT_EUNSUPPORTED, "filter length %d", filt_len);
    if (odd_mode < WT_MODE_ZERO || odd_mode > WT_MODE_SYMMETRIC) return fail(WT_EINVAL, "unknown padding mode %d", odd_mode);
    if (!dec_lo || !dec_hi || !n || !padded || !nb_top || !nb_bot || !w_left || !w_right || !hi_out || !hi_stride)
        return fail(WT_EINVAL, "NULL argument");
    if (batch == 0) return 0;
    if (!x || !lo_out) return fail(WT_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return matrix_fwd_t<float>(levels, filt_len, dec_lo, dec_hi, n, padded, odd_mode, nb_top, nb_bot, w_left,
                                   w_right, blocks, x, batch, x_stride, hi_out, hi_stride, lo_out, lo_stride,
                                   scratch, scratch_bytes, allow_fused, st);
    return matrix_fwd_t<double>(levels, filt_len, dec_lo, dec_hi, n, padded, odd_mode, nb_top, nb_bot, w_left,
                                w_right, blocks, x, batch, x_stride, hi_out, hi_stride, lo_out, lo_stride, scratch,
                                scratch_bytes, allow_fused, st);
}

int wt_matrix_inv(int dtype, int levels, int filt_len, const double* rec_lo, const double* rec_hi,
                  const int64_t* n, const int64_t* next_len, const int32_t* nb_top, const int32_t* nb_bot,
                  const int32_t* w_left, const int32_t* w_right, const void* blocks, const void* lo_in,
                  int64_t lo_stride, const void* const* hi_in, const int64_t* hi_stride, int64_t batch, void* y,
                  int64_t y_stride, void* scratch, size_t scratch_bytes, int allow_fused, void* stream) {
    if (dtype != WT_F32 && dtype != WT_F64) return fail(WT_EINVAL, "dtype must be WT_F32 or WT_F64");
    if (levels < 1) return fail(WT_EINVAL, "levels must be >= 1");
    if (filt_len < 2 || filt_len > WT_MAX_FILT_LEN) return fail(WT_EUNSUPPORTED, "filter length %d", filt_len);
    if (!rec_lo || !rec_hi || !n || !next_len || !nb_top || !nb_bot || !w_left || !w_right || !hi_in || !hi_stride)
        return fail(WT_EINVAL, "NULL argument");
    if (batch == 0) return 0;
    if (!lo_in || !y) return fail(WT_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return matrix_inv_t<float>(levels, filt_len, rec_lo, rec_hi, n, next_len, nb_top, nb_bot, w_left, w_right,
                                   blocks, lo_in, lo_stride, hi_in, hi_stride, batch, y, y_stride, scratch,
                                   scratch_bytes, allow_fused, st);
    return matrix_inv_t<double>(levels, filt_len, rec_lo, rec_hi, n, next_len, nb_top, nb_bot, w_left, w_right,
                                blocks, lo_in, lo_stride, hi_in, hi_stride, batch, y, y_stride, scratch,
                                scratch_bytes, allow_fused, st);
}

int wt_matrix_axis_fwd(int dtype, int filt_len, const double* dec_lo, const double* dec_hi, int64_t n, int padded,
                       int odd_mode, int nb_top, int nb_bot, int w_left, int w_right, const void* blocks, const void* x,
                       int64_t outer, int64_t inner, int64_t x_outer_stride, int64_t x_axis_stride, void* y,
                       int64_t y_outer_stride, int64_t y_axis_stride, void* stream) {
    int rc = matrix_axis_check(dtype, filt_len, dec_lo, dec_hi, n, nb_top, nb_bot, w_left, w_right, blocks, x, y, outer, inner);
    if (rc) return rc;
    if (odd_mode < WT_MODE_ZERO || odd_mode > WT_MODE_SYMMETRIC) return fail(WT_EINVAL, "padding mode %d", odd_mode);
    const int64_t n_in = n - (padded ? 1 : 0);
    if (n_in < 1) return fail(WT_ESHAPE, "empty axis");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return matrix_axis_t<float>(false, filt_len, dec_lo, dec_hi, n, n_in, n, odd_mode, nb_top, nb_bot, w_left, w_right, blocks,
                                    x, outer, inner, x_outer_stride, x_axis_stride, y, y_outer_stride, y_axis_stride, st);
    return matrix_axis_t<double>(false, filt_len, dec_lo, dec_hi, n, n_in, n, odd_mode, nb_top, nb_bot, w_left, w_right, blocks,
                                 x, outer, inner, x_outer_stride, x_axis_stride, y, y_outer_stride, y_axis_stride, st);
}

int wt_matrix_axis_inv(int dtype, int filt_len, const double* rec_lo, const double* rec_hi, int64_t n, int64_t keep,
                       int nb_top, int nb_bot, int w_left, int w_right, const void* blocks, const void* x, int64_t outer,
                       int64_t inner, int64_t x_outer_stride, int64_t x_axis_stride, void* y, int64_t y_outer_stride,
                       int64_t y_axis_stride, void* stream) {
    int rc = matrix_axis_check(dtype, filt_len, rec_lo, rec_hi, n, nb_top, nb_bot, w_left, w_right, blocks, x, y, outer, inner);
    if (rc) return rc;
    if (keep < 0 || keep > n) return fail(WT_ESHAPE, "keep %lld of %lld samples", (long long)keep, (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == WT_F32)
        return matrix_axis_t<float>(true, filt_len, rec_lo, rec_hi, n, n, keep, WT_MODE_ZERO, nb_top, nb_bot, w_left, w_right, blocks,
                                    x, outer, inner, x_outer_stride, x_axis_stride, y, y_outer_stride, y_axis_stride, st);
    return matrix_axis_t<double>(true, filt_len, rec_lo, rec_hi, n, n, keep, WT_MODE_ZERO, nb_top, nb_bot, w_left, w_right, blocks,
                                 x, outer, inner, x_outer_stride, x_axis_stride, y, y_outer_stride, y_axis_stride, st);
}

int wt_tap_corr(int dtype, int filt_len, const void* coeff_lo, const void* coeff_hi, int64_t coeff_stride,
                const void* sig, int64_t sig_stride, int64_t rows, int64_t m, int64_t n, double* out, void* stream) {
    if (dtype != WT_F32 && dtype != WT_F64) return fail(WT_EINVAL, "dtype must be WT_F32 or WT_F64");
    if (filt_len < 2 || filt_len > WT_MAX_FILT_LEN) return fail(WT_EUNSUPPORTED, "filter length %d", filt_len);
    if (!out || rows < 0 || m < 0 || n < 0 || m >= (int64_t(1) << 30) || n >= (int64_t(1) << 31) - 2 * WT_MAX_FILT_LEN)
        return fail(WT_EINVAL, "bad argument");
    if (rows > 0 && m > 0 && (!coeff_lo || !coeff_hi || !sig)) return fail(WT_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = dtype == WT_F32
        ? launch_tap_corr<float>((const float*)coeff_lo, (const float*)coeff_hi, coeff_stride, (const float*)sig, sig_stride,
                                 rows, (int)m, (int)n, filt_len, out, st)
        : launch_tap_corr<double>((const double*)coeff_lo, (const double*)coeff_hi, coeff_stride, (const double*)sig,
                                  sig_stride, rows, (int)m, (int)n, filt_len, out, st);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if (e != cudaSuccess) return cuda_fail(e, "tap_corr_kernel");
    return 0;
}

uint64_t wt_launch_count(void) { return g_launches.load(); }
void wt_launch_count_reset(void) { g_launches.store(0); }

int wt_set_knob(const char* name, long long value) {
    const int k = knob_find(name);
    if (k < 0) return fail(WT_EINVAL, "unknown knob '%s'", name ? name : "(null)");
    knob_table().v[k].store(value, std::memory_order_relaxed);
    return 0;
}
int wt_unset_knob(const char* name) { return wt_set_knob(name, KNOB_UNSET); }
int wt_get_knob(const char* name, long long* value) {
    const int k = knob_find(name);
    if (k < 0) return fail(WT_EINVAL, "unknown knob '%s'", name ? name : "(null)");
    const long long v = knob_table().v[k].load(std::memory_order_relaxed);
    if (value) *value = v == KNOB_UNSET ? 0 : v;
    return v == KNOB_UNSET ? 0 : 1;
}

}  // extern "C"
