/*
 * wtb200.h -- C ABI of the B200-native fast wavelet transform (libwtb200.so).
 *
 * This is the drop-in boundary for the ONE hot path of v0lta/PyTorch-Wavelet-Toolbox
 * (ptwt): the multi-level analysis / synthesis filter bank and the boundary-filter
 * matrix FWT.  ptwt has no FFI of its own (it is pure Python that calls torch ops);
 * each entry point below therefore names the reference *Python* body it replaces:
 *
 *   wt_dwt_fwd      <- the level loop of wavedec / wavedec2 / wavedec3
 *                      src/ptwt/conv_transform.py:133-141   (F.pad -> conv1d(stride=2) -> split)
 *                      src/ptwt/conv_transform_2.py:142-149 (F.pad -> conv2d(stride=2) -> split)
 *                      src/ptwt/conv_transform_3.py:122-141 (F.pad -> conv3d(stride=2) -> split)
 *   wt_dwt_inv      <- the level loop of waverec / waverec2 / waverec3
 *                      src/ptwt/conv_transform.py:184-199   (stack -> conv_transpose1d -> crop)
 *                      src/ptwt/conv_transform_2.py:208-249
 *                      src/ptwt/conv_transform_3.py:191-249
 *   wt_matrix_fwd   <- MatrixWavedec.__call__ level loop, src/ptwt/matmul_transform.py:409-425
 *                      (odd-length pad -> torch.sparse.mm(A_level, lo) -> split)
 *   wt_matrix_inv   <- MatrixWaverec.__call__ level loop, src/ptwt/matmul_transform.py:682-699
 *                      (cat -> torch.sparse.mm(S_level, .) -> trim)
 *   wt_matrix_axis_fwd / wt_matrix_axis_inv
 *                   <- the per-axis products of the separable MatrixWavedec2/3 and MatrixWaverec2/3,
 *                      src/ptwt/matmul_transform_2.py:514-531, :797-806; matmul_transform_3.py:255-262, :476-479
 *
 * Conventions
 *   - plain C, no C++ / torch types; every function returns 0 on success, a negative
 *     WT_E* code for a bad argument, or a positive cudaError_t.  wt_last_error()
 *     returns a thread-local message for the last failure on this thread.
 *   - all device buffers are owned by the caller (PyTorch's caching allocator on the
 *     Python side).  The library never allocates or frees device memory in the
 *     device-pointer entry points, never synchronises the device, and keeps no
 *     reference to any argument after it returns.  Work is enqueued on `stream`
 *     (a cudaStream_t passed as void*).
 *   - process-wide state the library DOES keep: (1) one auxiliary non-blocking stream and two events per
 *     device, created on first use and never destroyed: large 2-D analyses (batch >= 16, >= 2^27 samples,
 *     >= 2 levels) run the second half of the batch on it, forked from / joined back into `stream` with
 *     those events, so the call still behaves as if everything ran in `stream` order (no host
 *     synchronisation; disabled while `stream` is being captured into a CUDA graph, or with the switch
 *     NO_AUX_STREAM); (2) the per-kernel dynamic shared-memory opt-in (set once per device and kernel);
 *     (3) the launch counter and the tuning switches at the end of this header.
 *   - filter taps are HOST arrays of double in PyWavelets order (un-flipped dec_lo /
 *     dec_hi / rec_lo / rec_hi, reference src/ptwt/_util.py:95-126); they are rounded
 *     to the compute dtype inside and travel as kernel parameters, so concurrent
 *     streams may use different wavelets.
 *   - extents are ordered slow -> fast (dims[ndim-1] is the contiguous axis);
 *     strides are in ELEMENTS.
 *   - sub-band index k in [0, 2^ndim): k = sum_a hi(a) << (ndim-1-a), axis 0 = slowest,
 *     hi(a) = 1 when the high-pass filter was applied along axis a.
 *       3-D: k = 0..7 = lll, llh, lhl, lhh, hll, hlh, hhl, hhh with the first letter on the
 *            slowest axis -- the reference's own order (src/ptwt/_util.py:926-934), i.e.
 *            keys aad, ada, add, daa, dad, dda, ddd for k = 1..7
 *            (src/ptwt/conv_transform_3.py:131-141).
 *       2-D: k = 1 is lo_H hi_W (reference "hl" = vertical), k = 2 is hi_H lo_W (reference
 *            "lh" = horizontal), k = 3 diagonal (src/ptwt/_util.py:901-905,
 *            src/ptwt/conv_transform_2.py:145-149).
 *       1-D: k = 1 is the detail band.
 */
#ifndef WTB200_H
#define WTB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WT_VERSION 100 /* 0.1.0 */

/* dtype */
#define WT_F32 0
#define WT_F64 1

/* boundary modes (ptwt BoundaryMode, src/ptwt/constants.py:85; torch names in
 * src/ptwt/_util.py:36-44) */
#define WT_MODE_ZERO 0      /* "zero"      -> F.pad constant 0            */
#define WT_MODE_CONSTANT 1  /* "constant"  -> F.pad replicate             */
#define WT_MODE_REFLECT 2   /* "reflect"   -> F.pad reflect (no edge repeat) */
#define WT_MODE_PERIODIC 3  /* "periodic"  -> F.pad circular              */
#define WT_MODE_SYMMETRIC 4 /* "symmetric" -> _pad_symmetric (edge repeated) */

/* error codes (negative) */
#define WT_EINVAL (-1)   /* malformed argument                                  */
#define WT_ESHAPE (-2)   /* extents inconsistent with the reference's formulae  */
#define WT_EWORKSPACE (-3) /* workspace too small                               */
#define WT_EUNSUPPORTED (-4)

#define WT_MAX_NDIM 3
#define WT_MAX_FILT_LEN 128

/* One decomposition level of the padded transform, as laid out by the caller.
 * dims[] are the coefficient extents of THIS level; they must equal
 * floor((n_prev + L - 1) / 2) per axis (reference _get_pad, src/ptwt/_util.py:198-228).
 * detail bands k = 1 .. 2^ndim-1 live at  details + (k-1)*band_stride ;
 * the approximation band (k = 0) lives at `approx` (the returned cA for the coarsest
 * level, caller-provided scratch for the others).
 * SCRATCH SEMANTICS (analysis): the `approx` buffers of all but the coarsest level must hold
 * `batch` items, but their contents are UNSPECIFIED on return -- the library processes the
 * batch in chunks and reuses the first few item slots so that the intermediate approximations
 * stay resident in L2 and never travel to HBM.  A caller that wants cA_l of an intermediate
 * level runs a transform with `levels = l`. */
typedef struct wt_level {
    void* details;
    void* approx;
    int64_t dims[WT_MAX_NDIM];
    int64_t strides[WT_MAX_NDIM];        /* element strides inside one detail band */
    int64_t approx_strides[WT_MAX_NDIM]; /* element strides inside the approximation band */
    int64_t details_batch_stride;
    int64_t band_stride;
    int64_t approx_batch_stride;
} wt_level;

int wt_version(void);
const char* wt_last_error(void);

/* Number of SMs / whether a usable sm_100 device is current.  Returns 0 and fills
 * the outputs, or a cudaError_t. */
int wt_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* Coefficient extent of one level along one axis: floor((n + L - 1) / 2) for even L
 * (general L: (n + padl + padr - L)/2 + 1 with the reference's pad amounts). */
int64_t wt_coeff_len(int64_t n, int filt_len);

/* Bytes of workspace wt_dwt_fwd / wt_dwt_inv need for the given problem, exactly: 0 when the call runs on the fused
 * kernels, which need none, else the requirement of the general path.  Which of the two runs a call depends on its
 * arguments here alone, so this query and the transform always agree.  inverse: 0 analysis, 1 synthesis; bit 1 is
 * retired and ignored (2 and 3 give what 0 and 1 give).  dims are the extents of x (analysis) or of y (synthesis).
 * Arguments the transform rejects give 0. */
size_t wt_dwt_workspace_bytes(int ndim, int dtype, int levels, int filt_len, int64_t batch,
                              const int64_t* dims, int inverse);

/* Multi-level analysis.  x is [batch, dims...] with element strides x_strides[ndim] and
 * batch stride x_batch_stride.  levels_desc[0] is the FINEST level (level 1),
 * levels_desc[levels-1] the coarsest.  mode: WT_MODE_*.
 * For ndim >= 2, x, every detail band and every approximation must have an innermost stride of 1 (WT_EINVAL).
 * A call that returns WT_EINVAL, WT_ESHAPE or WT_EWORKSPACE (wt_dwt_inv alike) has launched nothing; only a CUDA
 * error can come back after launches were made. */
int wt_dwt_fwd(int ndim, int dtype, int mode, int levels, int filt_len,
               const double* dec_lo, const double* dec_hi,
               const void* x, int64_t batch, const int64_t* dims,
               const int64_t* x_strides, int64_t x_batch_stride,
               const wt_level* levels_desc,
               void* workspace, size_t workspace_bytes, void* stream);

/* Multi-level synthesis: consumes levels_desc[levels-1] (coarsest; its `approx` is the
 * input cA) down to levels_desc[0]; intermediate reconstructions are written to the
 * `approx` scratch of the next finer level; the final signal goes to y.
 * out_dims[] are the extents of y; per axis they must be 2*c - L + 2 of level 1, and
 * for every level the reconstructed extent may exceed the next finer level's extent
 * by exactly one sample (the reference trims it, src/ptwt/_util.py:231-244). */
int wt_dwt_inv(int ndim, int dtype, int levels, int filt_len,
               const double* rec_lo, const double* rec_hi,
               void* y, int64_t batch, const int64_t* out_dims,
               const int64_t* y_strides, int64_t y_batch_stride,
               const wt_level* levels_desc,
               void* workspace, size_t workspace_bytes, void* stream);

/* Boundary-filter matrix FWT (MatrixWavedec).  Per level l (0 = finest):
 *   n[l]        even length the level operator acts on (after the optional one-sample
 *               pad of an odd input, reference matmul_transform.py:334-341),
 *   padded[l]   1 if the level input had n[l]-1 samples and is extended by one sample
 *               using odd_mode (WT_MODE_*),
 *   nb_top[l], nb_bot[l]  number of orthogonalised boundary rows at the top / bottom of
 *               EACH half (lo and hi); nb = nb_top + nb_bot rows per half, top rows first,
 *   w_left[l], w_right[l] column support of those rows: the first w_left and the last
 *               w_right columns (the QR leaves round-off sized entries of a top row in the
 *               right corner and vice versa; they are kept, like the reference keeps them),
 *   blocks      device array, compute dtype; for each level in order: lo_left
 *               [nb x w_left], lo_right [nb x w_right], hi_left, hi_right (row-major).
 * x is [batch, n0] contiguous rows (n0 = n[0] - padded[0]).  hi_out[l] receives the detail
 * of level l ([batch, n[l]/2], row stride hi_stride[l]); lo_out the coarsest approximation.
 * scratch must hold 2 * batch * (n[0]/2) elements.
 * allow_fused: non-zero lets consecutive unpadded levels run in one kernel that keeps the approximation
 * in shared memory; that kernel cannot reach the cross-corner entries of the boundary rows (a top row's
 * entries in the right window and vice versa), so the caller sets it only when those entries are
 * negligible (the Python layer: <= 1e-13, true for float64 operators). */
int wt_matrix_fwd(int dtype, int levels, int filt_len,
                  const double* dec_lo, const double* dec_hi,
                  const int64_t* n, const int32_t* padded, int odd_mode,
                  const int32_t* nb_top, const int32_t* nb_bot,
                  const int32_t* w_left, const int32_t* w_right, const void* blocks,
                  const void* x, int64_t batch, int64_t x_stride,
                  void* const* hi_out, const int64_t* hi_stride,
                  void* lo_out, int64_t lo_stride,
                  void* scratch, size_t scratch_bytes, int allow_fused, void* stream);

/* MatrixWaverec: the mirror image.  Taps are the FLIPPED reconstruction filters'
 * source, i.e. pass rec_lo / rec_hi un-flipped (reference flips them itself,
 * matmul_transform.py:110-112); blocks are the boundary rows of S^T per level with the
 * same layout as above.  next_len[l] is the number of samples kept from the level-l
 * reconstruction (n[l] or n[l]-1, reference matmul_transform.py:691-699).  allow_fused as in
 * wt_matrix_fwd: non-zero lets groups of untrimmed levels run as one kernel that keeps the
 * intermediate approximations on chip and drops the cross-corner round-off entries. */
int wt_matrix_inv(int dtype, int levels, int filt_len,
                  const double* rec_lo, const double* rec_hi,
                  const int64_t* n, const int64_t* next_len,
                  const int32_t* nb_top, const int32_t* nb_bot,
                  const int32_t* w_left, const int32_t* w_right, const void* blocks,
                  const void* lo_in, int64_t lo_stride,
                  const void* const* hi_in, const int64_t* hi_stride,
                  int64_t batch, void* y, int64_t y_stride,
                  void* scratch, size_t scratch_bytes, int allow_fused, void* stream);

/* One level of the 1-D boundary-wavelet operator along an arbitrary axis of a [outer, n, inner]
 * tensor whose inner index is contiguous -- the building block of the SEPARABLE 2-D / 3-D matrix
 * transforms (reference src/ptwt/matmul_transform_2.py:514-531 "batch_mm(fwt_col_matrix, ...)",
 * src/ptwt/matmul_transform_3.py:255-262 "_batch_dim_mm(mat, lll, dim)").
 *   analysis:  x [outer, n - padded, inner] -> y [outer, n, inner], low-pass rows 0..n/2-1 then
 *              high-pass rows n/2..n-1 along the axis (the reference's "A x, then split");
 *              padded = 1 appends one sample along the axis per odd_mode first.
 *   synthesis: x [outer, n, inner] (lo | hi along the axis) -> y [outer, keep, inner], keep <= n.
 * blocks: device array, the level's boundary rows as in wt_matrix_fwd / wt_matrix_inv
 * (lo_left, lo_right, hi_left, hi_right).  Strides are in elements. */
int wt_matrix_axis_fwd(int dtype, int filt_len, const double* dec_lo, const double* dec_hi,
                       int64_t n, int padded, int odd_mode,
                       int nb_top, int nb_bot, int w_left, int w_right, const void* blocks,
                       const void* x, int64_t outer, int64_t inner,
                       int64_t x_outer_stride, int64_t x_axis_stride,
                       void* y, int64_t y_outer_stride, int64_t y_axis_stride, void* stream);

int wt_matrix_axis_inv(int dtype, int filt_len, const double* rec_lo, const double* rec_hi,
                       int64_t n, int64_t keep,
                       int nb_top, int nb_bot, int w_left, int w_right, const void* blocks,
                       const void* x, int64_t outer, int64_t inner,
                       int64_t x_outer_stride, int64_t x_axis_stride,
                       void* y, int64_t y_outer_stride, int64_t y_axis_stride, void* stream);

/* Gradient of one transform level with respect to the filter taps along the contiguous axis (learnable wavelets:
 * the reference's filters are nn.Parameters, src/ptwt/wavelets_learnable.py:167-189, and enter its convolutions through
 * src/ptwt/_util.py:129-141).  out[k * L + t] = sum_{r, i} coeff_k[r, i] * sig[r, 2 i + t + 2 - L]  (k = 0 lo, 1 hi;
 * samples outside [0, n) count as zero), accumulated in float64 into the DEVICE array out[2 * L] (zeroed here).
 *   analysis level (zero extension of the explicitly extended input x):  coeff = upstream gradient of the band,
 *       sig = x;   d dec_k[m] = out[k][L - 1 - m]
 *   synthesis level: coeff = the band, sig = upstream gradient of the cropped output;  d rec_k[t] = out[k][t]
 * rows of coeff_* are coeff_stride elements apart (m coefficients each), rows of sig sig_stride apart (n samples). */
int wt_tap_corr(int dtype, int filt_len, const void* coeff_lo, const void* coeff_hi, int64_t coeff_stride,
                const void* sig, int64_t sig_stride, int64_t rows, int64_t m, int64_t n, double* out, void* stream);

/* Stationary wavelet transform (ptwt.swt / ptwt.iswt), periodic extension, 1-D along contiguous rows of n samples.
 *   wt_swt_fwd  <- the level loop of swt,  src/ptwt/stationary_transform.py:96-106
 *                  (_circular_pad -> conv1d(dilation 2^(j-1)) -> split)
 *   wt_swt_inv  <- the level loop of iswt, src/ptwt/stationary_transform.py:139-151
 *                  (stack -> _circular_pad -> conv_transpose1d(dilation 2^(j-1), groups 2) -> mean)
 * Taps are host doubles in WINDOW order (not PyWavelets order), with any scale folded in; hl = L/2 - 1, L even:
 *   analysis   c_lo/hi[i] = sum_m f_lo/hi[m] a[(i + d (m - hl)) mod n]        swt: f = dec[::-1]
 *   synthesis  y[i] = sum_m g_lo[m] a[(i + d (hl - m)) mod n] + g_hi[m] c[same]  iswt: g = 0.5 * rec
 * The two forms are adjoint: analysis with f = 0.5 rec is the gradient of synthesis, synthesis with g = dec[::-1]
 * the gradient of analysis.
 * wt_swt_fwd writes [cA_J, cD_J, ..., cD_1] as bands of `out` (band b at out + b * out_band_stride, batch item at
 * + item * out_batch_stride); wt_swt_inv reads cA_J from `approx` and cD_j from details + (levels - j) * band stride.
 * tables: NULL, or `levels` device pointers (level j at [j-1]); a non-NULL entry replaces the periodic index of that
 * level by a CSR table: int32 rowptr[n + 1], then from int32 offset 2 * ((n + 2) / 2) the (source index, tap) int32
 * pairs of every output (the reference's _circular_pad when a pad exceeds n, or its transpose for the adjoint).
 * workspace: wt_swt_workspace_bytes() bytes (0 when the levels run in one launch). */
size_t wt_swt_workspace_bytes(int dtype, int levels, int filt_len, int64_t batch, int64_t n,
                              const void* const* tables, int inverse);
int wt_swt_fwd(int dtype, int levels, int filt_len, const double* f_lo, const double* f_hi, const void* x,
               int64_t batch, int64_t n, int64_t x_batch_stride, void* out, int64_t out_batch_stride,
               int64_t out_band_stride, const void* const* tables, void* workspace, size_t workspace_bytes,
               void* stream);
int wt_swt_inv(int dtype, int levels, int filt_len, const double* g_lo, const double* g_hi, const void* approx,
               int64_t approx_batch_stride, const void* details, int64_t details_batch_stride,
               int64_t details_band_stride, int64_t batch, int64_t n, void* y, int64_t y_batch_stride,
               const void* const* tables, void* workspace, size_t workspace_bytes, void* stream);

/* 2-D stationary transform (swt2 / iswt2; the reference has no such function, PyWavelets' swt2 with trim_approx=True,
 * norm=False), built from one level of ONE axis per call.  A pass filters `batch` contiguous rows of n samples with
 * the periodic forms above at dilation `dilation` (in samples) instead of 2^(j-1):
 *   along the contiguous axis of [.., H, W] planes: rows of n = W samples (batch = planes * H), dilation d = 2^(j-1);
 *   along the other axis: each dense H x W plane (row pitch W) is ONE row of n = H W samples at dilation d W, which
 *   wraps d rows modulo H and keeps the column.
 * `sets` (1 or 2) band sets run in one call; each array holds one pointer / batch stride per set.
 *   wt_swt_pass_fwd: x[s] -> lo[s] (f_lo), hi[s] (f_hi)          wt_swt_pass_inv: y[s] = synthesis of lo[s], hi[s]
 * The two sets take one launch when the pass runs on tiles, one launch each otherwise.  A pass needs no workspace.
 * wt_swt2_workspace_bytes: the buffers the caller's level cascade keeps between passes for `levels` levels of `batch`
 * H x W planes, each dense: the two bands of the contiguous-axis pass, plus one approximation plane when levels > 1.
 * Arguments outside the transform's domain give 0.
 * wt_swt_pass_plan: how a pass of rows of n samples at `dilation` runs, without running it.  Returns 1 for tiles and
 * fills tile[4] = {D, M, C, R}: the row seen as M rows of D samples, C rows owned per tile (C == M: whole columns, no
 * halo), R columns per tile; returns 0 for the per-level kernel (straight from global memory), or a WT_E* code. */
int wt_swt_pass_plan(int dtype, int inverse, int filt_len, int64_t n, int64_t dilation, int64_t* tile);
size_t wt_swt2_workspace_bytes(int dtype, int levels, int64_t batch, int64_t h, int64_t w);
int wt_swt_pass_fwd(int dtype, int filt_len, const double* f_lo, const double* f_hi, int64_t dilation, int sets,
                    const void* const* x, const int64_t* x_batch_stride, void* const* lo, const int64_t* lo_batch_stride,
                    void* const* hi, const int64_t* hi_batch_stride, int64_t batch, int64_t n, void* stream);
int wt_swt_pass_inv(int dtype, int filt_len, const double* g_lo, const double* g_hi, int64_t dilation, int sets,
                    const void* const* lo, const int64_t* lo_batch_stride, const void* const* hi,
                    const int64_t* hi_batch_stride, void* const* y, const int64_t* y_batch_stride, int64_t batch,
                    int64_t n, void* stream);

/* Continuous wavelet transform (ptwt.cwt), src/ptwt/continuous_transform.py:103-137 (per scale: FFT of the
 * filter and the data, product, inverse FFT, diff, crop; then stack), as uniformly partitioned overlap-save in
 * float64 (csrc/cwt.cuh).  Hop H = 2^(fft_log2 - 1), FFT size F = 2H, fft_log2 in 6..12; nb = ceil(n / H).
 * A channel is one complex-wavelet scale (complex_out != 0) or a pair of real-wavelet scales whose taps are packed
 * as real + i * imaginary (complex_out == 0).  Channel c's FIR is  y_c[t] = sum_j taps_c[j] x[t + d_c H + e_c - j]
 * (0 <= e_c < H); its taps are cut into P_c parts of H.
 *   wt_cwt_filter_spectra: spectra[r] = FFT(taps[r] zero-padded to F) / F, in bit-reversed bin order, for `parts`
 *                          rows of H complex128 taps (all device buffers; twiddles[k] = exp(-2 pi i k / F), k < F / 2,
 *                          complex128).
 *   wt_cwt_fwd: meta = device int32 [channels][6] = {first part row, P_c, d_c, scale s1, scale s2 or -1, e_c};
 *               x [batch] rows of n samples (WT_F32/WT_F64, unit stride) -> float64 (complex_out == 0: s1 gets the
 *               real part, s2 the imaginary part) or complex128 coefficients at
 *               out + s * out_scale_stride + item * out_batch_stride + t (strides in elements of the output type).
 *   wt_cwt_adj: the adjoint, gx[item][m] = Re sum_c sum_t conj(taps_c[t + d_c H + e_c - m]) gy_c[t], gy laid out like
 *               wt_cwt_fwd's output, gx in `dtype`.
 * workspace: wt_cwt_workspace_bytes() bytes (the batch runs in chunks that fit a fixed budget, two launches each). */
size_t wt_cwt_workspace_bytes(int fft_log2, int64_t batch, int64_t n, int64_t channels, int adjoint);
int wt_cwt_filter_spectra(int fft_log2, int64_t parts, const void* taps, const void* twiddles, void* spectra,
                          void* stream);
int wt_cwt_fwd(int dtype, int fft_log2, int64_t channels, const int32_t* meta, const void* spectra,
               const void* twiddles, int complex_out, const void* x, int64_t batch, int64_t n, int64_t x_batch_stride,
               void* out, int64_t out_scale_stride, int64_t out_batch_stride, void* workspace, size_t workspace_bytes,
               void* stream);
int wt_cwt_adj(int dtype, int fft_log2, int64_t channels, const int32_t* meta, const void* spectra,
               const void* twiddles, int complex_out, const void* gy, int64_t out_scale_stride,
               int64_t out_batch_stride, int64_t batch, int64_t n, void* gx, int64_t gx_batch_stride,
               void* workspace, size_t workspace_bytes, void* stream);

/* Counters for bench.py's gpu_launches claim: kernels launched by this library on this
 * process since the last reset. */
uint64_t wt_launch_count(void);
void wt_launch_count_reset(void);

/* Tuning / test switches (NOT part of the drop-in surface).  Every switch is also read ONCE from the
 * environment variable WTB200_<NAME> when the library is first used; no transform call reads the environment.
 * Names: DISABLE_FUSED (general kernels only), NO_WPAIR (one launch per 2-D analysis level), WPAIR_SEG,
 * WPAIR_MIN, WPAIR_DEEP, FUSE2 (opt-in two-level 2-D strip kernel), CHUNK, STREAMS, NO_AUX_STREAM, NO_DMMA, MATF_K, MATI_K, ... (csrc/knobs.cuh).
 * wt_set_knob returns 0 or WT_EINVAL for an unknown name; wt_get_knob returns 1 and the value when the switch
 * is set, 0 when it is not, WT_EINVAL for an unknown name. */
int wt_set_knob(const char* name, long long value);
int wt_unset_knob(const char* name);
int wt_get_knob(const char* name, long long* value);

#ifdef __cplusplus
}
#endif
#endif /* WTB200_H */
