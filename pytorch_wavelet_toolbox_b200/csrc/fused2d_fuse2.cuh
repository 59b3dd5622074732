// fused2d_fuse2.cuh -- TWO consecutive 2-D analysis levels (float32, even filter length <= 8) in one launch of
// the strip kernel, so the first level's approximation band never reaches HBM.
//
// With one launch per level that band is written by level l and read back by level l+1.  Here a CTA runs
// fwd2d_strip_f32_kernel's level-l pipeline (TMA ring of input chunks, row pass, column pass) over 64
// approximation columns and hands each chunk's 16 approximation rows to level l+1 through shared memory:
//
//   * strip: a CTA owns TW2 = 28 level-(l+1) columns.  Their windows read approximation columns
//     [2 X0 - HALO, 2 X0 + 56); the CTA computes [2 X0 - 8, 2 X0 + 56) (left halo rounded to 16 bytes) and
//     stores the level-l details of the 56 columns it owns only;
//   * per chunk: the level-l column pass writes the approximation rows to a buffer; edge strips overwrite its
//     out-of-range columns with the boundary extension of the approximation band (the sources lie in the
//     strip: the last strip is moved left when needed); a level-(l+1) row pass turns each buffered row into one
//     low-pass and one high-pass line of a 32-line ring indexed by (row & 31); a level-(l+1) column pass reads L
//     lines per output row -- above and below the band it reads the line of the extension source row -- and
//     stores the four bands with 128-bit stores;
//   * segments: level-(l+1) rows are processed 8 per chunk, lagging one chunk behind level l; chunk 0 only fills
//     the rings (the segment restart, 16 approximation rows).  The bottom segments start early enough that the
//     extension sources of the last rows are computed by the CTA itself.
//
// Every output is formed by the same per-output FMA sequence as with one strip-kernel launch per level
// (row_filter, col_filter2x4 order) from the same float32 approximation values, so the result is bit-identical.
//
// Algorithmic bytes: 4 B * (H*W read + 3*Mh1*Mw1 + 4*Mh2*Mw2 written).  Opt-in with FUSE2=1 (see try_fuse2).
// Resources (sm_90a, L = 8): 80 registers, no spills, 74.5 KB dynamic shared memory, 3 CTAs (24 warps) per SM.
#pragma once

#include "fused2d.cuh"

namespace wtb {

struct Fuse2Params {
    const float* x;              // level-l input [batch, H, W]
    int64_t x_bs, x_rs;
    float* d1[3];                // level-l detail bands k = 1, 2, 3
    int64_t d1_bs[3], d1_rs[3];
    float* o2[4];                // level-(l+1) bands k = 0 (approximation), 1, 2, 3
    int64_t o2_bs[4], o2_rs[4];
    int H, W, Mh1, Mw1, Mh2, Mw2;
    int seg_rows;                // level-(l+1) rows per segment (multiple of 8)
    int mode, batch0;
    float2 pl[4], ph[4], bl[8], bh[8];   // paired taps, see row_filter / col_filter2x4
};

template <int L>
struct Fuse2Geom {
    using G1 = Fwd2dGeom<L, 64, 4>;                 // level l: the float32 strip kernel's geometry
    static constexpr int TW1 = 64, HALO = L - 2, H2 = HALO / 2;
    static constexpr int HL = 8;                    // approximation columns left of the first owned window
    static constexpr int OFF2 = HL - HALO;
    static constexpr int TW2 = (TW1 - HL) / 2;      // level-(l+1) columns per strip
    static constexpr int NG2 = TW2 / 4;             // 4-column groups per level-(l+1) row
    static constexpr int CH = G1::CH;               // approximation rows per chunk
    static constexpr int CH2 = CH / 2;              // level-(l+1) rows per chunk
    static constexpr int AP = TW1 + 4;              // pitch of the approximation buffer
    static constexpr int RING2 = 32, LP = 32;       // level-(l+1) line ring: lines, pitch
    static constexpr int MIR = L + 2;
    static constexpr int NT = G1::NTHREADS;
    static constexpr size_t SMEM = 2 * G1::stage_bytes(4) + 2 * (size_t)(G1::RING + MIR) * G1::MP * 4 +
                                   (size_t)CH * AP * 4 + 2 * (size_t)RING2 * LP * 4 + 64;
    static_assert(L % 2 == 0 && L >= 2 && L <= 8, "fuse2 kernel: even filter length <= 8");
    static_assert(HALO <= HL && 2 * TW2 + HL == TW1 && TW2 % 4 == 0 && TW2 <= LP, "strip geometry");
    static_assert(2 * CH * NG2 <= NT && 4 * CH2 * NG2 <= NT, "one level-(l+1) item per thread");
    // the ring holds the last two chunks' lines: the windows of the chunk's outputs (CH + HALO lines) and, at
    // the bottom of the band, the extension sources (rows >= Mh1 - L) for L <= 9
    static_assert(RING2 == 2 * CH && RING2 >= CH + HALO && (RING2 & (RING2 - 1)) == 0, "line ring");
};

template <int L>
__global__ void __launch_bounds__(Fuse2Geom<L>::NT, 3)
fwd2d_fuse2_f32_kernel(const __grid_constant__ Fuse2Params p, const __grid_constant__ CUtensorMap tmap) {
    using F = Fuse2Geom<L>;
    using Gm = typename F::G1;
    constexpr int HAL = Gm::HAL, HALO = Gm::HALO, CH = Gm::CH, IN_ROWS = Gm::IN_ROWS, SW = Gm::SW;
    constexpr int MP = Gm::MP, RING = Gm::RING, NT = F::NT, MIR = F::MIR, NCG = F::TW1 / 4;
    constexpr int TW1 = F::TW1, TW2 = F::TW2, NG2 = F::NG2, CH2 = F::CH2, AP = F::AP, LP = F::LP, H2 = F::H2;
    constexpr int RMASK = F::RING2 - 1;
    static_assert(NT == 2 * (CH / 2) * NCG, "one level-l column-pass item per thread");

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_in = reinterpret_cast<float*>(smem_raw);       // [2][IN_ROWS][SW]
    float* s_lo = s_in + 2 * IN_ROWS * SW;                  // [RING + MIR][MP]
    float* s_hi = s_lo + (RING + MIR) * MP;
    float* s_a = s_hi + (RING + MIR) * MP;                  // [CH][AP] approximation rows of the chunk
    float* s_l2 = s_a + CH * AP;                            // [RING2][LP] level-(l+1) low-pass lines
    float* s_h2 = s_l2 + F::RING2 * LP;                     // [RING2][LP] level-(l+1) high-pass lines
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_h2 + F::RING2 * LP);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = p.batch0 + blockIdx.z;
    const int X0n = blockIdx.x * TW2;                       // first level-(l+1) column this strip stores
    const int X0 = min(X0n, (p.Mw1 / 2) & ~3);              // first level-(l+1) column computed
    const int A0 = 2 * X0 - F::HL;                          // first approximation column computed
    const int Y0 = blockIdx.y * p.seg_rows;
    if (Y0 >= p.Mh2) return;
    const int Y1 = min(Y0 + p.seg_rows, p.Mh2);
    const int Yb = min(Y0 - CH2, (p.Mh1 - L - H2) >> 1);    // level-(l+1) row of chunk 0
    const int yb = 2 * Yb;                                  // approximation row of chunk 0
    const int c_in0 = 2 * A0 - HAL;
    const int r_in0 = 2 * yb;
    const int nchunks = (Y1 - Yb + CH2 - 1) / CH2;
    const int c_need1 = 2 * min(A0 + TW1, p.Mw1);
    const int r_need1 = 2 * min(yb + CH * nchunks, p.Mh1);

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
    const float* __restrict__ xb = p.x + (int64_t)b * p.x_bs;

    // level-l column pass: (lo|hi array, row pair, 4-column group).  The lo array yields the approximation
    // (to s_a) and band 2; the hi array bands 1 and 3.
    const int half = tid / (NT / 2);
    const int rem = tid - half * (NT / 2);
    const int rp = rem / NCG, cg = rem - rp * NCG;
    const int yl = 2 * rp;
    const float* cring = (half ? s_hi : s_lo) + 4 * cg;
    const int gx = A0 + 4 * cg;
    const bool own1 = gx >= 2 * X0n && gx < min(2 * (X0n + TW2), p.Mw1);
    const int own_y0 = 2 * Y0, own_y1 = min(2 * Y1, p.Mh1);
    float* const pL = half ? p.d1[0] + (int64_t)b * p.d1_bs[0] + gx : nullptr;
    float* const pH = p.d1[1 + half] + (int64_t)b * p.d1_bs[1 + half] + gx;
    const int64_t rsL = p.d1_rs[0], rsH = p.d1_rs[1 + half];

    // edge strips: the approximation columns outside [0, Mw1) are replaced by their extension sources
    const bool edge = A0 < 0 || A0 + TW1 > p.Mw1;

    int ring_base = 0;
    for (int c = 0; c < nchunks; ++c) {
        const int stage = c & 1;
        float* tile = s_in + stage * IN_ROWS * SW;
        const int r_base = r_in0 + c * IN_ROWS;

        mbar_wait(&bars[stage], (uint32_t)((c >> 1) & 1));
        if (p.mode != WT_MODE_ZERO)
            patch_tile_f32<SW, IN_ROWS, NT>(tile, xb, p.x_rs, p.H, p.W, p.mode, c_in0, r_base, c_need1, r_need1, tid);

        strip_row_pass_f32<L, TW1>(tile, s_lo, s_hi, ring_base, p.pl, p.ph, lane, warp);
        __syncthreads();

        if (tid == 0 && c + 2 < nchunks) {
            fence_proxy_async();
            mbar_expect_tx(&bars[stage], (uint32_t)Gm::stage_bytes(4));
            tma_load_3d(tile, &tmap, &bars[stage], c_in0, r_in0 + (c + 2) * IN_ROWS, b);
        }

        // ---- level-l column pass: details to HBM, the approximation to s_a ------------------------------
        {
            int row0 = ring_base + 2 * yl - HALO;
            if (row0 < 0) row0 += RING;
            else if (row0 >= RING) row0 -= RING;
            float2 accL[2][2], accH[2][2];
            col_filter2x4<L>(cring + row0 * MP, MP, p.bl, p.bh, accL, accH);
            const int gyc = yb + c * CH + yl;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float4 vL = make_float4(accL[r][0].x, accL[r][0].y, accL[r][1].x, accL[r][1].y);
                const float4 vH = make_float4(accH[r][0].x, accH[r][0].y, accH[r][1].x, accH[r][1].y);
                if (!half) *reinterpret_cast<float4*>(s_a + (yl + r) * AP + 4 * cg) = vL;
                const int gy = gyc + r;
                if (own1 && gy >= own_y0 && gy < own_y1) {
                    if (half) *reinterpret_cast<float4*>(pL + (int64_t)gy * rsL) = vL;
                    *reinterpret_cast<float4*>(pH + (int64_t)gy * rsH) = vH;
                }
            }
        }
        __syncthreads();

        if (edge) {
            float v[CH * TW1 / NT];
#pragma unroll
            for (int i = 0; i < CH * TW1 / NT; ++i) {
                const int idx = tid + i * NT, r = idx / TW1, q = idx - r * TW1;
                const int col = A0 + q;
                v[i] = s_a[r * AP + q];
                if (col < 0 || col >= p.Mw1) {
                    const int src = ext_index32(col, p.Mw1, p.mode), s = src - A0;
                    v[i] = (src >= 0 && s >= 0 && s < TW1) ? s_a[r * AP + s] : 0.f;
                }
            }
            __syncthreads();
#pragma unroll
            for (int i = 0; i < CH * TW1 / NT; ++i) {
                const int idx = tid + i * NT, r = idx / TW1, q = idx - r * TW1;
                s_a[r * AP + q] = v[i];
            }
            __syncthreads();
        }

        // ---- level-(l+1) row pass: thread <-> (low|high-pass, approximation row, 4 output columns) ---------
        // per output the even / odd paired sums of row_filter
        if (tid < 2 * CH * NG2) {
            const int hp = tid / (CH * NG2), q = tid - hp * (CH * NG2);
            const int r = q / NG2, g = q - r * NG2;
            const float* src = s_a + r * AP + 8 * g;
            const float2* taps = hp ? p.ph : p.pl;
            float v[16];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float4 t = *reinterpret_cast<const float4*>(src + 4 * k);
                v[4 * k] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w;
            }
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float2 a = make_float2(0.f, 0.f);
#pragma unroll
                for (int m = 0; m < L / 2; ++m)
                    a = ffma2(taps[m], make_float2(v[2 * e + 2 * m + F::OFF2], v[2 * e + 2 * m + F::OFF2 + 1]), a);
                o[e] = a.x + a.y;
            }
            const int line = (yb + c * CH + r) & RMASK;
            *reinterpret_cast<float4*>((hp ? s_h2 : s_l2) + line * LP + 4 * g) = make_float4(o[0], o[1], o[2], o[3]);
        }
        __syncthreads();

        // ---- level-(l+1) column pass: thread <-> (lo|hi lines, vertical low|high-pass, output row, 4 columns) --
        // Chunk c holds the rows of outputs Yb + 8 c + [0, 8); chunk 0's outputs lie above the segment.
        if (c > 0 && tid < 4 * CH2 * NG2) {
            const int h = tid / (2 * CH2 * NG2), q0 = tid - h * (2 * CH2 * NG2);
            const int vh = q0 / (CH2 * NG2), q = q0 - vh * (CH2 * NG2);
            const int yr = q / NG2, g = q - yr * NG2;
            const int Y = Yb + c * CH2 + yr, X = X0 + 4 * g;
            const float* lines = (h ? s_h2 : s_l2) + 4 * g;
            const float2* taps = vh ? p.bh : p.bl;
            const int r0 = 2 * Y - HALO;
            float2 a0 = make_float2(0.f, 0.f), a1 = make_float2(0.f, 0.f);
            if (r0 >= 0 && r0 + L <= p.Mh1) {
#pragma unroll
                for (int j = 0; j < L; ++j) {
                    const float4 f = *reinterpret_cast<const float4*>(lines + ((r0 + j) & RMASK) * LP);
                    a0 = ffma2(taps[j], make_float2(f.x, f.y), a0);
                    a1 = ffma2(taps[j], make_float2(f.z, f.w), a1);
                }
            } else {   // window over the top / bottom edge: lines of the extension sources
                for (int j = 0; j < L; ++j) {
                    const int sr = ext_index32(r0 + j, p.Mh1, p.mode);
                    float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (sr >= 0) f = *reinterpret_cast<const float4*>(lines + (sr & RMASK) * LP);
                    a0 = ffma2(taps[j], make_float2(f.x, f.y), a0);
                    a1 = ffma2(taps[j], make_float2(f.z, f.w), a1);
                }
            }
            const int k = 2 * vh + h;   // band: the lo lines yield k = 0, 2; the hi lines k = 1, 3
            if (Y >= Y0 && Y < Y1 && X >= X0n && X < p.Mw2)
                *reinterpret_cast<float4*>(p.o2[k] + (int64_t)b * p.o2_bs[k] + (int64_t)Y * p.o2_rs[k] + X) =
                    make_float4(a0.x, a0.y, a1.x, a1.y);
        }
        // no barrier: the next writes of s_lo / s_hi, s_a and the line ring are each behind one of the next
        // chunk's barriers, and all readers of those buffers in this chunk are ahead of it
        ring_base += IN_ROWS;
        if (ring_base >= RING) ring_base -= RING;
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// Returns true when the two levels were launched here (*err carries the launch status).  Declines (returns false)
// levels smaller than FUSE2_MIN in either direction and layouts without 128-bit stores.
constexpr int FUSE2_MIN = 32;

template <int L>
static bool launch_fwd2d_fuse2(const float* x, int64_t B, int H, int W, int64_t x_bs, int64_t x_rs, const wt_level& l1,
                               const wt_level& l2, int mode, const Taps<float>& taps, cudaStream_t st,
                               uint64_t* launches, cudaError_t* err) {
    using F = Fuse2Geom<L>;
    Fuse2Params p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.x_bs = x_bs; p.x_rs = x_rs; p.H = H; p.W = W;
    p.Mh1 = (int)l1.dims[0]; p.Mw1 = (int)l1.dims[1]; p.Mh2 = (int)l2.dims[0]; p.Mw2 = (int)l2.dims[1];
    if (p.Mh1 < FUSE2_MIN || p.Mw1 < FUSE2_MIN) return false;
    if (l1.strides[1] != 1 || l2.strides[1] != 1 || l2.approx_strides[1] != 1) return false;
    for (int k = 0; k < 3; ++k) {
        p.d1[k] = (float*)l1.details + (int64_t)k * l1.band_stride;
        p.d1_bs[k] = l1.details_batch_stride; p.d1_rs[k] = l1.strides[0];
    }
    p.o2[0] = (float*)l2.approx; p.o2_bs[0] = l2.approx_batch_stride; p.o2_rs[0] = l2.approx_strides[0];
    for (int k = 1; k < 4; ++k) {
        p.o2[k] = (float*)l2.details + (int64_t)(k - 1) * l2.band_stride;
        p.o2_bs[k] = l2.details_batch_stride; p.o2_rs[k] = l2.strides[0];
    }
    // 128-bit stores: every band row starts on a 16-byte boundary and its pitch covers the rounded-up width
    for (int k = 0; k < 3; ++k)
        if (((uintptr_t)p.d1[k] & 15) || (p.d1_bs[k] & 3) || (p.d1_rs[k] & 3) || p.d1_rs[k] < (p.Mw1 + 3) / 4 * 4) return false;
    for (int k = 0; k < 4; ++k)
        if (((uintptr_t)p.o2[k] & 15) || (p.o2_bs[k] & 3) || (p.o2_rs[k] & 3) || p.o2_rs[k] < (p.Mw2 + 3) / 4 * 4) return false;
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof(tmap));
    if (!make_tmap_3d<float>(&tmap, x, B, H, W, x_bs, x_rs, F::G1::SW, F::G1::IN_ROWS)) return false;
    p.mode = mode;
    for (int m = 0; m < L / 2; ++m) {
        p.pl[m] = make_float2(taps.lo[L - 1 - 2 * m], taps.lo[L - 2 - 2 * m]);
        p.ph[m] = make_float2(taps.hi[L - 1 - 2 * m], taps.hi[L - 2 - 2 * m]);
    }
    for (int j = 0; j < L; ++j) {
        p.bl[j] = make_float2(taps.lo[L - 1 - j], taps.lo[L - 1 - j]);
        p.bh[j] = make_float2(taps.hi[L - 1 - j], taps.hi[L - 1 - j]);
    }
    // segments: each restarts with one chunk of 8 level-(l+1) rows, so long ones (~2-3 % restart work) unless
    // the grid would fill the machine fewer than 8 times
    const int nstrip = (p.Mw2 + F::TW2 - 1) / F::TW2;
    int nseg = (p.Mh2 + 383) / 384;
    while ((int64_t)nseg * nstrip * B < 8 * 3 * (int64_t)sm_count() && (p.Mh2 + nseg - 1) / nseg > 32) ++nseg;
    const int seg = ((p.Mh2 + nseg - 1) / nseg + F::CH2 - 1) / F::CH2 * F::CH2;
    nseg = (p.Mh2 + seg - 1) / seg;
    p.seg_rows = seg;
    auto kern = fwd2d_fuse2_f32_kernel<L>;
    *err = ensure_dyn_smem(kern, F::SMEM);
    if (*err != cudaSuccess) return true;
    for (int64_t b0 = 0; b0 < B; b0 += 65535) {
        p.batch0 = (int)b0;
        const int nb = (int)((B - b0) < 65535 ? (B - b0) : 65535);
        dim3 grid(nstrip, nseg, nb);
        kern<<<grid, F::NT, F::SMEM, st>>>(p, tmap);
        ++*launches;
        *err = cudaGetLastError();
        if (*err != cudaSuccess) return true;
    }
    return true;
}

template <typename T>
static bool try_fuse2(const T*, int64_t, int, int, int64_t, int64_t, const wt_level&, const wt_level&, int, int,
                      const Taps<T>&, cudaStream_t, uint64_t*, cudaError_t*) {
    return false;
}
template <>
bool try_fuse2<float>(const float* x, int64_t B, int H, int W, int64_t x_bs, int64_t x_rs, const wt_level& l1,
                      const wt_level& l2, int L, int mode, const Taps<float>& taps, cudaStream_t st,
                      uint64_t* launches, cudaError_t* err) {
    // Opt-in (WTB200_FUSE2=1 / wt_set_knob("FUSE2", 1)): bit-identical to one launch per level with 20 % fewer DRAM
    // bytes at levels 1-2, but slower on an H100 80GB HBM3 at a 400 W power limit -- levels 1-2 of 64 x 4096^2 db4
    // 5.81 ms against 5.38 ms for two strip-kernel launches, and slower at every shape tools/time_fwd2d_pairs.py
    // times, levels 3-4 included -- so it is not the default.  With NO_FFMA2 the per-level path uses the unpaired
    // kernel, whose FMA order this kernel does not reproduce.
    if (!knob_on(K_FUSE2) || knob_on(K_NO_FFMA2) || mode == WT_MODE_PERIODIC) return false;
    switch (L) {
        case 2: return launch_fwd2d_fuse2<2>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
        case 4: return launch_fwd2d_fuse2<4>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
        case 6: return launch_fwd2d_fuse2<6>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
        case 8: return launch_fwd2d_fuse2<8>(x, B, H, W, x_bs, x_rs, l1, l2, mode, taps, st, launches, err);
        default: return false;
    }
}

}  // namespace wtb
