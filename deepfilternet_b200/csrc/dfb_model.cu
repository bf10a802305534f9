// dfb_model.cu -- the DNN of the enhancement path (encoder convs, grouped linears, GRUs, ERB and
// DF decoders) as hand-written sm_90a kernels plus the executor behind dfb_model_* / dfb_enhance.
//
// Reference semantics (paths relative to /root/reference/DeepFilterNet/df):
//   Conv2dNormAct / ConvTranspose2dNormAct   modules.py:18-72, 75-126
//   GroupedLinearEinsum                       modules.py:741-780
//   SqueezedGRU_S / SqueezedGRU               modules.py:702-738 / 663-699  (torch.nn.GRU inside)
//   Encoder / ErbDecoder / DfDecoder          deepfilternet3.py:100-331, deepfilternet2.py:98-371
//   DfNet.forward                             deepfilternet3.py:389-456,   deepfilternet2.py:481-505
//
// HBM layout: every activation is channel-last [B, T, F, C=64] (C fastest) so a 1x1 conv is a
// row-major [rows, 64] x [64, 64] product and depthwise taps are +-64-float neighbours;
// embeddings are [B*T, D] row-major.  BatchNorm is folded on the host (weights.py).
// Arithmetic: the contractions (GRU recurrence and input projections, separable blocks' 1x1 convs, grouped linears, DF
// pathway conv) run on the BF16x3 tensor-core kernels of dfb_tc.cu / dfb_gl.cu (fp32-level accuracy, DESIGN.md section 6);
// the kernels in this file are IEEE fp32 FFMA.  Accumulation order differs from ATen's, which is inside the 1e-4 RMS
// parity bound (tests/test_gpu_parity.py).
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <numeric>
#include <string>

#include "dfb_common.cuh"
#include "dfb_dwpw.cuh"
#include "dfb_ptx.cuh"

namespace dfb {


enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_TANH = 2, ACT_SIGMOID = 3 };

__device__ __forceinline__ float act_apply(float x, int act) {
    switch (act) {
        case ACT_RELU: return fmaxf(x, 0.f);
        case ACT_TANH: return tanhf(x);
        case ACT_SIGMOID: return 1.f / (1.f + expf(-x));
        default: return x;
    }
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ------------------------------------------------------- input convs (erb_conv0, df_conv0) ----
// Dense CIN -> 64 conv, kernel (kt,3), causal in time, BN folded, ReLU.
//   erb_conv0 (CIN = 1): modules.py:18-72 with in_ch = 1 (groups = 1, not separable).
//   df_conv0  (CIN = 2): grouped 2 -> 64 (kt,3) conv followed by the 64 x 64 1x1 conv and BN.  The two
//     linear maps are composed on the host (weights.py): W[dt][df][ri][n] = sum_{c in group ri}
//     dw[dt][df][c] * pw[c][n], so the 64-wide intermediate never exists: 18 instead of 73 MACs per output.
// Feature look-ahead: deepfilternet3.py:359,409-410.
// in  x [B,T,F,CIN]; out [B,T,F,64].  One CTA = kInFrames frames; thread = (f slot, channel quad), taps in registers.
constexpr int kInFrames = 8;
template <int CIN>
__global__ void __launch_bounds__(256)
k_conv_in(const float *__restrict__ x, const float *__restrict__ w /*[kt][3][CIN][64]*/, const float *__restrict__ bias,
          float *__restrict__ out, int T, int F, int kt, int lookahead, int Tsx /* frames per stream in x */,
          int Tx /* feature frames that exist; beyond = end of the stream = zero */,
          int tp_min /* 0: the features are shifted by the look-ahead, then padded causally (DeepFilterNet2 / 3, pad_feat);
                        -lookahead: the conv itself pads (kt-1-la, la) around the unshifted features (DeepFilterNet v1) */,
          const RaggedRow *__restrict__ rg /* ragged batch: stream b's features end at its own frame count */, int64_t w0 /* absolute frame of window row 0 */,
          const int64_t *__restrict__ first /* streaming slots: stream b's shifted features start at its own first frame */) {
    extern __shared__ float s_in[];  // [(kInFrames + kt - 1)][(F + 2) * CIN]
    const int b = blockIdx.y, t0 = blockIdx.x * kInFrames;
    const int rows = kInFrames + kt - 1, ld = (F + 2) * CIN;
    if (rg) Tx = min(Tx, (int)(rg[b].Tf - w0));
    if (first) tp_min = max(tp_min, stream_first(first, b, w0));
    for (int i = threadIdx.x; i < rows * ld; i += blockDim.x) {
        int r = i / ld, j = i - r * ld;
        int f = j / CIN - 1, ci = j - (f + 1) * CIN;
        int tp = t0 - (kt - 1) + r;  // time index in the look-ahead shifted feature sequence
        float v = 0.f;
        if (f >= 0 && f < F && tp >= tp_min && tp + lookahead < Tx) v = x[(((int64_t)b * Tsx + tp + lookahead) * F + f) * CIN + ci];
        s_in[i] = v;
    }
    const int cq = threadIdx.x & 15, fl = threadIdx.x >> 4;  // 16 channel quads x 16 f per pass
    // taps of this thread's channel quad as two packed fp32 pairs (f2_fma: one FFMA per channel)
    unsigned long long wr[9 * CIN][2];
#pragma unroll
    for (int i = 0; i < 9 * CIN; i++) {
        const float4 v = (i >= (3 - kt) * 3 * CIN) ? *reinterpret_cast<const float4 *>(w + (i - (3 - kt) * 3 * CIN) * kCh + cq * 4)
                                                   : make_float4(0.f, 0.f, 0.f, 0.f);
        wr[i][0] = f2_pack(v.x, v.y); wr[i][1] = f2_pack(v.z, v.w);
    }
    const float4 bv = *reinterpret_cast<const float4 *>(bias + cq * 4);
    const unsigned long long b01 = f2_pack(bv.x, bv.y), b23 = f2_pack(bv.z, bv.w);
    __syncthreads();
    for (int fr = 0; fr < kInFrames; fr++) {
        int t = t0 + fr;
        if (t >= T) break;
        for (int f = fl; f < F; f += 16) {
            unsigned long long a01 = b01, a23 = b23;
#pragma unroll
            for (int dt = 0; dt < 3; dt++) {
                if (dt < 3 - kt) continue;
                const float *row = s_in + (fr + dt - (3 - kt)) * ld + f * CIN;  // f-1 .. f+1 -> +0 .. +2
#pragma unroll
                for (int j = 0; j < 3 * CIN; j++) {
                    const float xv = row[j];
                    const unsigned long long xx = f2_pack(xv, xv);
                    a01 = f2_fma(xx, wr[dt * 3 * CIN + j][0], a01);
                    a23 = f2_fma(xx, wr[dt * 3 * CIN + j][1], a23);
                }
            }
            float4 acc;
            f2_unpack(a01, acc.x, acc.y); f2_unpack(a23, acc.z, acc.w);
            acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f);
            *reinterpret_cast<float4 *>(out + (((int64_t)b * T + t) * F + f) * kCh + cq * 4) = acc;
        }
    }
}

// ------------------------------------------------- depthwise (+pathway) -> 1x1 -> ReLU ----
// One fused kernel for a "separable" block of the reference (modules.py:49-71, 104-125):
//   prologue  A[r][c] = sum_{dt,df} dw[dt][df][c] * X[t-(kt-1)+dt][fi(fo,df)][c]
//             with X = in (+ relu(path * ps + pb) when a pathway tensor is given; that is
//             `convNp(eN) + prev`, deepfilternet3.py:250-253)
//   GEMM      out[r][n] = relu(sum_c A[r][c] * pw[c][n] + b[n])
// The FFMA version of k_dwpw_bx (dfb_tc.cu) for the blocks that one does not build: DeepFilterNet v1's blocks with a
// look-ahead and its two-time-tap transposed convs.
// Modes: S1 stride 1, S2 stride 2 (fi = 2 fo + df - 1), T2 transposed stride 2
// (out[2j] = w1 x[j]; out[2j+1] = w2 x[j] + w0 x[j+1]; ConvTranspose2d padding 1, output_padding 1).
// Tile: NF frames x Fout rows (R = NF * Fout <= 128, multiple of 4); thread tile 4 rows x 8 cols.
template <int MODE>
__global__ void __launch_bounds__(256) k_dwpw(DwPwParams p) {
    extern __shared__ __align__(16) float smem[];
    float *Ws = smem;                 // [64][64]
    float *As = smem + kCh * kCh;     // [R][kLdA]
    const int b = blockIdx.y, t0 = blockIdx.x * p.NF;
    const int tid = threadIdx.x;
    const int nf = min(p.NF, p.T - t0);
    const int R = nf * p.Fout;        // rows actually present
    const int Rfull = p.NF * p.Fout;
    for (int i = tid; i < kCh * kCh / 4; i += 256)
        reinterpret_cast<float4 *>(Ws)[i] = reinterpret_cast<const float4 *>(p.pw)[i];
    // ---- prologue: thread = (row slot, channel quad)
    {
        const int cq = tid & 15;
        DwTaps taps;
        dw_load_taps(p, cq, taps);
        for (int r = tid >> 4; r < Rfull; r += 16) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < R) {
                const int fr = r / p.Fout, fo = r - fr * p.Fout;
                acc = dw_prologue<MODE>(p, taps, b, t0 + fr, fo, cq);
            }
            *reinterpret_cast<float4 *>(As + r * kLdA + cq * 4) = acc;
        }
    }
    __syncthreads();
    // ---- GEMM: thread (rg, cg): rows rg + RG * i (i < 4), cols 8 cg .. 8 cg + 7
    const int RG = Rfull >> 2;
    const int cgid = tid & 7, rg = tid >> 3;
    if (rg >= RG) return;
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i][j] = 0.f;
#pragma unroll 4
    for (int k = 0; k < kCh; k += 4) {
        float4 a[4];
#pragma unroll
        for (int i = 0; i < 4; i++) a[i] = *reinterpret_cast<const float4 *>(As + (rg + RG * i) * kLdA + k);
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
            float4 w0 = *reinterpret_cast<const float4 *>(Ws + (k + kk) * kCh + cgid * 8);
            float4 w1 = *reinterpret_cast<const float4 *>(Ws + (k + kk) * kCh + cgid * 8 + 4);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                float av = kk == 0 ? a[i].x : kk == 1 ? a[i].y : kk == 2 ? a[i].z : a[i].w;
                acc[i][0] += av * w0.x; acc[i][1] += av * w0.y; acc[i][2] += av * w0.z; acc[i][3] += av * w0.w;
                acc[i][4] += av * w1.x; acc[i][5] += av * w1.y; acc[i][6] += av * w1.z; acc[i][7] += av * w1.w;
            }
        }
    }
    const float4 b0 = *reinterpret_cast<const float4 *>(p.bias + cgid * 8);
    const float4 b1 = *reinterpret_cast<const float4 *>(p.bias + cgid * 8 + 4);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int r = rg + RG * i;
        if (r >= R) continue;
        int fr = r / p.Fout, fo = r - fr * p.Fout;
        float *dst = p.out + ((int64_t)b * p.T + t0 + fr) * p.out_fs + fo * kCh + cgid * 8;
        float4 o0 = make_float4(fmaxf(acc[i][0] + b0.x, 0.f), fmaxf(acc[i][1] + b0.y, 0.f),
                                fmaxf(acc[i][2] + b0.z, 0.f), fmaxf(acc[i][3] + b0.w, 0.f));
        float4 o1 = make_float4(fmaxf(acc[i][4] + b1.x, 0.f), fmaxf(acc[i][5] + b1.y, 0.f),
                                fmaxf(acc[i][6] + b1.z, 0.f), fmaxf(acc[i][7] + b1.w, 0.f));
        *reinterpret_cast<float4 *>(dst) = o0;
        *reinterpret_cast<float4 *>(dst + 4) = o1;
    }
}

// ------------------------------------------------------------------ grouped linear ----
// Y[m, g*Hg + n] = act( sum_i X[m, g*Ig + i] * W[g][i][n] + bias ) * oscale + ooffset + R[m, ...]
// (GroupedLinearEinsum, modules.py:766-776.)  The FFMA version of k_gl_bx (dfb_gl.cu) for the shapes that one does not
// build: the N = 1 heads, DeepFilterNet v1's GroupedLinear with bias, weights without a tensor-core image.
// CTA tile 64 rows x 64 cols (one group, or a 64-wide slice of a wide group); K chunks of 32.
struct GlParams {
    const float *x; int64_t ldx;
    const float *w;          // [G][Ig][Hg]
    const float *bias;       // [G*Hg] or null
    const float *res; int64_t ldr;  // optional residual, added after the activation
    float *y; int64_t ldy;
    int64_t M;
    int G, Ig, Hg, act;
    float oscale, ooffset;
    unsigned short *y_hi, *y_lo;  // optional BF16 hi/lo planes of y (same pitch): operand of a tensor-core GEMM
};
constexpr int kGlBM = 64, kGlBN = 64, kGlBK = 32, kGlMaxGpc = 4;

// Narrow groups (Hg = 16 or 32) are packed kGpc = 64 / Hg per CTA so that all 256 threads own real
// output columns (the first version ran one group per CTA: 25 % of the threads active for Hg = 16).
__global__ void __launch_bounds__(256) k_grouped_linear(GlParams p) {
    __shared__ __align__(16) float As[kGlMaxGpc][kGlBM][kGlBK + 4];
    __shared__ __align__(16) float Ws[kGlBK][kGlBN];
    const int gpc = (p.Hg < kGlBN && kGlBN % p.Hg == 0) ? min(kGlBN / p.Hg, p.G) : 1;  // groups per CTA
    const int tiles_per_group = (p.Hg + kGlBN - 1) / kGlBN;                         // > 1 only when gpc == 1
    const int gb = blockIdx.y / tiles_per_group, nt = blockIdx.y - gb * tiles_per_group;
    const int g0 = gb * gpc;                       // first group of this CTA
    const int n0 = nt * kGlBN;                     // column offset inside the group (gpc == 1)
    const int wcols = gpc > 1 ? p.Hg : min(kGlBN, p.Hg - n0);  // valid columns per group in this tile
    const int ngrp = min(gpc, p.G - g0);
    const int64_t m0 = (int64_t)blockIdx.x * kGlBM;
    const int tid = threadIdx.x;
    const int tc = tid & 15, tr = tid >> 4;  // thread tile: rows tr + 16 i, cols 4 tc .. 4 tc + 3
    const int gsub = gpc > 1 ? (tc * 4) / p.Hg : 0;  // which of the CTA's groups this thread's columns belong to
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
    // loader roles are fixed per thread (no per-element division): A tile -- row ar + 32 i of group ags, k quad akq;
    // W tile -- column quad wn (group wgs, in-group offset wnn), rows wk + 16 i
    const int akq = (tid & 7) * 4, ar = tid >> 3;
    const int wn = (tid & 15) * 4, wk = tid >> 4;
    int wgs = 0, wnn = n0 + wn;
    if (gpc > 1) { wgs = wn / p.Hg; wnn = wn - wgs * p.Hg; }
    const bool wvec = (p.Hg & 3) == 0;                       // a column quad never straddles a group and is 16-byte aligned
    const bool wok = gpc > 1 ? wgs < ngrp : wn < wcols;
    const float *xrow[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int64_t m = m0 + ar + 32 * i;
        xrow[i] = m < p.M ? p.x + m * p.ldx + (int64_t)g0 * p.Ig + akq : nullptr;
    }
    const float *wbase = p.w + ((int64_t)(g0 + wgs) * p.Ig) * p.Hg + wnn;
    for (int k0 = 0; k0 < p.Ig; k0 += kGlBK) {
        const int kc = min(kGlBK, p.Ig - k0);
        // A tiles: per group 64 rows x 32 k  (8 threads x float4 per row)
        for (int gs = 0; gs < ngrp; gs++) {
#pragma unroll
            for (int i = 0; i < 2; i++) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (xrow[i] && akq < kc) v = *reinterpret_cast<const float4 *>(xrow[i] + gs * p.Ig + k0);
                *reinterpret_cast<float4 *>(&As[gs][ar + 32 * i][akq]) = v;
            }
        }
        // W tile: 32 k x 64 columns (column n -> group n / Hg when several groups share the CTA)
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int k = wk + 16 * i;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k < kc && wok) {
                const float *src = wbase + (int64_t)(k0 + k) * p.Hg;
                if (wvec) {
                    if (gpc > 1 || wn + 3 < wcols) v = *reinterpret_cast<const float4 *>(src);
                    else { v.x = src[0]; if (wn + 1 < wcols) v.y = src[1]; if (wn + 2 < wcols) v.z = src[2]; }
                } else {
                    const int lim = gpc > 1 ? p.Hg - wnn : wcols - wn;
                    v.x = src[0]; if (lim > 1) v.y = src[1]; if (lim > 2) v.z = src[2]; if (lim > 3) v.w = src[3];
                }
            }
            *reinterpret_cast<float4 *>(&Ws[k][wn]) = v;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kGlBK; k += 4) {
            float4 a[4];
#pragma unroll
            for (int i = 0; i < 4; i++) a[i] = *reinterpret_cast<const float4 *>(&As[gsub][tr + 16 * i][k]);
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
                float4 w = *reinterpret_cast<const float4 *>(&Ws[k + kk][tc * 4]);
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    float av = kk == 0 ? a[i].x : kk == 1 ? a[i].y : kk == 2 ? a[i].z : a[i].w;
                    acc[i][0] += av * w.x; acc[i][1] += av * w.y; acc[i][2] += av * w.z; acc[i][3] += av * w.w;
                }
            }
        }
        __syncthreads();
    }
    // columns of this thread: group g0 + gsub, inside-group offset nn0 .. nn0 + 3
    const int nn0 = gpc > 1 ? tc * 4 - gsub * p.Hg : n0 + tc * 4;
    if (gsub >= ngrp) return;
    const int colbase = (g0 + gsub) * p.Hg + nn0;
    const int nvalid = min(4, p.Hg - nn0);  // <= 0 when the thread's columns are past the group end
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int64_t m = m0 + tr + 16 * i;
        if (m >= p.M || nvalid <= 0) continue;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            v[j] = acc[i][j];
            if (j < nvalid) {
                const int col = colbase + j;
                if (p.bias) v[j] += p.bias[col];
                v[j] = act_apply(v[j], p.act) * p.oscale + p.ooffset;
                if (p.res) v[j] += p.res[m * p.ldr + col];
            }
        }
        float *dst = p.y + m * p.ldy + colbase;
        if (nvalid == 4 && (((uintptr_t)dst) & 15) == 0) {
            *reinterpret_cast<float4 *>(dst) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
            for (int j = 0; j < nvalid; j++) dst[j] = v[j];
        }
        if (p.y_hi) {
            unsigned short hi[4], lo[4];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                __nv_bfloat16 hb = __float2bfloat16_rn(v[j]);
                hi[j] = __bfloat16_as_ushort(hb);
                lo[j] = __bfloat16_as_ushort(__float2bfloat16_rn(v[j] - __bfloat162float(hb)));
            }
            unsigned short *dh = p.y_hi + m * p.ldy + colbase, *dl = p.y_lo + m * p.ldy + colbase;
            if (nvalid == 4 && (((uintptr_t)dh) & 7) == 0) {
                *reinterpret_cast<uint2 *>(dh) = make_uint2(hi[0] | (uint32_t)hi[1] << 16, hi[2] | (uint32_t)hi[3] << 16);
                *reinterpret_cast<uint2 *>(dl) = make_uint2(lo[0] | (uint32_t)lo[1] << 16, lo[2] | (uint32_t)lo[3] << 16);
            } else {
                for (int j = 0; j < nvalid; j++) { dh[j] = hi[j]; dl[j] = lo[j]; }
            }
        }
    }
}

// --------------------------------------------------------------- ERB mask output conv ----
// m[b,t,f] = sigmoid( sum_{dt,df,c} w[dt][df][c] * X[t-(kt-1)+dt][f+df-1][c] + bias ),
// X = relu(e0 * ps + pb) + d1   (conv0_out(conv0p(e0) + e1), deepfilternet3.py:253).
// One warp walks kMaskChunk consecutive frames of one stream; X rows of the current and the
// previous frame are staged in shared memory ([E+2][65] floats, zero rows at f = -1, E).
constexpr int kMaskWarps = 4, kMaskChunk = 8, kMaskLd = kCh + 1;
__global__ void __launch_bounds__(32 * kMaskWarps)
k_mask_out(const float *__restrict__ e0, const float *__restrict__ d1, const float *__restrict__ ps,
           const float *__restrict__ pb, const float *__restrict__ w /*[kt][3][64]*/,
           const float *__restrict__ bias_p, float *__restrict__ m, int T, int E, int kt,
           const int64_t *__restrict__ first /* streaming slots (stream_first) or null */, int64_t w0) {
    extern __shared__ float smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.y;
    const int t0 = (blockIdx.x * kMaskWarps + warp) * kMaskChunk;
    const int t_first = stream_first(first, b, w0);   // the previous-frame tap of frame t_first is padding
    float *buf = smem + warp * 2 * (E + 2) * kMaskLd;  // two frames
    float *ws = smem + kMaskWarps * 2 * (E + 2) * kMaskLd;  // [kt*3*64] shared by all warps
    for (int i = threadIdx.x; i < kt * 3 * kCh; i += blockDim.x) ws[i] = w[i];
    for (int i = lane; i < 2 * (E + 2) * kMaskLd; i += 32) buf[i] = 0.f;
    __syncthreads();
    if (t0 >= T) return;
    const int t1 = min(t0 + kMaskChunk, T);
    const float2 ps2 = *reinterpret_cast<const float2 *>(ps + lane * 2);
    const float2 pb2 = *reinterpret_cast<const float2 *>(pb + lane * 2);
    const float bias = bias_p[0];
    for (int t = (kt > 1 && t0 > 0) ? t0 - 1 : t0; t < t1; t++) {
        float *cur = buf + (t & 1) * (E + 2) * kMaskLd;
        const float *prv = buf + ((t & 1) ^ 1) * (E + 2) * kMaskLd;
        const int64_t base = ((int64_t)b * T + t) * E * kCh;
        for (int f = 0; f < E; f++) {
            float2 e = *reinterpret_cast<const float2 *>(e0 + base + f * kCh + lane * 2);
            float2 d = *reinterpret_cast<const float2 *>(d1 + base + f * kCh + lane * 2);
            cur[(f + 1) * kMaskLd + lane * 2] = fmaxf(e.x * ps2.x + pb2.x, 0.f) + d.x;
            cur[(f + 1) * kMaskLd + lane * 2 + 1] = fmaxf(e.y * ps2.y + pb2.y, 0.f) + d.y;
        }
        __syncwarp();
        if (t >= t0) {
            for (int f = lane; f < E; f += 32) {
                float acc = bias;
                for (int dt = 0; dt < kt; dt++) {
                    // dt = kt-1 is the current frame; dt = kt-2 the previous one (kt <= 2)
                    const float *src = (dt == kt - 1) ? cur : prv;
                    if (dt != kt - 1 && t <= t_first) continue;
                    for (int df = 0; df < 3; df++) {
                        const float *xr = src + (f + df) * kMaskLd;
                        const float *wr = ws + (dt * 3 + df) * kCh;
#pragma unroll 16
                        for (int c = 0; c < kCh; c++) acc += xr[c] * wr[c];
                    }
                }
                m[((int64_t)b * T + t) * E + f] = sigmoidf_(acc);
            }
        }
        __syncwarp();
    }
}

// ------------------------------------------------- DeepFilterNet v1: gather-sum, pathway 1x1 ----
// out[m][k] = act( sum_i src_i[m][idx_i[k]] ), optionally also as BF16 hi / lo planes.  DeepFilterNet v1 flattens channel-major
// into its grouped layers and interleaves ("shuffles") their outputs (deepfilternet.py:135-139,183-185; modules.py:651-654,
// 807-812) while the device tensors are channel-last: every such re-ordering, and the sum over the GRU layers' outputs
// (add_outputs, modules.py:655-656), is one pass of this kernel with host-built index tables (weights.py: v1.idx_*).
struct GatherParams {
    const float *src[3]; long long ld[3]; const int *idx[3]; int n;
    float *out; long long ldo;
    unsigned short *hi, *lo; long long ldp;
    int K, relu;
};
__global__ void __launch_bounds__(256) k_gather_sum(GatherParams p) {
    const long long m = blockIdx.x;
    for (int k = threadIdx.x; k < p.K; k += 256) {
        float v = 0.f;
#pragma unroll
        for (int i = 0; i < 3; i++)
            if (i < p.n) v += p.src[i][m * p.ld[i] + p.idx[i][k]];
        if (p.relu) v = fmaxf(v, 0.f);
        if (p.out) p.out[m * p.ldo + k] = v;
        if (p.hi) {
            unsigned short h, l;
            bf16_split(v, h, l);
            p.hi[m * p.ldp + k] = h; p.lo[m * p.ldp + k] = l;
        }
    }
}

// coefs[r][k] = tanh(coefs[r][k]) + relu(sum_c c0[r][c] w[c][k] + b[k]),  r = (b, t, f), k < 2 O: the dense 1x1 pathway conv
// df_convp (deepfilternet.py:210-212) on top of the df_fc_out pre-activations already in `coefs` (deepfilternet.py:224-228)
template <int O2>
__global__ void __launch_bounds__(128) k_convp_v1(const float *__restrict__ c0, const float *__restrict__ w /*[64][O2]*/,
                                                   const float *__restrict__ bias, float *__restrict__ coefs, long long rows) {
    __shared__ float ws[kCh * O2];
    __shared__ float bs[O2];
    for (int i = threadIdx.x; i < kCh * O2; i += 128) ws[i] = w[i];
    if (threadIdx.x < O2) bs[threadIdx.x] = bias[threadIdx.x];
    __syncthreads();
    const long long r = (long long)blockIdx.x * 128 + threadIdx.x;
    if (r >= rows) return;
    float acc[O2];
#pragma unroll
    for (int k = 0; k < O2; k++) acc[k] = bs[k];
    const float4 *x = reinterpret_cast<const float4 *>(c0 + r * kCh);
#pragma unroll 4
    for (int q = 0; q < kCh / 4; q++) {
        const float4 v = x[q];
#pragma unroll
        for (int k = 0; k < O2; k++)
            acc[k] += v.x * ws[(4 * q) * O2 + k] + v.y * ws[(4 * q + 1) * O2 + k] + v.z * ws[(4 * q + 2) * O2 + k] + v.w * ws[(4 * q + 3) * O2 + k];
    }
    float *o = coefs + r * O2;
#pragma unroll
    for (int k = 0; k < O2; k++) o[k] = tanhf(o[k]) + fmaxf(acc[k], 0.f);
}

constexpr int kMaxO2 = 16;  // largest 2 * df_order dfb_model_create accepts
constexpr int kMaxLookahead = 3;  // largest conv_lookahead / df_lookahead dfb_model_create accepts

}  // namespace dfb

// =========================================================================== executor =====
using namespace dfb;


// carried hidden states of one GRU stack between time chunks: h = [layers][Bs][H]; t0 = first frame the recurrences run.
// Bs is the stream count the state was allocated for: a chunk may run only a prefix B <= Bs of the streams (ragged batch)
// first / w0: streaming slots, each stream's first frame (stream_first) or null
struct GruChunk { float *h; bool have_state; int t0; int Bs; const int64_t *first; int64_t w0; const unsigned char *run = nullptr; };

// Weight tables: device pointers into the weight slab, bound once by dfb_model_create for the layers the configured
// forward pass runs.  A tensor that pass does not read stays null.
struct Wb { const float *w = nullptr, *b = nullptr; };  // input conv, head, DeepFilterNet v1 grouped linear with bias
struct Blk { const float *dw = nullptr, *pw = nullptr, *b = nullptr, *pw_sw = nullptr; };  // separable block (pw: v1)
struct PathW { const float *s = nullptr, *b = nullptr; };  // decoder pathway: relu(x * s + b)
// grouped linear [G][I/G][H/G]; bx: its tensor-core image `img` was uploaded and the shape is built, so it runs on the
// tensor-core kernel, which reads its input as BF16 planes only
struct Gl { const float *w = nullptr, *img = nullptr; int G = 0, I = 0, H = 0; bool bx = false; };
struct GruLayer { const float *w_hh, *b_ih, *b_hh, *w_ih_hi, *w_ih_lo; };  // w_ih_hi / lo: BF16 planes, two per float

struct NetW {  // DeepFilterNet2 / 3 (forward_body)
    Wb erb_conv0, df_conv0, lsnr, df_fc_a /* DeepFilterNet2 */, conv0_out;
    Blk erb_conv1, erb_conv2, erb_conv3, df_conv1, convt3, convt2, convt1;
    PathW conv3p, conv2p, conv1p, conv0p;
    Gl df_fc_emb, enc_in, enc_out, df_skip, df_in, df_out, erb_in, erb_out;
    std::vector<GruLayer> enc_gru, df_gru, erb_gru;
    struct { const float *w_sw, *w2, *b; } df_convp{};  // bound for a built df_order / df_pathway_kt (df_convp_built)
    bool fused_emb = false;  // df_conv1 + df_fc_emb run as one kernel (k_dwpw_gl); df_fc_emb's fp32 weight is not read then
};

struct NetWV1 {  // DeepFilterNet v1 (forward_v1)
    Wb erb_conv0, df_conv0, df_fc_emb, erb_fc_emb, lsnr, df_fc_a, df_convp, conv0_out;
    Blk erb_conv1, erb_conv2, erb_conv3, df_conv1, conv3p, conv2p, conv1p, conv0p, convt3, convt2, convt1;
    std::vector<GruLayer> enc_gru, df_gru;  // one GroupedGRULayer each
    struct { const float *w_t, *b, *w_hi, *w_lo; } df_fc_out{};  // w_hi / w_lo (BF16x3 GEMM) optional
    const float *ones = nullptr, *zeros = nullptr;
    const int *idx_c1 = nullptr, *idx_e3 = nullptr, *idx_shuf = nullptr, *idx_id = nullptr, *idx_dec = nullptr, *idx_gshuf = nullptr;
};

struct dfb_model {
    int device;
    dfb_model_config cfg;
    NetW net;      // model_kind 2 / 3
    NetWV1 net1;   // model_kind 1
    std::map<std::string, std::pair<const float *, int64_t>> dbg;  // activations of the last forward
    float *slab = nullptr;
    long long *gru_dbg = nullptr;  // device buffer for dfb_debug_gru_timing, [gru_dbg_steps][8]
    int gru_dbg_steps = 0;
    Arena arena;
    int dev_chunks = 0, host_chunks = 4, n_lanes = 2;   // chunk pipeline (dfb_model_set_chunking); dev_chunks 0 = auto
    int post_filter = 0, mask_only = 0;       // optional stages (dfb_model_set_options)
    int gating_mode = 0;                      // DFB_GATING_APPLY / DFB_GATING_RUNTIME (dfb_model_set_gating_mode)
    float pf_beta = 0.02f;
    size_t max_workspace = size_t(40) << 30;  // dfb_enhance chunks / groups the batch so that the arena stays below this
                                              // (40 GB: room for the batch itself and its output on an 80 GB H100)
    std::vector<int64_t> erb_widths;          // band table the model was built for (checked against the dfb_state)
    Arena aux_arena;                          // carried stream state + stream table of one dfb_enhance* stream group
    cudaStream_t stream = nullptr;
    cudaStream_t h2d = nullptr, d2h = nullptr;  // copy streams of the host batch path (both copy engines next to the compute)
    // One forward pass hops from the caller's stream onto the lane's internal streams: `hi` (ERB branch) and `aux` (DF
    // branch) for the encoder phase, `dhi` / `daux` at the greatest priority for the decoder phase (the recurrences are
    // the critical chain), `low` (least priority) for work off the critical path that only fills idle SMs.  Two lanes:
    // consecutive time chunks alternate between them, so that the encoder phase of chunk c + 1 overlaps the decoder
    // phase of chunk c (lane 1 has its own arena; everything outside the chunk loop uses lane 0).
    struct Lane {
        cudaStream_t main = nullptr, hi = nullptr, aux = nullptr, dhi = nullptr, daux = nullptr, low = nullptr;
        cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_fork_enc = nullptr, ev_join_enc = nullptr, ev_in = nullptr,
                    ev_out = nullptr, ev_c0 = nullptr, ev_convp = nullptr, ev_skip = nullptr, ev_done = nullptr;
        unsigned char *rt = nullptr;   // runtime gating mode's run flags and compacted DF pathway rows (grow-only)
        size_t rt_cap = 0;
    } lanes[2];
    Arena arena1;                           // lane 1's activations (lane 0 uses `arena`)
    // offline resamplers of rated batches (dfb_model_add_rate): the registered rates, their directions (rate_up[i] /
    // rate_down[i] for rates[i]; on the device as [up directions | down directions]) and their tap buffers
    std::vector<int> rates;
    std::vector<RateDir> rate_up, rate_down;
    std::vector<float *> rate_taps;
    RateDir *d_rate_dirs = nullptr;
    uint64_t fingerprint = 0;               // the config and the weight bytes (model_fingerprint): what a session blob names
};

// A 64-bit fingerprint of a model: its config, its ERB band widths, then every tensor's name, size and bytes in name order (the order the
// caller lists them in does not matter).  It tells session blobs (dfb_stream_export_sessions) of different models apart;
// it is not a cryptographic hash.
static uint64_t fp_mix(uint64_t h, const void *p, size_t n) {
    const unsigned char *b = static_cast<const unsigned char *>(p);
    size_t i = 0;
    for (; i + 8 <= n; i += 8) {
        uint64_t w;
        memcpy(&w, b + i, 8);
        h = (h ^ w) * 0x9E3779B97F4A7C15ull;
        h ^= h >> 29;
    }
    uint64_t w = n;
    for (size_t k = 0; i < n; i++, k++) w ^= (uint64_t)b[i] << (8 * (k % 8));
    h = (h ^ w) * 0xBF58476D1CE4E5B9ull;
    return h ^ (h >> 31);
}
static uint64_t model_fingerprint(const dfb_model_config &c, const int64_t *erb_widths, const dfb_tensor *tensors, int n_tensors) {
    uint64_t h = fp_mix(0x6466623230307366ull, &c, sizeof c);
    if (erb_widths) h = fp_mix(h, erb_widths, sizeof(int64_t) * (size_t)c.nb_erb);   // the ERB bands the model was built for
    std::map<std::string, int> order;
    for (int i = 0; i < n_tensors; i++) order[tensors[i].name] = i;
    for (const auto &kv : order) {
        const dfb_tensor &t = tensors[kv.second];
        h = fp_mix(h, kv.first.data(), kv.first.size());
        h = fp_mix(h, t.data, (size_t)t.numel * sizeof(float));
    }
    return h;
}

// Looks the uploaded tensors up by name.  The first missing or wrong-sized one (numel < 0: any size) becomes the bind's
// error; lookups after it return null.
struct Binder {
    const std::map<std::string, std::pair<const float *, int64_t>> &t;
    int rc = DFB_OK;
    const float *opt(const std::string &n) const { auto it = t.find(n); return it == t.end() ? nullptr : it->second.first; }
    const float *need(const std::string &n, int64_t numel) {
        auto it = t.find(n);
        if (!rc && it == t.end()) rc = fail(DFB_ERR_INVALID, "missing weight tensor '%s'", n.c_str());
        if (!rc && numel >= 0 && it->second.second != numel)
            rc = fail(DFB_ERR_INVALID, "weight tensor '%s' has %lld elements, expected %lld", n.c_str(), (long long)it->second.second, (long long)numel);
        return rc ? nullptr : it->second.first;
    }
    Wb wb(const std::string &n, int64_t nw, int64_t nb) { return {need(n + ".w", nw), need(n + ".b", nb)}; }
    PathW path(const std::string &n) { return {need(n + ".s", kCh), need(n + ".b", kCh)}; }
    Blk blk(const std::string &n, int64_t n_dw, bool pw, bool pw_sw) {
        return {need(n + ".dw", n_dw), pw ? need(n + ".pw", kCh * kCh) : nullptr, need(n + ".b", kCh), pw_sw ? need(n + ".pw_sw", kCh * kCh) : nullptr};
    }
    Gl gl(const std::string &n, int G, int I, int H, bool fp32 = true) {  // fp32 = false: only the tensor-core image is read
        const float *img = opt(n + "_bx");
        int gpc, hgp, stg;
        return {fp32 ? need(n, (int64_t)I * H / G) : nullptr, img, G, I, H,
                img && I % G == 0 && H % G == 0 && gl_bx_geometry(G, I / G, H / G, &gpc, &hgp, &stg)};
    }
    std::vector<GruLayer> gru(const std::string &n, int layers, int H) {  // every recurrence the forward passes run is H -> H
        std::vector<GruLayer> v;
        for (int l = 0; l < layers; l++) {
            const std::string p = n + ".l" + std::to_string(l);
            v.push_back({need(p + ".w_hh", (int64_t)3 * H * H), need(p + ".b_ih", 3 * H), need(p + ".b_hh", 3 * H),
                         need(p + ".w_ih_hi", (int64_t)3 * H * H / 2), need(p + ".w_ih_lo", (int64_t)3 * H * H / 2)});
        }
        return v;
    }
};

static int bind_net(const dfb_model_config &c, Binder &b, NetW &w) {
    const int E = c.nb_erb, Fd = c.nb_df, H = c.emb_hidden, Hd = c.df_hidden, O2 = 2 * c.df_order;
    const int ED = E / 4 * kCh, emb_in_dim = c.enc_concat ? 2 * ED : ED, emb_dim = c.model_kind == 2 ? H : ED;
    w.erb_conv0 = b.wb("enc.erb_conv0", c.inp_kt * 3 * kCh, kCh); w.df_conv0 = b.wb("enc.df_conv0", c.inp_kt * 3 * 2 * kCh, kCh);
    auto blk = [&](const char *n) { return b.blk(n, -1, false, true); };
    w.erb_conv1 = blk("enc.erb_conv1"); w.erb_conv2 = blk("enc.erb_conv2"); w.erb_conv3 = blk("enc.erb_conv3"); w.df_conv1 = blk("enc.df_conv1");
    w.convt3 = blk("erb_dec.convt3"); w.convt2 = blk("erb_dec.convt2"); w.convt1 = blk("erb_dec.convt1");
    w.conv3p = b.path("erb_dec.conv3p"); w.conv2p = b.path("erb_dec.conv2p"); w.conv1p = b.path("erb_dec.conv1p"); w.conv0p = b.path("erb_dec.conv0p");
    w.enc_in = b.gl("enc.emb_gru.in.gl", c.g_enc_in, emb_in_dim, H);
    // df_conv1 + df_fc_emb run fused when df_fc_emb's shape is built and enc.emb_gru.in reads emb_in as BF16 planes (the
    // FFMA grouped linear would read the fp32 tensor, which the fused kernel does not write); weights.py packs the
    // tensor-core images of every such shape
    const int I = Fd / 2 * kCh, G = c.g_df_fc_emb, Ge = c.g_enc_in;
    int de_s, de_st, gpc, hgp, stg;
    w.fused_emb = G > 0 && I % G == 0 && ED % G == 0 && df_emb_geometry(Fd, G, I / G, ED / G, c.conv_kt, &de_s, &de_st) &&
                  Ge > 0 && emb_in_dim % Ge == 0 && H % Ge == 0 && gl_bx_geometry(Ge, emb_in_dim / Ge, H / Ge, &gpc, &hgp, &stg);
    w.df_fc_emb = b.gl("enc.df_fc_emb.gl", G, I, ED, !w.fused_emb);
    if (w.fused_emb && (!w.df_fc_emb.img || !w.enc_in.bx) && !b.rc)
        b.rc = fail(DFB_ERR_INVALID, "df_fc_emb / enc.emb_gru.in: tensor-core weight images missing");
    if (c.g_enc_out) w.enc_out = b.gl("enc.emb_gru.out.gl", c.g_enc_out, H, ED);
    if (c.g_df_skip) w.df_skip = b.gl("df_dec.df_skip.gl", c.g_df_skip, emb_dim, Hd);
    w.df_in = b.gl("df_dec.df_gru.in.gl", c.g_df_in, emb_dim, Hd);
    w.df_out = b.gl("df_dec.df_out.gl", c.g_df_out, Hd, Fd * O2);
    w.erb_in = b.gl("erb_dec.emb_gru.in.gl", c.g_erb_in, emb_dim, H);
    w.erb_out = b.gl("erb_dec.emb_gru.out.gl", c.g_erb_out, H, ED);
    w.enc_gru = b.gru("enc.emb_gru", c.enc_gru_layers, H); w.df_gru = b.gru("df_dec.df_gru", c.df_gru_layers, Hd);
    w.erb_gru = b.gru("erb_dec.emb_gru", c.erb_gru_layers, H);
    w.lsnr = b.wb("enc.lsnr", emb_dim, 1); w.conv0_out = b.wb("erb_dec.conv0_out", c.conv_kt * 3 * kCh, 1);
    if (c.model_kind == 2) w.df_fc_a = b.wb("df_dec.df_fc_a", Hd, 1);
    if (df_convp_built(c.df_order, c.df_pathway_kt))
        w.df_convp = {b.need("df_dec.df_convp.w_sw", kCh * kCh), b.need("df_dec.df_convp.w2", O2 * O2), b.need("df_dec.df_convp.b", O2)};
    // a group width that is not a multiple of 4 has no tensor-core image and the FFMA kernel refuses it (run_gl): refuse
    // the model here instead of at its first forward pass
    const std::pair<const char *, const Gl *> gls[] = {{"df_fc_emb", &w.df_fc_emb}, {"enc.emb_gru.in", &w.enc_in}, {"enc.emb_gru.out", &w.enc_out},
                                                       {"df_dec.df_skip", &w.df_skip}, {"df_dec.df_gru.in", &w.df_in}, {"df_dec.df_out", &w.df_out},
                                                       {"erb_dec.emb_gru.in", &w.erb_in}, {"erb_dec.emb_gru.out", &w.erb_out}};
    for (const auto &g : gls)
        if (!b.rc && g.second->G > 0 && ((g.second->I / g.second->G) % 4 || (g.second->G > 1 && (g.second->H / g.second->G) % 4)))
            b.rc = fail(DFB_ERR_UNSUPPORTED, "grouped linear %s: %d x %d in %d groups (built kernels: group widths that are multiples of 4)",
                        g.first, g.second->I, g.second->H, g.second->G);
    return b.rc;
}

static int bind_v1(const dfb_model_config &c, Binder &b, NetWV1 &w) {
    const int Fd = c.nb_df, H = c.emb_hidden, O2 = 2 * c.df_order, N = Fd * O2, kt = c.conv_kt;
    w.ones = b.need("v1.ones", kCh); w.zeros = b.need("v1.zeros", kCh);
    auto idx = [&](const char *n, int numel) { return reinterpret_cast<const int *>(b.need(n, numel)); };
    w.idx_c1 = idx("v1.idx_c1", Fd / 2 * kCh); w.idx_e3 = idx("v1.idx_e3", H); w.idx_shuf = idx("v1.idx_shuf", H);
    w.idx_id = idx("v1.idx_id", H); w.idx_dec = idx("v1.idx_dec", H); w.idx_gshuf = idx("v1.idx_gshuf", H);
    // the tensor-core version of a block (pw_sw) is built for blocks without look-ahead whose transposed convs have one time tap
    auto blk = [&](const char *n, int mode, int bkt, int la) { return b.blk(n, bkt * 3 * kCh, true, la == 0 && !(mode == DW_T2 && bkt != 1)); };
    w.erb_conv1 = blk("enc.erb_conv1", DW_S2, kt, c.conv_lookahead > 1 ? 1 : 0); w.erb_conv2 = blk("enc.erb_conv2", DW_S2, kt, c.conv_lookahead > 2 ? 1 : 0);
    w.erb_conv3 = blk("enc.erb_conv3", DW_S1, kt, 0); w.df_conv1 = blk("enc.df_conv1", DW_S2, kt, 0);
    w.conv3p = blk("erb_dec.conv3p", DW_S1, 1, 0); w.conv2p = blk("erb_dec.conv2p", DW_S1, 1, 0);
    w.conv1p = blk("erb_dec.conv1p", DW_S1, 1, 0); w.conv0p = blk("erb_dec.conv0p", DW_S1, 1, 0);
    w.convt3 = blk("erb_dec.convt3", DW_S1, kt, 0); w.convt2 = blk("erb_dec.convt2", DW_T2, kt, 0); w.convt1 = blk("erb_dec.convt1", DW_T2, kt, 0);
    w.erb_conv0 = b.wb("enc.erb_conv0", c.inp_kt * 3 * kCh, kCh); w.df_conv0 = b.wb("enc.df_conv0", c.inp_kt * 3 * 2 * kCh, kCh);
    w.df_fc_emb = {b.need("enc.df_fc_emb.gl", (int64_t)Fd / 2 * kCh * H / c.g_df_fc_emb), b.need("enc.df_fc_emb.bias", H)};
    w.erb_fc_emb = {b.need("erb_dec.fc_emb.gl", (int64_t)H * H / c.g_erb_in), b.need("erb_dec.fc_emb.bias", H)};
    for (int l = 0; l < c.enc_gru_layers; l++) w.enc_gru.push_back(b.gru("enc.emb_gru.g" + std::to_string(l), 1, H)[0]);
    for (int l = 0; l < c.df_gru_layers; l++) w.df_gru.push_back(b.gru("df_dec.df_gru.g" + std::to_string(l), 1, H)[0]);
    w.lsnr = b.wb("enc.lsnr", H, 1); w.df_fc_a = b.wb("df_dec.df_fc_a", H, 1);
    const bool planes = b.opt("df_dec.df_fc_out.w_hi");  // BF16x3 GEMM operand, else the FFMA grouped linear reads w_t
    w.df_fc_out = {b.need("df_dec.df_fc_out.w_t", (int64_t)H * N), b.need("df_dec.df_fc_out.b", N),
                   planes ? b.need("df_dec.df_fc_out.w_hi", (int64_t)H * N / 2) : nullptr, planes ? b.need("df_dec.df_fc_out.w_lo", (int64_t)H * N / 2) : nullptr};
    w.df_convp = b.wb("df_dec.df_convp", kCh * O2, O2); w.conv0_out = b.wb("erb_dec.conv0_out", kt * 3 * kCh, 1);
    return b.rc;
}

extern "C" int dfb_model_create(dfb_model **out, int device, const dfb_model_config *cfg, const dfb_tensor *tensors,
                                int n_tensors, const int64_t *erb_widths) {
    if (!out || !cfg || !tensors) return fail(DFB_ERR_INVALID, "null argument");
    *out = nullptr;
    if (cfg->conv_ch != kCh) return fail(DFB_ERR_UNSUPPORTED, "conv_ch = %d (built kernels: 64)", cfg->conv_ch);
    if (cfg->model_kind < 1 || cfg->model_kind > 3) return fail(DFB_ERR_UNSUPPORTED, "model_kind %d", cfg->model_kind);
    if (cfg->model_kind == 1 && (cfg->emb_hidden != cfg->df_hidden || cfg->emb_hidden != cfg->nb_erb / 4 * kCh || cfg->conv_kt != 2 ||
                                 cfg->inp_kt != 2 || cfg->df_order != 5))
        return fail(DFB_ERR_UNSUPPORTED, "DeepFilterNet v1: only the shipped topology is built (hidden = conv_ch * nb_erb / 4, kt 2, order 5)");
    if (cfg->conv_kt < 1 || cfg->conv_kt > 2 || cfg->inp_kt < 1 || cfg->inp_kt > 3)
        return fail(DFB_ERR_UNSUPPORTED, "conv kernel time taps (%d, %d) unsupported", cfg->conv_kt, cfg->inp_kt);
    if ((cfg->emb_hidden != 256 && cfg->emb_hidden != 512) || (cfg->df_hidden != 256 && cfg->df_hidden != 512))
        return fail(DFB_ERR_UNSUPPORTED, "GRU hidden sizes (%d, %d): built kernels cover 256 and 512", cfg->emb_hidden,
                    cfg->df_hidden);
    if (cfg->nb_erb % 8 || cfg->nb_erb > 64 || cfg->nb_df % 8 || cfg->nb_df > 128 || 2 * cfg->df_order > kMaxO2)
        return fail(DFB_ERR_UNSUPPORTED, "nb_erb / nb_df / df_order outside the built kernels");
    // the input convs read feature frame t + conv_lookahead for every t >= 0 (k_conv_in), the deep filter frames
    // t - (df_order - 1 - df_lookahead) ... t + df_lookahead: a negative look-ahead would read before the buffers.  The
    // chunked and streaming paths are tested up to look-ahead 3 (tests/test_gpu_parity.py); DeepFilterNet v1 spreads its
    // conv look-ahead over erb_conv0-2 and is built for the shipped 2 only
    if (cfg->conv_lookahead < 0 || cfg->df_lookahead < 0 || cfg->conv_lookahead > kMaxLookahead || cfg->df_lookahead > kMaxLookahead ||
        (cfg->model_kind == 1 && cfg->conv_lookahead != 2))
        return fail(DFB_ERR_UNSUPPORTED, "look-ahead (conv %d, df %d): built kernels take look-aheads 0..%d (DeepFilterNet v1: conv 2)",
                    cfg->conv_lookahead, cfg->df_lookahead, kMaxLookahead);
    int rc = use_device(device);
    if (rc) return rc;
    dfb_model *m = new dfb_model();
    m->device = device;
    m->cfg = *cfg;
    if (erb_widths) m->erb_widths.assign(erb_widths, erb_widths + cfg->nb_erb);
    if (const char *e = getenv("DFB_DEVICE_CHUNKS")) m->dev_chunks = atoi(e) > 0 ? atoi(e) : 0;
    if (const char *e = getenv("DFB_HOST_CHUNKS")) m->host_chunks = atoi(e) > 0 ? atoi(e) : 1;
    if (const char *e = getenv("DFB_LANES")) m->n_lanes = atoi(e) == 1 ? 1 : 2;
    if (const char *e = getenv("DFB_MAX_WORKSPACE_MB")) {
        const long long mb = atoll(e);
        if (mb > 0) m->max_workspace = (size_t)mb << 20;
    }
    // upload: one slab
    size_t total = 0;
    for (int i = 0; i < n_tensors; i++) total += ((size_t)tensors[i].numel * 4 + 255) & ~size_t(255);
    if (cudaMalloc(&m->slab, total + 256) != cudaSuccess) {
        delete m;
        return fail(DFB_ERR_OOM, "cudaMalloc(%zu) for weights failed", total);
    }
    size_t off = 0;
    std::map<std::string, std::pair<const float *, int64_t>> t;
    for (int i = 0; i < n_tensors; i++) {
        const dfb_tensor &tt = tensors[i];
        if (!tt.name || !tt.data || tt.numel <= 0) { dfb_model_free(m); return fail(DFB_ERR_INVALID, "bad tensor %d", i); }
        float *dst = (float *)((char *)m->slab + off);
        if (cudaMemcpy(dst, tt.data, (size_t)tt.numel * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
            dfb_model_free(m);
            return fail(DFB_ERR_CUDA, "weight upload failed");
        }
        t[tt.name] = {dst, tt.numel};
        off += ((size_t)tt.numel * 4 + 255) & ~size_t(255);
    }
    m->fingerprint = model_fingerprint(*cfg, erb_widths, tensors, n_tensors);
    Binder b{t};
    if ((rc = cfg->model_kind == 1 ? bind_v1(*cfg, b, m->net1) : bind_net(*cfg, b, m->net))) {
        dfb_model_free(m);
        return rc;
    }
    int prio_least = 0, prio_greatest = 0;
    cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
    // numerically greater = lower priority; the encoder phase sits one level below the decoder phase
    int prio_enc = prio_greatest + 1;
    if (prio_enc > prio_least) prio_enc = prio_least;
    bool ok = cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaStreamCreateWithFlags(&m->h2d, cudaStreamNonBlocking) == cudaSuccess &&
              cudaStreamCreateWithFlags(&m->d2h, cudaStreamNonBlocking) == cudaSuccess;
    for (auto &L : m->lanes) {
        ok = ok && cudaStreamCreateWithPriority(&L.main, cudaStreamNonBlocking, prio_enc) == cudaSuccess &&
             cudaStreamCreateWithPriority(&L.hi, cudaStreamNonBlocking, prio_enc) == cudaSuccess &&
             cudaStreamCreateWithPriority(&L.aux, cudaStreamNonBlocking, prio_enc) == cudaSuccess &&
             cudaStreamCreateWithPriority(&L.dhi, cudaStreamNonBlocking, prio_greatest) == cudaSuccess &&
             cudaStreamCreateWithPriority(&L.daux, cudaStreamNonBlocking, prio_greatest) == cudaSuccess &&
             cudaStreamCreateWithPriority(&L.low, cudaStreamNonBlocking, prio_least) == cudaSuccess;
        for (cudaEvent_t *e : {&L.ev_fork, &L.ev_join, &L.ev_fork_enc, &L.ev_join_enc, &L.ev_in, &L.ev_out, &L.ev_c0, &L.ev_convp,
                               &L.ev_skip, &L.ev_done})
            ok = ok && cudaEventCreateWithFlags(e, cudaEventDisableTiming) == cudaSuccess;
    }
    if (!ok) {
        dfb_model_free(m);
        return fail(DFB_ERR_CUDA, "stream creation failed");
    }
    *out = m;
    return DFB_OK;
}

extern "C" void dfb_model_free(dfb_model *m) {
    if (!m) return;
    cudaSetDevice(m->device);
    m->arena.release();
    m->arena1.release();
    m->aux_arena.release();
    if (m->h2d) cudaStreamDestroy(m->h2d);
    if (m->d2h) cudaStreamDestroy(m->d2h);
    if (m->slab) cudaFree(m->slab);
    for (float *p : m->rate_taps) cudaFree(p);
    if (m->d_rate_dirs) cudaFree(m->d_rate_dirs);
    if (m->stream) cudaStreamDestroy(m->stream);
    for (auto &L : m->lanes) {
        for (cudaStream_t st : {L.main, L.hi, L.aux, L.dhi, L.daux, L.low})
            if (st) cudaStreamDestroy(st);
        for (cudaEvent_t e : {L.ev_fork, L.ev_join, L.ev_fork_enc, L.ev_join_enc, L.ev_in, L.ev_out, L.ev_c0, L.ev_convp, L.ev_skip, L.ev_done})
            if (e) cudaEventDestroy(e);
        if (L.rt) cudaFree(L.rt);
    }
    delete m;
}

// Debug: when `steps` > 0, every following GRU launch of at most `steps` steps stamps clock64() phases of CTA 0 into a
// device buffer [steps][8] (k_gru_tc: 0 step start, 1 state arrived, 2 MMAs done, 3 gates done, 4 slice sent; the kernel
// writes one row per step, so longer launches are not stamped); copies the rows of the armed buffer, at most `steps`
// of them, when called with h_out != NULL.
extern "C" int dfb_debug_gru_timing(dfb_model *m, int steps, long long *h_out) {
    if (!m) return fail(DFB_ERR_INVALID, "null model");
    cudaSetDevice(m->device);
    if (h_out && m->gru_dbg) {
        const int n = steps < m->gru_dbg_steps ? steps : m->gru_dbg_steps;
        DFB_CUDA(cudaDeviceSynchronize());
        if (n > 0) DFB_CUDA(cudaMemcpy(h_out, m->gru_dbg, sizeof(long long) * 8 * n, cudaMemcpyDeviceToHost));
    }
    if (m->gru_dbg) { cudaFree(m->gru_dbg); m->gru_dbg = nullptr; m->gru_dbg_steps = 0; }
    if (steps > 0 && !h_out) {
        DFB_CUDA(cudaMalloc(&m->gru_dbg, sizeof(long long) * 8 * steps));
        DFB_CUDA(cudaMemset(m->gru_dbg, 0, sizeof(long long) * 8 * steps));
        m->gru_dbg_steps = steps;
    }
    return DFB_OK;
}

extern "C" int64_t dfb_model_debug_fetch(dfb_model *m, const char *name, float *h_out, int64_t max_numel) {
    if (!m || !name || !h_out) return fail(DFB_ERR_INVALID, "null argument");
    auto it = m->dbg.find(name);
    if (it == m->dbg.end()) return fail(DFB_ERR_INVALID, "no activation named '%s'", name);
    int64_t n = it->second.second < max_numel ? it->second.second : max_numel;
    cudaSetDevice(m->device);
    if (cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpy(h_out, it->second.first, (size_t)n * 4, cudaMemcpyDeviceToHost) != cudaSuccess)
        return fail(DFB_ERR_CUDA, "debug fetch failed: %s", cudaGetErrorString(cudaGetLastError()));
    return n;
}

extern "C" int64_t dfb_model_workspace_bytes(const dfb_model *m) { return m ? (int64_t)m->arena.cap : 0; }

namespace {

int run_gl(cudaStream_t s, const float *x, int64_t ldx, const float *w, const float *bias, const float *res,
           int64_t ldr, float *y, int64_t ldy, int64_t M, int G, int I, int Hh, int act, float oscale = 1.f,
           float ooffset = 0.f, unsigned short *y_hi = nullptr, unsigned short *y_lo = nullptr) {
    GlParams p{x, ldx, w, bias, res, ldr, y, ldy, M, G, I / G, Hh / G, act, oscale, ooffset, y_hi, y_lo};
    if ((p.Ig % 4) || (ldx % 4)) return fail(DFB_ERR_UNSUPPORTED, "grouped linear: K not a multiple of 4");
    if (G > 1 && (p.Hg % 4)) return fail(DFB_ERR_UNSUPPORTED, "grouped linear: group width %d not a multiple of 4", p.Hg);
    int tiles = (p.Hg + kGlBN - 1) / kGlBN;
    int gpc = (p.Hg < kGlBN && kGlBN % p.Hg == 0) ? (kGlBN / p.Hg < G ? kGlBN / p.Hg : G) : 1;
    dim3 grid((unsigned)((M + kGlBM - 1) / kGlBM), (unsigned)(((G + gpc - 1) / gpc) * tiles));
    // DFB_PROF_DETAIL=1 splits the grouped linears by shape in the profile (I x H / G)
    static const bool detail = getenv("DFB_PROF_DETAIL") && atoi(getenv("DFB_PROF_DETAIL"));
    char name[64];
    if (detail) snprintf(name, sizeof name, "k_grouped_linear[%dx%d/%d]", I, Hh, G);
    else snprintf(name, sizeof name, "%s", p.G == 1 && p.bias && p.Hg >= 512 ? "k_grouped_linear[gru_proj]" : "k_grouped_linear");
    DFB_PROF(name, s);
    k_grouped_linear<<<grid, 256, 0, s>>>(p);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

// x [M, H] -> multi-layer GRU -> y [M, H]  (uses xproj scratch [M,3H] and h ping-pong buffers)
// x_hi/x_lo: BF16 planes of x (written by the producing grouped linear), pl_hi/pl_lo: scratch planes for the
// inter-layer hidden state, the input of the next layer's projection GEMM.
int run_gru(dfb_model *m, cudaStream_t s, const GruLayer *lw, int layers, int H, const float *res_last, float *y,
            float *xproj, int B, int T, const unsigned short *x_hi, const unsigned short *x_lo,
            unsigned short *pl_hi, unsigned short *pl_lo, int wide, unsigned short *out_hi, unsigned short *out_lo,
            bool *out_planes_ok, const GruChunk *ck) {
    if (out_planes_ok) *out_planes_ok = false;
    if (!x_hi || !x_lo || !pl_hi || !pl_lo) return fail(DFB_ERR_INVALID, "GRU: input planes and scratch planes are required");
    // time-chunked execution: the buffers hold T frames per stream, the recurrences run over frames [ck->t0, T) only and
    // continue from / leave behind the carried per-layer states; the projections simply cover every row
    const int t0 = ck ? ck->t0 : 0, Tn = T - t0;
    const int64_t M = (int64_t)B * T;
    const unsigned short *cur_hi = x_hi, *cur_lo = x_lo;
    for (int l = 0; l < layers; l++) {
        const GruLayer &g = lw[l];
        int rc;
        if ((rc = launch_gemm_bf16x3(s, cur_hi, cur_lo, H, g.w_ih_hi, g.w_ih_lo, g.b_ih, xproj, 3 * H, M, 3 * H, H))) return rc;
        const bool last = l == layers - 1;
        float *dst = last ? y : nullptr;   // a middle layer's output feeds only the next projection, which reads its planes
        float *hs = ck && ck->h ? ck->h + (int64_t)l * ck->Bs * H : nullptr;   // carried state of this layer [Bs][H], rows [0, B)
        GruWindow gw{ck && ck->have_state ? hs : nullptr, hs, t0, T, ck ? ck->first : nullptr, ck ? ck->w0 : 0, ck ? ck->run : nullptr};
        // the last layer's planes feed a grouped linear and include the residual; the others feed the next projection
        unsigned short *hi = last ? out_hi : pl_hi, *lo = last ? out_lo : pl_lo;
        if ((rc = launch_gru_tc(s, xproj, g.w_hh, g.b_hh, last ? res_last : nullptr, dst, hi, lo, B, Tn,
                                Tn <= m->gru_dbg_steps ? m->gru_dbg : nullptr, wide, last ? 1 : 0, &gw, H)))
            return rc;
        if (last && hi && out_planes_ok) *out_planes_ok = true;
        cur_hi = pl_hi; cur_lo = pl_lo;
        // middle layers may rewrite the scratch planes in place: the recurrence only reads xproj, which the
        // projection GEMM above has already produced from the previous contents of the planes.
    }
    return DFB_OK;
}

}  // namespace
namespace dfb {
template <int MODE>
int launch_dwpw_tc(cudaStream_t s, DwPwParams p, const float *w_sw, int B);
}
namespace {

template <int MODE>
int run_dwpw(cudaStream_t s, DwPwParams p, int B, const float *w_sw = nullptr) {
    if (w_sw) return launch_dwpw_tc<MODE>(s, p, w_sw, B);
    static PerDeviceOnce attr_once;
    const int smem = (kCh * kCh + 128 * kLdA) * 4;
    if (auto once_guard = attr_once.first()) {
        DFB_CUDA(cudaFuncSetAttribute(k_dwpw<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    }
    p.NF = 128 / p.Fout;
    if (p.NF < 1) p.NF = 1;
    if (p.NF * p.Fout > 128 || (p.NF * p.Fout) % 4) return fail(DFB_ERR_UNSUPPORTED, "dwpw tile: Fout = %d", p.Fout);
    dim3 grid((unsigned)((p.T + p.NF - 1) / p.NF), (unsigned)B);
    DFB_PROF("k_dwpw", s);
    k_dwpw<MODE><<<grid, 256, smem, s>>>(p);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

}  // namespace

// Buffers of one forward pass (all from the model arena).
struct FwdBufs {
    float *e0, *e1, *e2, *e3, *c0, *c1, *emb_in, *emb, *g_a, *g_b, *xproj, *dec_emb, *d3, *d2, *d1, *dfc;
    unsigned short *ga_hi, *ga_lo, *gh_hi, *gh_lo;  // BF16 planes of g_a / inter-layer h (tensor-core projections)
    // second set of GRU scratch: the DF decoder runs concurrently with the ERB decoder on another stream
    float *g_a2, *xproj2, *dfskip;
    unsigned short *ga2_hi, *ga2_lo, *gh2_hi, *gh2_lo;
    // BF16 hi / lo planes of the grouped linears' inputs (tensor-core path): c1, emb_in, GRU outputs, emb
    unsigned short *c1_hi, *c1_lo, *embin_hi, *embin_lo, *gb_hi, *gb_lo, *emb_hi, *emb_lo, *dfc_hi, *dfc_lo;
};

// DeepFilterNet v1 (forward_v1)
struct FwdBufsV1 {
    float *e0, *e1, *e2, *e3, *c0, *c1, *c1g, *cemb, *emb, *xproj, *xproj2, *y[3], *embo, *dec_old, *dec, *p3, *p2, *p1, *p0, *d3, *d2, *d1,
        *z[2], *dfc;
    unsigned short *emb_hi, *emb_lo, *y_hi[3], *y_lo[3], *embo_hi, *embo_lo, *z_hi[2], *z_lo[2], *dfc_hi, *dfc_lo, *scr_hi, *scr_lo;
};
static size_t fwd_plan_v1(const dfb_model_config &c, size_t M, Arena *a, FwdBufsV1 *f) {
    const int E = c.nb_erb, Fd = c.nb_df, H = c.emb_hidden;
    size_t bytes = 0;
    auto take = [&](size_t n) -> float * {
        bytes += (n * 4 + 255) & ~size_t(255);
        return a ? a->take<float>(n) : nullptr;
    };
    auto take16 = [&](size_t n) { return reinterpret_cast<unsigned short *>(take((n + 1) / 2)); };
    FwdBufsV1 t{};
    t.e0 = take(M * E * kCh); t.e1 = take(M * (E / 2) * kCh); t.e2 = take(M * (E / 4) * kCh); t.e3 = take(M * (E / 4) * kCh);
    t.c0 = take(M * Fd * kCh); t.c1 = take(M * (Fd / 2) * kCh); t.c1g = take(M * (Fd / 2) * kCh);
    t.cemb = take(M * H); t.emb = take(M * H); t.xproj = take(M * 3 * H); t.xproj2 = take(M * 3 * H);
    for (int i = 0; i < 3; i++) { t.y[i] = take(M * H); t.y_hi[i] = take16(M * H); t.y_lo[i] = take16(M * H); }
    for (int i = 0; i < 2; i++) { t.z[i] = take(M * H); t.z_hi[i] = take16(M * H); t.z_lo[i] = take16(M * H); }
    t.embo = take(M * H); t.dec_old = take(M * H); t.dec = take(M * H); t.dfc = take(M * H);
    t.p3 = take(M * (E / 4) * kCh); t.p2 = take(M * (E / 4) * kCh); t.p1 = take(M * (E / 2) * kCh); t.p0 = take(M * E * kCh);
    t.d3 = take(M * (E / 4) * kCh); t.d2 = take(M * (E / 2) * kCh); t.d1 = take(M * E * kCh);
    t.emb_hi = take16(M * H); t.emb_lo = take16(M * H); t.embo_hi = take16(M * H); t.embo_lo = take16(M * H);
    t.dfc_hi = take16(M * H); t.dfc_lo = take16(M * H); t.scr_hi = take16(M * H); t.scr_lo = take16(M * H);
    if (f) *f = t;
    return bytes + 4096;
}

// Carves the activations of `M` frames out of `a` (or only counts bytes when a == nullptr).
static size_t fwd_plan(const dfb_model_config &c, size_t M, Arena *a, FwdBufs *f) {
    if (c.model_kind == 1 && !a) return fwd_plan_v1(c, M, nullptr, nullptr);
    const int E = c.nb_erb, Fd = c.nb_df, H = c.emb_hidden, Hd = c.df_hidden;
    const int ED = E / 4 * kCh;
    const int emb_in_dim = c.enc_concat ? 2 * ED : ED;
    const int emb_dim = c.model_kind == 2 ? H : ED;
    const int Hmax = H > Hd ? H : Hd;
    size_t bytes = 0;
    auto take = [&](size_t n) -> float * {
        bytes += (n * 4 + 255) & ~size_t(255);
        return a ? a->take<float>(n) : nullptr;
    };
    FwdBufs t{};
    t.e0 = take(M * E * kCh); t.e1 = take(M * (E / 2) * kCh); t.e2 = take(M * (E / 4) * kCh);
    t.emb_in = take(M * emb_in_dim);
    t.e3 = c.enc_concat ? t.emb_in : take(M * ED);  // DFN2: e3 lives inside the concat buffer
    t.c0 = take(M * Fd * kCh); t.c1 = take(M * (Fd / 2) * kCh);
    t.emb = take(M * emb_dim);
    t.g_a = take(M * Hmax); t.g_b = take(M * Hmax);
    // the chunk planner sizes time windows by this plan's bytes per frame (so they decide the chunk boundaries, and with
    // them the output bits of long signals): buffers that the path no longer uses -- the GRU middle layers' fp32 outputs
    // here and below, c1's planes when k_dwpw_gl runs -- keep their place
    take(M * Hmax);
    t.xproj = take(M * 3 * Hmax);
    t.dec_emb = take(M * ED); t.d3 = take(M * ED); t.d2 = take(M * (E / 2) * kCh);
    t.d1 = take(M * E * kCh); t.dfc = take(M * Hmax);
    t.ga_hi = reinterpret_cast<unsigned short *>(take(M * Hmax / 2)); t.ga_lo = reinterpret_cast<unsigned short *>(take(M * Hmax / 2));
    t.gh_hi = reinterpret_cast<unsigned short *>(take(M * Hmax / 2)); t.gh_lo = reinterpret_cast<unsigned short *>(take(M * Hmax / 2));
    t.g_a2 = take(M * Hmax); take(M * Hmax); t.xproj2 = take(M * 3 * Hmax); t.dfskip = take(M * Hmax);
    t.ga2_hi = reinterpret_cast<unsigned short *>(take(M * Hmax / 2)); t.ga2_lo = reinterpret_cast<unsigned short *>(take(M * Hmax / 2));
    t.gh2_hi = reinterpret_cast<unsigned short *>(take(M * Hmax / 2)); t.gh2_lo = reinterpret_cast<unsigned short *>(take(M * Hmax / 2));
    auto take16 = [&](size_t n) { return reinterpret_cast<unsigned short *>(take((n + 1) / 2)); };
    t.c1_hi = take16(M * (Fd / 2) * kCh); t.c1_lo = take16(M * (Fd / 2) * kCh);
    t.embin_hi = take16(M * emb_in_dim); t.embin_lo = take16(M * emb_in_dim);
    t.gb_hi = take16(M * Hmax); t.gb_lo = take16(M * Hmax);
    t.emb_hi = take16(M * emb_dim); t.emb_lo = take16(M * emb_dim);
    t.dfc_hi = take16(M * Hmax); t.dfc_lo = take16(M * Hmax);
    if (f) *f = t;
    return bytes + 4096;
}

// Time-chunked execution (dfb_enhance's chunk loop, the streaming API): the window holds T frames per stream of which
// the first Rc were already processed by the previous chunk (halo: the feed-forward layers recompute them from the
// carried feature history, the recurrences skip them and continue from the carried hidden states).
struct ChunkCtx {
    int Rc;                        // halo frames at the head of the window
    int Tsx, Tx;                   // feature buffers: frames per stream, frames that exist (beyond = end of stream)
    float *h_enc, *h_erb, *h_df;   // carried GRU states [layers][B][H]
    bool have_state;               // false for the first chunk of a stream (states start at zero)
    float *dec_tail;               // (conv_kt == 2) last kHalo frames of dec_emb [B][kHalo][ED], right aligned
    int dec_tail_n;                // frames of dec_tail that are valid
    int lane;                      // which of the model's two stream / event sets (and arenas) this chunk runs on
    cudaEvent_t wait_dec;          // previous chunk finished (its decoder states / tails are final) or null
    int Bs;                        // streams the GRU states were allocated for (layer stride); the window runs rows [0, B)
    const RaggedRow *rows;         // ragged batch: per-stream frame counts (features end at rows[b].Tf), or null
    int64_t W0;                    // absolute frame of window row 0
    const int64_t *first;          // streaming slots: per-stream first frames (before them = padding), or null
    const struct GateRun *gate = nullptr;   // runtime gating mode, or null (apply mode: the decoders run every frame)
};
constexpr int kHalo = 8;           // >= temporal receptive field of every feed-forward chain of the shipped models

// ---- runtime gating mode (dfb_model_set_gating_mode, tract.rs:478-503): each decoder runs only on the frames the LSNR
// stage rule lets through, as if run alone on that subsequence.  The ERB decoder runs on frame t iff min <= lsnr <= max_erb,
// the DF decoder iff that holds and lsnr <= max_df (tract.rs:658-672), with the same comparisons as the apply kernel and
// k_spec_emit, so the stages applied and the frames run always agree.  Recurrences hold their state through the other
// frames (k_gru_tc HOLD); time-tap layers read the previous frames their decoder ran on: the DF pathway conv runs on each
// row's compacted run frames after the carried c0 of its last kt - 1 run frames, and (conv_kt == 2) the inputs of convt3 and
// of the mask head are filled forward from the ERB decoder's last run frame.
struct GateRun {
    const SlotCtl *ctl;            // per-row gating and thresholds, or null: every row gates with th when gate_all
    const LinkRow *links;          // link groups (channel 0 decides), or null
    float th[3];
    int gate_all;
    float *t_c0, *t_run;           // StreamState tails
    bool valid;                    // the tails hold the last DNN chunk's run frames; else it ran in apply mode, where every
                                   // frame ran: take them from the halo (frames before the window or a stream's start: zero)
    const unsigned char *halo;     // per row: 1 takes that row's tails from the halo, 0 from the tails; or null: !valid for all
};

struct GatePlan {
    const float *ll; const SlotCtl *ctl; const LinkRow *links; const int64_t *first;
    int64_t w0; float th[3]; int gate_all, T, Rc;
    unsigned char *erb_run, *df_run;   // [B][T] run flags of the window's new frames (halo rows: 1)
    int *erb_src;                      // [B][T] last ERB run frame <= t among the new frames, -1: none (the carried one)
    int *df_pos, *df_n;                // [B][T] DF run frames among the new frames before t; [B] their number
    // (conv_kt == 2) has_run [b * run_w]: the ERB decoder has run on a frame of stream b (carried; from_halo: every earlier
    // frame of the stream ran); erb_first [B]: the first frame the kt = 2 layers may read -- the stream's first frame once
    // the decoder has run, else its first run frame, so that the frames before it are padding, as tract's zero state is
    float *has_run; int run_w, from_halo;
    int64_t *erb_first;
    const unsigned char *halo;         // per-row from_halo (GateRun::halo), or null: from_halo for every row
};

// one CTA per row: flags in parallel over frame segments, then an exclusive scan of the segments' last ERB run frame and
// DF run count
__global__ void __launch_bounds__(256) k_gate_plan(GatePlan g) {
    __shared__ int s_last[256], s_cnt[256];
    const int b = blockIdx.x, tid = threadIdx.x, T = g.T;
    const int lb = g.links ? g.links[b].first : b;
    const bool gate = g.ctl ? g.ctl[b].gate != 0 : g.gate_all != 0;
    const float th0 = g.ctl ? g.ctl[b].th_min : g.th[0], th1 = g.ctl ? g.ctl[b].th_erb : g.th[1], th2 = g.ctl ? g.ctl[b].th_df : g.th[2];
    const int tf = stream_first(g.first, b, g.w0);
    const int per = (T - g.Rc + 255) / 256;
    const int t0 = g.Rc + tid * per, t1 = min(t0 + per, T);
    const int64_t row = (int64_t)b * T;
    for (int t = tid; t < g.Rc; t += 256) { g.erb_run[row + t] = 1; g.df_run[row + t] = 1; g.erb_src[row + t] = t; g.df_pos[row + t] = 0; }
    int last = -1, cnt = 0;
    for (int t = t0; t < t1; t++) {
        bool e = t >= tf, d = e;
        if (e && gate) {   // stage 2 or 3 of the apply kernel runs the ERB decoder, stage 3 also the DF decoder
            const float l = g.ll[(int64_t)lb * T + t];
            e = !(l < th0) && !(l > th1);
            d = e && !(l > th2);
        }
        g.erb_run[row + t] = e; g.df_run[row + t] = d;
        if (e) last = t;
        cnt += d;
    }
    int first_run = T;
    for (int t = t0; t < t1 && first_run == T; t++)
        if (g.erb_run[row + t]) first_run = t;
    s_last[tid] = last; s_cnt[tid] = cnt;
    __syncthreads();
    if (tid == 0) {
        int m = -1, c = 0;
        for (int i = 0; i < 256; i++) {
            const int lm = s_last[i], lc = s_cnt[i];
            s_last[i] = m; s_cnt[i] = c;
            if (lm > m) m = lm;
            c += lc;
        }
        g.df_n[b] = c;
    }
    __shared__ int s_first;
    if (tid == 0) s_first = T;
    __syncthreads();
    if (first_run < T) atomicMin(&s_first, first_run);
    __syncthreads();
    if (g.has_run && tid == 0) {
        float &h = g.has_run[(int64_t)b * g.run_w];
        const int64_t f0 = g.first ? g.first[b] : 0;
        const bool prev = (g.halo ? g.halo[b] : g.from_halo) ? g.Rc > 0 && g.w0 + g.Rc - 1 >= f0 : h != 0.f;
        g.erb_first[b] = prev ? f0 : g.w0 + s_first;
        h = prev || s_first < T ? 1.f : 0.f;
    }
    __syncthreads();
    last = s_last[tid]; cnt = s_cnt[tid];
    for (int t = t0; t < t1; t++) {
        if (g.erb_run[row + t]) last = t;
        g.erb_src[row + t] = last;
        g.df_pos[row + t] = cnt;
        cnt += g.df_run[row + t];
    }
}

// DF pathway input of the run frames, compacted: row b of P [B][Tp][W] is the c0 of its last K - 1 run frames before the
// window's new frames (the carried tail, or the halo: from_halo, or per row halo[b]), then c0 of its DF run frames among
// them.  grid (K - 1 + T - Rc, B)
__global__ void __launch_bounds__(256) k_gate_gather(const float *__restrict__ c0, const float *__restrict__ tail, float *__restrict__ P,
                                                     int T, int Rc, int K, int W, int Tp, const unsigned char *__restrict__ df_run,
                                                     const int *__restrict__ df_pos, int from_halo, const unsigned char *__restrict__ halo,
                                                     const int64_t *__restrict__ first, int64_t w0) {
    const int b = blockIdx.y, x = blockIdx.x;
    if (halo) from_halo = halo[b];
    const float4 *src = nullptr;
    int64_t dst;
    if (x < K - 1) {
        dst = (int64_t)b * Tp + x;
        if (!from_halo) src = reinterpret_cast<const float4 *>(tail + ((int64_t)b * (K - 1) + x) * W);
        else {
            const int t = Rc - (K - 1) + x;
            if (t >= 0 && t >= stream_first(first, b, w0)) src = reinterpret_cast<const float4 *>(c0 + ((int64_t)b * T + t) * W);
        }
    } else {
        const int t = Rc + x - (K - 1);
        if (!df_run[(int64_t)b * T + t]) return;
        dst = (int64_t)b * Tp + K - 1 + df_pos[(int64_t)b * T + t];
        src = reinterpret_cast<const float4 *>(c0 + ((int64_t)b * T + t) * W);
    }
    float4 *d = reinterpret_cast<float4 *>(P + dst * W);
    for (int i = threadIdx.x; i < W / 4; i += blockDim.x) d[i] = src ? src[i] : make_float4(0.f, 0.f, 0.f, 0.f);
}

// the compacted pathway term back to its frames (other frames, whose coefficients no stage applies: 0); grid (T, B)
__global__ void __launch_bounds__(256) k_gate_scatter(const float *__restrict__ Q, float *__restrict__ coefs, int T, int Rc, int K, int W,
                                                      int Tp, const unsigned char *__restrict__ df_run, const int *__restrict__ df_pos) {
    const int b = blockIdx.y, t = blockIdx.x;
    const int64_t i = (int64_t)b * T + t;
    const bool run = t >= Rc && df_run[i];
    const float *src = Q + ((int64_t)b * Tp + K - 1 + (run ? df_pos[i] : 0)) * W;
    float *dst = coefs + i * W;
    for (int k = threadIdx.x; k < W; k += blockDim.x) dst[k] = run ? src[k] : 0.f;
}

// the last K - 1 compacted rows (run frames) become the carried tail; grid (K - 1, B)
__global__ void __launch_bounds__(256) k_gate_tail(const float *__restrict__ P, float *__restrict__ tail, int K, int W, int Tp,
                                                   const int *__restrict__ df_n) {
    const int b = blockIdx.y, x = blockIdx.x;
    const float4 *src = reinterpret_cast<const float4 *>(P + ((int64_t)b * Tp + df_n[b] + x) * W);
    float4 *dst = reinterpret_cast<float4 *>(tail + ((int64_t)b * (K - 1) + x) * W);
    for (int i = threadIdx.x; i < W / 4; i += blockDim.x) dst[i] = src[i];
}

// (conv_kt == 2) the frames before a run frame, as the kt = 2 layers read them, are the ERB decoder's last run frame: fill
// rows [Rc - 1, T) of x [B][T][fs] (W values per frame) that are not run frames from the last run frame before them, or from
// the carried one (tail + off; from_halo, or per row halo[b]: row Rc - 1 as recomputed, zeros at a stream's start).  save:
// afterwards, copy row T - 1 to the carried one.  grid (T - Rc + 1, B)
struct FillSeg { float *x; int64_t fs; int W, off; };
__global__ void __launch_bounds__(256) k_gate_fill(FillSeg sg, float *__restrict__ tail, int tail_w, int T, int Rc,
                                                   const unsigned char *__restrict__ erb_run, const int *__restrict__ erb_src,
                                                   int from_halo, const unsigned char *__restrict__ halo, int save) {
    const int b = blockIdx.y;
    if (halo) from_halo = halo[b];
    float *trow = tail + (int64_t)b * tail_w + sg.off;
    float *xb = sg.x + (int64_t)b * T * sg.fs;
    if (save) {
        for (int k = threadIdx.x; k < sg.W; k += blockDim.x) trow[k] = xb[(int64_t)(T - 1) * sg.fs + k];
        return;
    }
    const int t = Rc - 1 + blockIdx.x;
    if (t < 0) return;
    const float *src;
    if (t == Rc - 1) {
        if (from_halo) return;
        src = trow;
    } else {
        if (erb_run[(int64_t)b * T + t]) return;
        const int j = erb_src[(int64_t)b * T + t];
        src = j >= 0 ? xb + (int64_t)j * sg.fs : from_halo ? (Rc > 0 ? xb + (int64_t)(Rc - 1) * sg.fs : nullptr) : trow;
    }
    for (int k = threadIdx.x; k < sg.W; k += blockDim.x) xb[(int64_t)t * sg.fs + k] = src ? src[k] : 0.f;
}

// grow-only device buffer of a lane (run flags + compacted pathway rows); the lane's decoder phases are serialised
static unsigned char *lane_rt(dfb_model::Lane &L, size_t bytes) {
    if (L.rt_cap < bytes) {
        if (L.rt) { cudaDeviceSynchronize(); cudaFree(L.rt); L.rt = nullptr; L.rt_cap = 0; }
        const size_t want = (bytes + bytes / 4 + (1u << 20)) & ~size_t((1u << 20) - 1);
        if (cudaMalloc(&L.rt, want) != cudaSuccess) { L.rt = nullptr; return nullptr; }
        L.rt_cap = want;
    }
    return L.rt;
}

static int forward_impl(dfb_model *m, Arena &arena, const float *d_feat_erb, const float *d_feat_spec, int B, int T,
                        float *d_m, float *d_coefs, float *d_lsnr, float *d_alpha, cudaStream_t s, ChunkCtx *cx = nullptr);

extern "C" int dfb_model_forward(dfb_model *m, const float *d_feat_erb, const float *d_feat_spec, int64_t B64,
                                 int64_t T64, float *d_m, float *d_coefs, float *d_lsnr, float *d_alpha,
                                 void *stream) {
    if (!m || !d_feat_erb || !d_feat_spec || !d_m || !d_coefs) return fail(DFB_ERR_INVALID, "null argument");
    if (B64 <= 0 || T64 <= 0) return DFB_OK;
    if (B64 > 65535) return fail(DFB_ERR_INVALID, "more than 65535 streams per call");
    DFB_CUDA(cudaSetDevice(m->device));
    int rc = m->arena.reserve(fwd_plan(m->cfg, (size_t)B64 * T64, nullptr, nullptr));
    if (rc) return rc;
    m->arena.reset();
    rc = forward_impl(m, m->arena, d_feat_erb, d_feat_spec, (int)B64, (int)T64, d_m, d_coefs, d_lsnr, d_alpha,
                      (cudaStream_t)stream);
    m->arena.reset();
    return rc;
}

static int forward_body(dfb_model *m, Arena &arena, const float *d_feat_erb, const float *d_feat_spec, int B, int T,
                        float *d_m, float *d_coefs, float *d_lsnr, float *d_alpha, cudaStream_t s_in, ChunkCtx *cx);

static int forward_v1(dfb_model *m, Arena &arena, const float *d_feat_erb, const float *d_feat_spec, int B, int T,
                      float *d_m, float *d_coefs, float *d_lsnr, float *d_alpha, cudaStream_t s_in, ChunkCtx *cx);

static int forward_impl(dfb_model *m, Arena &arena, const float *d_feat_erb, const float *d_feat_spec, int B, int T,
                        float *d_m, float *d_coefs, float *d_lsnr, float *d_alpha, cudaStream_t s_in, ChunkCtx *cx) {
    const int rc = m->cfg.model_kind == 1
        ? forward_v1(m, arena, d_feat_erb, d_feat_spec, B, T, d_m, d_coefs, d_lsnr, d_alpha, s_in, cx)
        : forward_body(m, arena, d_feat_erb, d_feat_spec, B, T, d_m, d_coefs, d_lsnr, d_alpha, s_in, cx);
    // a failed launch or CUDA call, or a shape the built kernels do not cover, returns early and may leave work on the
    // forked internal streams un-joined while the caller goes on to reuse the arena: drain the device before handing
    // the error back (error path only)
    if (rc) cudaDeviceSynchronize();
    return rc;
}

static int forward_body(dfb_model *m, Arena &arena, const float *d_feat_erb, const float *d_feat_spec, int B, int T,
                        float *d_m, float *d_coefs, float *d_lsnr, float *d_alpha, cudaStream_t s_in, ChunkCtx *cx) {
    const dfb_model_config &c = m->cfg;
    const NetW &w = m->net;
    const int Tsx = cx ? cx->Tsx : T, Tx = cx ? cx->Tx : T;
    const RaggedRow *rows = cx ? cx->rows : nullptr;
    const int64_t W0 = cx ? cx->W0 : 0;
    const int64_t *first = cx ? cx->first : nullptr;
    GruChunk ck_enc{cx ? cx->h_enc : nullptr, cx && cx->have_state, cx ? cx->Rc : 0, cx ? cx->Bs : B, first, W0};
    GruChunk ck_erb{cx ? cx->h_erb : nullptr, cx && cx->have_state, cx ? cx->Rc : 0, cx ? cx->Bs : B, first, W0};
    GruChunk ck_df{cx ? cx->h_df : nullptr, cx && cx->have_state, cx ? cx->Rc : 0, cx ? cx->Bs : B, first, W0};
    const GateRun *gate = cx ? cx->gate : nullptr;
    const int Rc = cx ? cx->Rc : 0;
    // DFB_SERIAL=1: everything on the caller's stream (profiling: per-kernel times without overlap)
    static const bool serial = getenv("DFB_SERIAL") && atoi(getenv("DFB_SERIAL"));
    dfb_model::Lane &L = m->lanes[cx ? cx->lane : 0];
    cudaStream_t s = serial ? s_in : L.hi;
    cudaStream_t sl = serial ? s_in : L.low;
    if (!serial) {
        DFB_CUDA(cudaEventRecord(L.ev_in, s_in));
        DFB_CUDA(cudaStreamWaitEvent(s, L.ev_in, 0));
    }
    auto finish = [&]() -> int {  // join the branches and hand the result back to the caller's stream
        DFB_CUDA(cudaStreamWaitEvent(s, L.ev_join, 0));
        if (!serial) {
            DFB_CUDA(cudaEventRecord(L.ev_out, s));
            DFB_CUDA(cudaStreamWaitEvent(s_in, L.ev_out, 0));
        }
        return DFB_OK;
    };
    const int64_t M = (int64_t)B * T;
    const int E = c.nb_erb, Fd = c.nb_df, H = c.emb_hidden, Hd = c.df_hidden;
    const int ED = E / 4 * kCh;  // embedding width (512)
    const int emb_in_dim = c.enc_concat ? 2 * ED : ED;
    const int emb_dim = c.model_kind == 2 ? H : ED;  // encoder output width
    int rc;
    FwdBufs f{};
    fwd_plan(c, (size_t)M, &arena, &f);
    if (!f.gh2_lo || !f.dfskip || !f.dfc_lo) return fail(DFB_ERR_OOM, "forward workspace exhausted for %lld frames", (long long)M);
    m->dbg.clear();
    m->dbg["e0"] = {f.e0, M * E * kCh}; m->dbg["e1"] = {f.e1, M * (E / 2) * kCh}; m->dbg["e2"] = {f.e2, M * (E / 4) * kCh};
    m->dbg["e3"] = {f.e3, c.enc_concat ? M * emb_in_dim : M * ED}; m->dbg["c0"] = {f.c0, M * Fd * kCh};
    m->dbg["c1"] = {f.c1, M * (Fd / 2) * kCh}; m->dbg["emb_in"] = {f.emb_in, M * emb_in_dim};
    m->dbg["emb"] = {f.emb, M * emb_dim}; m->dbg["dec_emb"] = {f.dec_emb, M * ED}; m->dbg["d3"] = {f.d3, M * ED};
    m->dbg["d2"] = {f.d2, M * (E / 2) * kCh}; m->dbg["d1"] = {f.d1, M * E * kCh}; m->dbg["dfc"] = {f.dfc, M * Hd};
    m->dbg["g_a"] = {f.g_a, M * (H > Hd ? H : Hd)}; m->dbg["g_b"] = {f.g_b, M * (H > Hd ? H : Hd)};
    m->dbg["xproj"] = {f.xproj, M * 3 * (H > Hd ? H : Hd)};
    // BF16 planes of emb_in, fetched as pairs of BF16 per float word
    m->dbg["emb_in_hi"] = {reinterpret_cast<const float *>(f.embin_hi), M * emb_in_dim / 2};
    m->dbg["emb_in_lo"] = {reinterpret_cast<const float *>(f.embin_lo), M * emb_in_dim / 2};
    // BF16 planes of the DF GRU's output (with its skip), the input df_out reads
    m->dbg["dfc_hi"] = {reinterpret_cast<const float *>(f.dfc_hi), M * Hd / 2};
    m->dbg["dfc_lo"] = {reinterpret_cast<const float *>(f.dfc_lo), M * Hd / 2};
    const int64_t e3_fs = c.enc_concat ? 2 * ED : ED;
    // fp32 activations that only feed the BF16 planes of a tensor-core consumer are not written (null): the input grouped
    // linears' g_a / g_a2 (DeepFilterNet2 adds them to the GRU output as a residual), the last-layer GRU outputs g_b (enc,
    // erb) and dfc (DeepFilterNet2's df_fc_a and skip read it); the GRUs' middle layers never write theirs (run_gru)
    const bool keep_ga = c.model_kind == 2;
    float *const enc_ga = w.enc_in.bx ? nullptr : f.g_a;
    float *const erb_ga = !keep_ga && w.erb_in.bx ? nullptr : f.g_a;
    float *const df_ga = !keep_ga && w.df_in.bx ? nullptr : f.g_a2;
    float *const enc_gb = w.enc_out.bx ? nullptr : f.g_b;
    float *const erb_gb = w.erb_out.bx ? nullptr : f.g_b;
    float *const dfc = c.model_kind != 2 && w.df_out.bx ? nullptr : f.dfc;
    if (!erb_ga) m->dbg.erase("g_a");
    if (!erb_gb) m->dbg.erase("g_b");
    if (!dfc) m->dbg.erase("dfc");
    // BF16 hi / lo planes [M][K] (row pitch `ld` elements) of a grouped linear's input; `ok` = already written by the producer
    struct Pl { unsigned short *hi, *lo; int64_t ld; bool ok; };
    Pl pl_c1{f.c1_hi, f.c1_lo, (int64_t)Fd / 2 * kCh, false}, pl_embin{f.embin_hi, f.embin_lo, emb_in_dim, false},
       pl_gb{f.gb_hi, f.gb_lo, H, false}, pl_emb{f.emb_hi, f.emb_lo, emb_dim, false}, pl_dfc{f.dfc_hi, f.dfc_lo, Hd, false},
       pl_ga{f.ga_hi, f.ga_lo, H, false}, pl_ga2{f.ga2_hi, f.ga2_lo, Hd, false};
    // planes of `x` for a tensor-core consumer: converts on `st` unless the producer already wrote them
    auto ensure_planes = [&](cudaStream_t st, const float *x, int64_t ldx, int K, Pl &pl) -> int {
        if (pl.ok) return DFB_OK;
        if (pl.ld != K) return fail(DFB_ERR_INVALID, "plane pitch mismatch");
        if (!x) return fail(DFB_ERR_INVALID, "planes requested of an activation whose fp32 form was not written");
        int r = launch_to_planes(st, x, ldx, M, K, pl.hi, pl.lo);
        if (!r) pl.ok = true;
        return r;
    };
    // grouped linear `g`: the BF16x3 tensor-core kernel when g.bx, else (or when that kernel cannot take the launch) the
    // FFMA kernel.  xin: planes of x (converted on demand); yout (optional): planes of y to produce,
    // ycol: column offset of y inside its plane buffer.  x / y may be null (fp32 form not written / not wanted) only where
    // g.bx holds: the FFMA kernel needs both, and a launch that cannot run without them is an error.
    auto gl = [&](cudaStream_t st, const Gl &g, const float *x, int64_t ldx, Pl *xin, int act,
                  const float *res, int64_t ldr, float *y, int64_t ldy, Pl *yout, int64_t ycol = 0) -> int {
        int r;
        unsigned short *yh = yout ? yout->hi + ycol : nullptr, *yl = yout ? yout->lo + ycol : nullptr;
        if (xin && g.bx) {
            if ((r = ensure_planes(st, x, ldx, g.I, *xin))) return r;
            r = launch_gl_bx(st, xin->hi, xin->lo, xin->ld, g.img, res, ldr, y, ldy, yh, yl, yout ? yout->ld : 0, M, g.G, g.I / g.G,
                             g.H / g.G, act, 1.f, 0.f);
            if (r != DFB_ERR_UNSUPPORTED) {
                if (!r && yout) yout->ok = true;
                return r;
            }
        }
        if (!x || !y)
            return fail(DFB_ERR_UNSUPPORTED, "grouped linear %dx%d/%d: the tensor-core kernel cannot take this launch and the fp32 %s "
                        "the FFMA kernel needs is not written", g.I, g.H, g.G, x ? "output" : "input");
        // NB: the FFMA kernel's plane output shares y's pitch, so it can only serve plane buffers with ld == ldy
        const bool ffma_planes = yout && yout->ld == ldy;
        r = run_gl(st, x, ldx, g.w, nullptr, res, ldr, y, ldy, M, g.G, g.I, g.H, act, 1.f, 0.f, ffma_planes ? yh : nullptr, ffma_planes ? yl : nullptr);
        if (!r && yout) yout->ok = ffma_planes;
        return r;
    };

    // ---- encoder (deepfilternet3.py:166-185)
    {
        dim3 grid((unsigned)((T + kInFrames - 1) / kInFrames), (unsigned)B);
        int smem = (kInFrames + c.inp_kt - 1) * (E + 2) * 4;
        DFB_PROF("k_conv_in[erb_conv0]", s);
        k_conv_in<1><<<grid, 256, smem, s>>>(d_feat_erb, w.erb_conv0.w, w.erb_conv0.b, f.e0, T, E, c.inp_kt, c.conv_lookahead, Tsx, Tx, 0, rows, W0, first);
        DFB_LAUNCH_CHECK();
    }
    // the DF-branch input convs run concurrently with the ERB-branch convs
    cudaStream_t sa = serial ? s : L.aux;
    DFB_CUDA(cudaEventRecord(L.ev_fork_enc, s));
    DFB_CUDA(cudaStreamWaitEvent(sa, L.ev_fork_enc, 0));
    // separable block k; its tensor-core kernel reads k.pw_sw, the swizzled BF16 hi | lo image of the [C_out][C_in] 1x1 weights
    auto mk = [&](const Blk &k, const float *in, int Fin, int64_t in_fs, float *out, int Fout, int64_t out_fs, int kt) {
        DwPwParams p{};
        p.in = in; p.Fin = Fin; p.in_fs = in_fs; p.out = out; p.Fout = Fout; p.out_fs = out_fs; p.kt = kt; p.T = T;
        p.lookahead = 0;
        p.first = first; p.w0 = W0; p.dw = k.dw; p.bias = k.b;
        return p;
    };
    {
        {
            dim3 grid((unsigned)((T + kInFrames - 1) / kInFrames), (unsigned)B);
            int smem = (kInFrames + c.inp_kt - 1) * (Fd + 2) * 2 * 4;
            DFB_PROF("k_conv_in[df_conv0]", sa);
            k_conv_in<2><<<grid, 256, smem, sa>>>(d_feat_spec, w.df_conv0.w, w.df_conv0.b, f.c0, T, Fd, c.inp_kt, c.conv_lookahead, Tsx, Tx, 0, rows, W0, first);
            DFB_LAUNCH_CHECK();
            DFB_CUDA(cudaEventRecord(L.ev_c0, sa));
        }
        if (w.fused_emb) m->dbg.erase("c1");
        if (!w.fused_emb) {
            DwPwParams p = mk(w.df_conv1, f.c0, Fd, (int64_t)Fd * kCh, f.c1, Fd / 2, (int64_t)Fd / 2 * kCh, c.conv_kt);
            // c1 only feeds df_fc_emb: its BF16 planes for the tensor-core kernel, and the fp32 tensor for the FFMA kernel,
            // which runs where df_fc_emb's shape has no tensor-core geometry (the planes alone left it reading unwritten c1)
            p.out_hi = pl_c1.hi; p.out_lo = pl_c1.lo; pl_c1.ok = true;
            if ((rc = run_dwpw<DW_S2>(sa, p, B, w.df_conv1.pw_sw))) return rc;
        }
        DFB_CUDA(cudaEventRecord(L.ev_join_enc, sa));
        // DF pathway conv (needs c0 only; its result is consumed by the very last DF-decoder kernel): on the
        // low-priority stream, so its CTAs only take SMs that the critical path -- the encoder convs now, the GRU
        // clusters later -- leaves idle (on the DF branch's own streams it delays df_fc_emb, which is on the critical path)
        if (!df_convp_built(c.df_order, c.df_pathway_kt))
            return fail(DFB_ERR_UNSUPPORTED, "df_order %d / df_pathway_kernel_size_t %d (built kernels: df_order 5, kt 1-5)",
                        c.df_order, c.df_pathway_kt);
        if (Fd % 2) return fail(DFB_ERR_UNSUPPORTED, "df pathway conv: odd nb_df");
        if (!gate) {   // (runtime gating mode: on the run frames only, after the gate plan below)
            DFB_CUDA(cudaStreamWaitEvent(sl, L.ev_c0, 0));
            // channel contraction on the tensor cores (BF16x3), shifted adds + 1x1 conv in the epilogue
            if ((rc = launch_df_convp_tc(sl, f.c0, w.df_convp.w_sw, w.df_convp.w2, w.df_convp.b, d_coefs, B, T, Fd, c.df_order,
                                         c.df_pathway_kt, first, W0)))
                return rc;
            DFB_CUDA(cudaEventRecord(L.ev_convp, sl));
        }
    }
    {
        DwPwParams p = mk(w.erb_conv1, f.e0, E, (int64_t)E * kCh, f.e1, E / 2, (int64_t)E / 2 * kCh, c.conv_kt);
        if ((rc = run_dwpw<DW_S2>(s, p, B, w.erb_conv1.pw_sw))) return rc;
        p = mk(w.erb_conv2, f.e1, E / 2, (int64_t)E / 2 * kCh, f.e2, E / 4, (int64_t)E / 4 * kCh, c.conv_kt);
        if ((rc = run_dwpw<DW_S2>(s, p, B, w.erb_conv2.pw_sw))) return rc;
        p = mk(w.erb_conv3, f.e2, E / 4, (int64_t)E / 4 * kCh, f.e3, E / 4, e3_fs, c.conv_kt);
        if (c.enc_concat) { p.out_hi = pl_embin.hi; p.out_lo = pl_embin.lo; }  // DFN2: e3 is the first half of emb_in
        if ((rc = run_dwpw<DW_S1>(s, p, B, w.erb_conv3.pw_sw))) return rc;

    }
    DFB_CUDA(cudaStreamWaitEvent(s, L.ev_join_enc, 0));  // c0 (and, unfused, c1's planes) ready
    {
        // cemb = relu(df_fc_emb(c1 flat)); emb_in = e3 flat + cemb  (DFN2: concat)
        const int I = Fd / 2 * kCh;
        if (w.fused_emb) {  // only emb_in's planes are written: enc.emb_gru.in reads nothing else
            const int G = c.g_df_fc_emb;
            rc = launch_df_emb(s, f.c0, M, T, Fd, c.conv_kt, w.df_conv1.dw, w.df_conv1.b, w.df_conv1.pw_sw, w.df_fc_emb.img, G, I / G, ED / G,
                               c.enc_concat ? nullptr : f.e3, ED, pl_embin.hi + (c.enc_concat ? ED : 0), pl_embin.lo + (c.enc_concat ? ED : 0),
                               pl_embin.ld, first, W0);
            if (!rc) pl_embin.ok = true;
            m->dbg.erase("emb_in");
        } else if (c.enc_concat) {  // the first half's planes were written by erb_conv3
            rc = gl(s, w.df_fc_emb, f.c1, I, &pl_c1, ACT_RELU, nullptr, 0, f.emb_in + ED, emb_in_dim, &pl_embin, ED);
        } else {
            rc = gl(s, w.df_fc_emb, f.c1, I, &pl_c1, ACT_RELU, f.e3, ED, f.emb_in, emb_in_dim, &pl_embin);
        }
        if (rc) return rc;
    }
    {
        // enc.emb_gru: linear_in + ReLU -> GRU -> [linear_out + ReLU]
        if ((rc = gl(s, w.enc_in, w.fused_emb ? nullptr : f.emb_in, emb_in_dim, &pl_embin, ACT_RELU, nullptr, 0, enc_ga, H, &pl_ga)))
            return rc;
        float *gout = c.g_enc_out ? enc_gb : f.emb;
        Pl &pl_gout = c.g_enc_out ? pl_gb : pl_emb;
        if ((rc = run_gru(m, s, w.enc_gru.data(), c.enc_gru_layers, H, nullptr, gout, f.xproj, B, T, f.ga_hi, f.ga_lo,
                          f.gh_hi, f.gh_lo, 0, pl_gout.hi, pl_gout.lo, &pl_gout.ok, cx ? &ck_enc : nullptr))) return rc;
        if (c.g_enc_out) {
            if ((rc = gl(s, w.enc_out, enc_gb, H, &pl_gb, ACT_RELU, nullptr, 0, f.emb, emb_dim, &pl_emb))) return rc;
        }
        // the decoders read emb's planes on two streams: make sure they exist before the fork
        if ((rc = ensure_planes(s, f.emb, emb_dim, emb_dim, pl_emb))) return rc;
        if (d_lsnr && (rc = run_gl(s, f.emb, emb_dim, w.lsnr.w, w.lsnr.b, nullptr, 0, d_lsnr, 1, M, 1, emb_dim, 1, ACT_SIGMOID, c.lsnr_scale,
                                   c.lsnr_offset)))
            return rc;
    }
    // runtime gating mode: which frames each decoder runs on, from the LSNR just computed
    const int Kp = c.df_pathway_kt, Wc = Fd * kCh, Wq = Fd * 2 * c.df_order, Tp = Kp - 1 + T - Rc;
    unsigned char *erb_run = nullptr, *df_run = nullptr;
    int *erb_src = nullptr, *df_pos = nullptr, *df_n = nullptr;
    float *gP = nullptr, *gQ = nullptr;
    const int tw_run = 2 * ED + 2 * E * kCh + 1;   // StreamState::t_run per row: dec_emb | e3 | d1 | e0 | has_run
    const int64_t *kt_first = first;               // first frames the ERB decoder's kt = 2 layers read from
    if (gate) {
        if (!d_lsnr) return fail(DFB_ERR_INVALID, "runtime gating without the LSNR head");
        auto al = [](size_t n) { return (n + 255) & ~size_t(255); };
        const size_t nf = (size_t)M, o1 = al(nf), o2 = o1 + al(nf), o3 = o2 + al(nf * 4), o4 = o3 + al(nf * 4), o5 = o4 + al((size_t)B * 4),
                     o6 = o5 + al((size_t)B * Tp * Wc * 4), o7 = o6 + al((size_t)B * Tp * Wq * 4), end = o7 + al((size_t)B * 8);
        unsigned char *rt = lane_rt(L, end);
        if (!rt) return fail(DFB_ERR_OOM, "runtime gating buffers (%zu bytes)", end);
        erb_run = rt; df_run = rt + o1; erb_src = reinterpret_cast<int *>(rt + o2); df_pos = reinterpret_cast<int *>(rt + o3);
        df_n = reinterpret_cast<int *>(rt + o4); gP = reinterpret_cast<float *>(rt + o5); gQ = reinterpret_cast<float *>(rt + o6);
        int64_t *erb_first = reinterpret_cast<int64_t *>(rt + o7);
        // the window's gating buffers; bytes and integers fetched as the float words that hold them (lane_rt's 256-byte
        // alignment keeps ceil(M / 4) words of the flag bytes in bounds)
        auto word = [](const void *p) { return reinterpret_cast<const float *>(p); };
        m->dbg["lsnr"] = {d_lsnr, M}; m->dbg["m"] = {d_m, M * E}; m->dbg["coefs"] = {d_coefs, (int64_t)M * Wq};
        m->dbg["gate_erb_run"] = {word(erb_run), (M + 3) / 4}; m->dbg["gate_df_run"] = {word(df_run), (M + 3) / 4};
        m->dbg["gate_erb_src"] = {word(erb_src), M}; m->dbg["gate_df_pos"] = {word(df_pos), M};
        m->dbg["gate_df_n"] = {word(df_n), B}; m->dbg["gate_erb_first"] = {word(erb_first), 2 * (int64_t)B};
        m->dbg["gate_P"] = {gP, (int64_t)B * Tp * Wc}; m->dbg["gate_Q"] = {gQ, (int64_t)B * Tp * Wq};
        // the ERB recurrence's output, as the BF16 planes erb_out reads (its fp32 form, g_b, is not always written)
        m->dbg["erb_gru_hi"] = {word(f.gb_hi), M * H / 2}; m->dbg["erb_gru_lo"] = {word(f.gb_lo), M * H / 2};
        GatePlan gp{d_lsnr, gate->ctl, gate->links, first, W0, {gate->th[0], gate->th[1], gate->th[2]}, gate->gate_all, T, Rc,
                    erb_run, df_run, erb_src, df_pos, df_n, c.conv_kt > 1 ? gate->t_run + tw_run - 1 : nullptr, tw_run,
                    gate->valid ? 0 : 1, erb_first, gate->halo};
        kt_first = erb_first;
        {
            dfb::ProfScope prof_scope__("k_gate_plan", s);   // (not on the enhancement path bench.py models: see launch_spec_ingest)
            k_gate_plan<<<B, 256, 0, s>>>(gp);
            DFB_LAUNCH_CHECK();
        }
        ck_erb.run = erb_run;
        ck_df.run = df_run;
        // the pathway conv over each row's compacted run frames, after the carried c0 of its last Kp - 1: on the
        // low-priority stream, beside the decoders' recurrences (it reads the tail the previous chunk's decoder phase wrote)
        DFB_CUDA(cudaEventRecord(L.ev_c0, s));
        DFB_CUDA(cudaStreamWaitEvent(sl, L.ev_c0, 0));
        if (cx->wait_dec) DFB_CUDA(cudaStreamWaitEvent(sl, cx->wait_dec, 0));
        {
            dfb::ProfScope prof_scope__("k_gate_gather", sl);   // (see k_gate_plan)
            k_gate_gather<<<dim3((unsigned)(Tp), (unsigned)B), 256, 0, sl>>>(f.c0, gate->t_c0, gP, T, Rc, Kp, Wc, Tp, df_run, df_pos,
                                                                           gate->valid ? 0 : 1, gate->halo, first, W0);
            DFB_LAUNCH_CHECK();
            if (Kp > 1) {
                k_gate_tail<<<dim3((unsigned)(Kp - 1), (unsigned)B), 256, 0, sl>>>(gP, gate->t_c0, Kp, Wc, Tp, df_n);
                DFB_LAUNCH_CHECK();
            }
        }
        if ((rc = launch_df_convp_tc(sl, gP, w.df_convp.w_sw, w.df_convp.w2, w.df_convp.b, gQ, B, Tp, Fd, c.df_order, Kp, nullptr, 0)))
            return rc;
        {
            dfb::ProfScope prof_scope__("k_gate_scatter", sl);   // (see k_gate_plan)
            k_gate_scatter<<<dim3((unsigned)T, (unsigned)B), 256, 0, sl>>>(gQ, d_coefs, T, Rc, Kp, Wq, Tp, df_run, df_pos);
            DFB_LAUNCH_CHECK();
        }
        DFB_CUDA(cudaEventRecord(L.ev_convp, sl));
    }
    // fork: the two decoders only share read-only encoder outputs
    // the encoder phase is done (ev_fork also tells the next time chunk that it may start); the decoder phase runs on the
    // lane's greatest-priority streams and, in the chunk pipeline, after the previous chunk's decoder has finished
    DFB_CUDA(cudaEventRecord(L.ev_fork, s));
    if (!serial) { s = L.dhi; sa = L.daux; DFB_CUDA(cudaStreamWaitEvent(s, L.ev_fork, 0)); }
    DFB_CUDA(cudaStreamWaitEvent(sa, L.ev_fork, 0));
    if (cx && cx->wait_dec) {
        DFB_CUDA(cudaStreamWaitEvent(s, cx->wait_dec, 0));
        DFB_CUDA(cudaStreamWaitEvent(sa, cx->wait_dec, 0));
    }
    // DFN3's grouped-linear skip around the DF GRU does not depend on the recurrence: evaluate it here (the ERB
    // branch has the slack) and let the last GRU layer add it as its output residual, instead of a kernel on the
    // DF branch's tail, which is the critical path of the decoder phase
    // the two decoders' recurrences run concurrently and only so many clusters of 8 CTAs are co-resident: one branch uses 32
    // streams per cluster for batches above 64 (DFB_WIDE_BRANCH=erb|df|both|none selects which, for experiments)
    static const char *wide_env = getenv("DFB_WIDE_BRANCH");
    const int wide_df = !wide_env || !strcmp(wide_env, "df") || !strcmp(wide_env, "both");
    const int wide_erb = wide_env && (!strcmp(wide_env, "erb") || !strcmp(wide_env, "both"));
    const bool early_skip = c.g_df_skip && c.model_kind != 2;
    if (early_skip) {
        if ((rc = gl(s, w.df_skip, f.emb, emb_dim, &pl_emb, ACT_NONE, nullptr, 0, f.dfskip, Hd, nullptr))) return rc;
        DFB_CUDA(cudaEventRecord(L.ev_skip, s));
    }
    // ---- DF decoder (deepfilternet3.py:323-331), on the auxiliary stream (forked after the encoder)
    {
        cudaStream_t s = sa;  // shadows the caller stream inside this block
        if ((rc = gl(s, w.df_in, f.emb, emb_dim, &pl_emb, ACT_RELU, nullptr, 0, df_ga, Hd, &pl_ga2))) return rc;
        const float *res = c.model_kind == 2 ? f.g_a2 : (early_skip ? f.dfskip : nullptr);
        if (early_skip) DFB_CUDA(cudaStreamWaitEvent(s, L.ev_skip, 0));
        if ((rc = run_gru(m, s, w.df_gru.data(), c.df_gru_layers, Hd, res, dfc, f.xproj2, B, T, f.ga2_hi, f.ga2_lo,
                          f.gh2_hi, f.gh2_lo, wide_df, pl_dfc.hi, pl_dfc.lo, &pl_dfc.ok, cx ? &ck_df : nullptr))) return rc;
        if (c.g_df_skip && !early_skip) {
            if ((rc = gl(s, w.df_skip, f.emb, emb_dim, &pl_emb, ACT_NONE, f.dfc, Hd, f.dfc, Hd, nullptr))) return rc;
            pl_dfc.ok = false;
        }
        if (d_alpha && c.model_kind == 2 &&  // alpha = sigmoid(df_fc_a(c)), deepfilternet2.py:368
            (rc = run_gl(s, f.dfc, Hd, w.df_fc_a.w, w.df_fc_a.b, nullptr, 0, d_alpha, 1, M, 1, Hd, 1, ACT_SIGMOID))) return rc;
        const int O2 = 2 * c.df_order;
        // coefs = tanh(df_out(c)) + df_convp(c0); the pathway term was written by k_df_convp_tc on the low-priority stream
        DFB_CUDA(cudaStreamWaitEvent(s, L.ev_convp, 0));
        if ((rc = gl(s, w.df_out, dfc, Hd, &pl_dfc, ACT_TANH, d_coefs, (int64_t)Fd * O2, d_coefs, (int64_t)Fd * O2, nullptr))) return rc;
    }
    DFB_CUDA(cudaEventRecord(L.ev_join, sa));
    // ---- ERB decoder (deepfilternet3.py:245-254)
    {
        if ((rc = gl(s, w.erb_in, f.emb, emb_dim, &pl_emb, ACT_RELU, nullptr, 0, erb_ga, H, &pl_ga))) return rc;
        // DFN2 (SqueezedGRU): identity skip around the GRU, y = GRU(x) + x  (modules.py:695-697)
        const float *res = c.model_kind == 2 ? f.g_a : nullptr;
        pl_gb.ok = false;
        if ((rc = run_gru(m, s, w.erb_gru.data(), c.erb_gru_layers, H, res, erb_gb, f.xproj, B, T, f.ga_hi, f.ga_lo,
                          f.gh_hi, f.gh_lo, wide_erb, pl_gb.hi, pl_gb.lo, &pl_gb.ok, cx ? &ck_erb : nullptr))) return rc;
        if ((rc = gl(s, w.erb_out, erb_gb, H, &pl_gb, ACT_RELU, nullptr, 0, f.dec_emb, ED, nullptr))) return rc;
        if (cx && cx->dec_tail && c.conv_kt > 1) {
            // kt = 2 decoder convs look one frame back into the halo, where this window's recurrence did not run: restore
            // dec_emb there from the previous chunk, then keep this window's last frames for the next one
            const size_t fb = sizeof(float) * ED;
            const int nl = cx->Rc < cx->dec_tail_n ? cx->Rc : cx->dec_tail_n;
            if (cx->have_state && nl > 0)
                DFB_CUDA(cudaMemcpy2DAsync(f.dec_emb + (size_t)(cx->Rc - nl) * ED, fb * T, cx->dec_tail + (size_t)(kHalo - nl) * ED,
                                           fb * kHalo, fb * nl, B, cudaMemcpyDeviceToDevice, s));
            const int ns = T < kHalo ? T : kHalo;
            DFB_CUDA(cudaMemcpy2DAsync(cx->dec_tail + (size_t)(kHalo - ns) * ED, fb * kHalo, f.dec_emb + (size_t)(T - ns) * ED, fb * T,
                                       fb * ns, B, cudaMemcpyDeviceToDevice, s));
            cx->dec_tail_n = ns;
        }
        // (runtime gating, kt = 2) convt3 and the mask head read the ERB decoder's previous run frame
        auto fill = [&](FillSeg sg, int save) -> int {
            dfb::ProfScope prof_scope__("k_gate_fill", s);   // (see k_gate_plan)
            k_gate_fill<<<dim3((unsigned)(save ? 1 : T - Rc + 1), (unsigned)B), 256, 0, s>>>(sg, gate->t_run, tw_run, T, Rc, erb_run, erb_src,
                                                                                          gate->valid ? 0 : 1, gate->halo, save);
            DFB_LAUNCH_CHECK();
            return DFB_OK;
        };
        const bool fill_kt = gate && c.conv_kt > 1;
        const FillSeg sg_dec{f.dec_emb, ED, ED, 0}, sg_e3{f.e3, e3_fs, ED, ED}, sg_d1{f.d1, (int64_t)E * kCh, E * kCh, 2 * ED},
                      sg_e0{f.e0, (int64_t)E * kCh, E * kCh, 2 * ED + E * kCh};
        if (fill_kt) {
            for (const FillSeg &sg : {sg_dec, sg_e3}) if ((rc = fill(sg, 0))) return rc;
            for (const FillSeg &sg : {sg_dec, sg_e3}) if ((rc = fill(sg, 1))) return rc;
        }
        DwPwParams p = mk(w.convt3, f.dec_emb, E / 4, ED, f.d3, E / 4, ED, c.conv_kt);
        p.first = kt_first;
        p.path = f.e3; p.path_fs = e3_fs; p.ps = w.conv3p.s; p.pb = w.conv3p.b;
        if ((rc = run_dwpw<DW_S1>(s, p, B, w.convt3.pw_sw))) return rc;
        p = mk(w.convt2, f.d3, E / 4, ED, f.d2, E / 2, (int64_t)E / 2 * kCh, 1);
        p.path = f.e2; p.path_fs = (int64_t)E / 4 * kCh; p.ps = w.conv2p.s; p.pb = w.conv2p.b;
        if ((rc = run_dwpw<DW_T2>(s, p, B, w.convt2.pw_sw))) return rc;
        p = mk(w.convt1, f.d2, E / 2, (int64_t)E / 2 * kCh, f.d1, E, (int64_t)E * kCh, 1);
        p.path = f.e1; p.path_fs = (int64_t)E / 2 * kCh; p.ps = w.conv1p.s; p.pb = w.conv1p.b;
        // kt = 1 models: the mask head is evaluated in convt1's epilogue and d1 never leaves the SM
        const bool fused_mask = c.conv_kt == 1 && 128 % E == 0;
        if (fused_mask) {
            p.mk_e0 = f.e0; p.mk_ps = w.conv0p.s; p.mk_pb = w.conv0p.b; p.mk_w = w.conv0_out.w; p.mk_bias = w.conv0_out.b; p.mk_out = d_m;
            p.out = nullptr;
            m->dbg.erase("d1");
        }
        if ((rc = run_dwpw<DW_T2>(s, p, B, w.convt1.pw_sw))) return rc;
        if (fused_mask) return finish();
        static PerDeviceOnce attr_once;
        int smem = (kMaskWarps * 2 * (E + 2) * kMaskLd + c.conv_kt * 3 * kCh) * 4;
        if (auto once_guard = attr_once.first()) {  // sized for the largest supported configuration (nb_erb 64, kt 2)
            DFB_CUDA(cudaFuncSetAttribute(k_mask_out, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (kMaskWarps * 2 * (64 + 2) * kMaskLd + 2 * 3 * kCh) * 4));
        }
        if (fill_kt) {
            for (const FillSeg &sg : {sg_d1, sg_e0}) if ((rc = fill(sg, 0))) return rc;
            for (const FillSeg &sg : {sg_d1, sg_e0}) if ((rc = fill(sg, 1))) return rc;
        }
        int per_cta = kMaskWarps * kMaskChunk;
        dim3 grid((unsigned)((T + per_cta - 1) / per_cta), (unsigned)B);
        DFB_PROF("k_mask_out", s);
        k_mask_out<<<grid, 32 * kMaskWarps, smem, s>>>(f.e0, f.d1, w.conv0p.s, w.conv0p.b, w.conv0_out.w, w.conv0_out.b, d_m, T, E, c.conv_kt, kt_first, W0);
        DFB_LAUNCH_CHECK();
    }
    return finish();
}

// ------------------------------------------------------------------ DeepFilterNet v1 ----
// deepfilternet.py:64-279.  Same kernels as the other models where the layer shapes coincide (input convs, separable conv
// blocks, GRU recurrence + projections, mask head); what differs is expressed around them:
//   * convkxf pads (k - 1 - lookahead, lookahead) frames inside the conv (modules.py:151-154): k_conv_in with tp_min =
//     -lookahead, the depthwise prologue with p.lookahead
//   * pathway convs are full 1x1 convs (depthwise 1x1 + 1x1 + BN + ReLU): the separable kernel with a one-tap depthwise
//   * decoder transposed convs have two time taps (reversed on upload)
//   * GroupedLinear (bias, shuffle) / GroupedGRU (G = 8, shuffle between layers, add_outputs): FFMA grouped linear with bias;
//     every GroupedGRULayer runs as ONE dense H-wide recurrence with block-diagonal weights (the shuffle of its input folded
//     into W_ih), the re-orderings and the sum of layer outputs are k_gather_sum passes
//   * df_fc_out is a dense H -> nb_df * 2 O linear (BF16x3 GEMM), tanh and the 1x1 pathway conv are added by k_convp_v1
//   * DfOp blends the deep-filtered DF bins with the masked spectrum by alpha (apply kernel)
// One window = the whole signal (pick_chunk): the in-conv look-ahead makes the zero padding at the END of the signal part of
// every layer, which a window that stops short of it cannot reproduce.
static int forward_v1(dfb_model *m, Arena &arena, const float *d_feat_erb, const float *d_feat_spec, int B, int T,
                      float *d_m, float *d_coefs, float *d_lsnr, float *d_alpha, cudaStream_t s_in, ChunkCtx *cx) {
    const dfb_model_config &c = m->cfg;
    const NetWV1 &w = m->net1;
    if (cx && (cx->Rc != 0 || cx->have_state)) return fail(DFB_ERR_UNSUPPORTED, "DeepFilterNet v1 runs as one window per signal");
    const int Tsx = cx ? cx->Tsx : T, Tx = cx ? cx->Tx : T;
    static const bool serial = getenv("DFB_SERIAL") && atoi(getenv("DFB_SERIAL"));
    dfb_model::Lane &L = m->lanes[cx ? cx->lane : 0];
    cudaStream_t s = serial ? s_in : L.hi, sa = serial ? s_in : L.aux;
    if (!serial) {
        DFB_CUDA(cudaEventRecord(L.ev_in, s_in));
        DFB_CUDA(cudaStreamWaitEvent(s, L.ev_in, 0));
    }
    const int64_t M = (int64_t)B * T;
    const int E = c.nb_erb, Fd = c.nb_df, H = c.emb_hidden, O2 = 2 * c.df_order, kt = c.conv_kt;
    int rc;
    FwdBufsV1 f{};
    fwd_plan_v1(c, (size_t)M, &arena, &f);
    if (!f.scr_lo) return fail(DFB_ERR_OOM, "forward workspace exhausted for %lld frames", (long long)M);
    m->dbg.clear();
    m->dbg["e0"] = {f.e0, M * E * kCh}; m->dbg["e1"] = {f.e1, M * (E / 2) * kCh}; m->dbg["e2"] = {f.e2, M * (E / 4) * kCh};
    m->dbg["e3"] = {f.e3, M * (E / 4) * kCh}; m->dbg["c0"] = {f.c0, M * Fd * kCh}; m->dbg["c1"] = {f.c1, M * (Fd / 2) * kCh};
    m->dbg["cemb"] = {f.cemb, M * H}; m->dbg["emb_in"] = {f.emb, M * H}; m->dbg["emb"] = {f.embo, M * H};
    m->dbg["dec_emb"] = {f.dec, M * H}; m->dbg["d3"] = {f.d3, M * (E / 4) * kCh}; m->dbg["d2"] = {f.d2, M * (E / 2) * kCh};
    m->dbg["d1"] = {f.d1, M * E * kCh}; m->dbg["dfc"] = {f.dfc, M * H}; m->dbg["y0"] = {f.y[0], M * H};
    // every GRU layer's output (y: encoder, z: DF decoder) and the decoder pathways, for the layer-by-layer tests
    for (int l = 1; l < c.enc_gru_layers && l < 3; l++) m->dbg["y" + std::to_string(l)] = {f.y[l], M * H};
    for (int l = 0; l < c.df_gru_layers && l < 2; l++) m->dbg["z" + std::to_string(l)] = {f.z[l], M * H};
    m->dbg["p3"] = {f.p3, M * (E / 4) * kCh}; m->dbg["p2"] = {f.p2, M * (E / 4) * kCh};
    m->dbg["p1"] = {f.p1, M * (E / 2) * kCh}; m->dbg["p0"] = {f.p0, M * E * kCh};
    auto gather = [&](cudaStream_t st, int n, const float *const *src, const int64_t *ld, const int *const *idx, int K, int relu,
                      float *out, unsigned short *hi, unsigned short *lo) -> int {
        GatherParams g{};
        for (int i = 0; i < n; i++) { g.src[i] = src[i]; g.ld[i] = ld[i]; g.idx[i] = idx[i]; }
        g.n = n; g.out = out; g.ldo = K; g.hi = hi; g.lo = lo; g.ldp = K; g.K = K; g.relu = relu;
        DFB_PROF("k_gather_sum", st);
        k_gather_sum<<<(unsigned)M, 256, 0, st>>>(g);
        DFB_LAUNCH_CHECK();
        return DFB_OK;
    };
    // separable block k: depthwise (kt x 3, look-ahead la) -> 1x1 -> BN -> ReLU, input = in (+ path); on the tensor-core
    // kernel where k.pw_sw is bound
    auto block = [&](cudaStream_t st, const Blk &k, int mode, const float *in, int Fin, float *out, int Fout, int bkt, int la,
                     const float *path) -> int {
        DwPwParams p{};
        p.dw = k.dw; p.pw = k.pw; p.bias = k.b; p.in = in; p.Fin = Fin; p.in_fs = (int64_t)Fin * kCh; p.out = out; p.Fout = Fout; p.out_fs = (int64_t)Fout * kCh; p.kt = bkt; p.T = T;
        p.lookahead = la;
        if (path) { p.path = path; p.path_fs = p.in_fs; p.ps = w.ones; p.pb = w.zeros; }   // the pathway tensor is already >= 0
        if (mode == DW_S1) return run_dwpw<DW_S1>(st, p, B, k.pw_sw);
        if (mode == DW_S2) return run_dwpw<DW_S2>(st, p, B, k.pw_sw);
        return run_dwpw<DW_T2>(st, p, B, k.pw_sw);
    };
    // ---- encoder, deepfilternet.py:122-141
    DFB_CUDA(cudaEventRecord(L.ev_fork_enc, s));
    DFB_CUDA(cudaStreamWaitEvent(sa, L.ev_fork_enc, 0));
    {
        dim3 grid((unsigned)((T + kInFrames - 1) / kInFrames), (unsigned)B);
        const int la = c.conv_lookahead > 0 ? 1 : 0;
        {
            DFB_PROF("k_conv_in[erb_conv0]", s);
            k_conv_in<1><<<grid, 256, (kInFrames + c.inp_kt - 1) * (E + 2) * 4, s>>>(d_feat_erb, w.erb_conv0.w, w.erb_conv0.b, f.e0, T, E, c.inp_kt, la,
                                                                                      Tsx, Tx, -la, nullptr, 0, nullptr);
            DFB_LAUNCH_CHECK();
        }
        DFB_PROF("k_conv_in[df_conv0]", sa);
        k_conv_in<2><<<grid, 256, (kInFrames + c.inp_kt - 1) * (Fd + 2) * 2 * 4, sa>>>(d_feat_spec, w.df_conv0.w, w.df_conv0.b, f.c0, T, Fd, c.inp_kt,
                                                                                      c.conv_lookahead, Tsx, Tx, -c.conv_lookahead, nullptr, 0, nullptr);
        DFB_LAUNCH_CHECK();
    }
    if ((rc = block(sa, w.df_conv1, DW_S2, f.c0, Fd, f.c1, Fd / 2, kt, 0, nullptr))) return rc;
    {   // cemb = df_fc_emb(c1 channel-major), pre-shuffle order
        const float *src[1] = {f.c1}; const int64_t ld[1] = {(int64_t)Fd / 2 * kCh}; const int *ix[1] = {w.idx_c1};
        if ((rc = gather(sa, 1, src, ld, ix, Fd / 2 * kCh, 0, f.c1g, nullptr, nullptr))) return rc;
        const int I = Fd / 2 * kCh;
        if ((rc = run_gl(sa, f.c1g, I, w.df_fc_emb.w, w.df_fc_emb.b, nullptr, 0, f.cemb, H, M, c.g_df_fc_emb, I, H, ACT_NONE))) return rc;
    }
    DFB_CUDA(cudaEventRecord(L.ev_join_enc, sa));
    if ((rc = block(s, w.erb_conv1, DW_S2, f.e0, E, f.e1, E / 2, kt, c.conv_lookahead > 1 ? 1 : 0, nullptr)) ||
        (rc = block(s, w.erb_conv2, DW_S2, f.e1, E / 2, f.e2, E / 4, kt, c.conv_lookahead > 2 ? 1 : 0, nullptr)) ||
        (rc = block(s, w.erb_conv3, DW_S1, f.e2, E / 4, f.e3, E / 4, kt, 0, nullptr)))
        return rc;
    DFB_CUDA(cudaStreamWaitEvent(s, L.ev_join_enc, 0));
    {   // emb = e3 (channel-major flatten) + shuffle(cemb)
        const float *src[2] = {f.e3, f.cemb}; const int64_t ld[2] = {H, H}; const int *ix[2] = {w.idx_e3, w.idx_shuf};
        if ((rc = gather(s, 2, src, ld, ix, H, 0, f.emb, f.emb_hi, f.emb_lo))) return rc;
    }
    // GroupedGRU: layer l as a dense recurrence, out = sum_l shuffle(y_l) (l < last) + y_last
    auto ggru = [&](cudaStream_t st, const GruLayer *g, int layers, unsigned short *x_hi, unsigned short *x_lo, float **y,
                    unsigned short **y_hi, unsigned short **y_lo, float *xproj, float *hbase, float *out, unsigned short *out_hi,
                    unsigned short *out_lo) -> int {
        unsigned short *ch = x_hi, *cl = x_lo;
        for (int l = 0; l < layers; l++) {
            GruChunk ck{hbase ? hbase + (int64_t)l * B * H : nullptr, false, 0, B, nullptr, 0};
            bool ok = false;
            int r = run_gru(m, st, &g[l], 1, H, nullptr, y[l], xproj, B, T, ch, cl, f.scr_hi, f.scr_lo, 0, y_hi[l], y_lo[l], &ok,
                            hbase ? &ck : nullptr);
            if (r) return r;
            ch = y_hi[l]; cl = y_lo[l];
        }
        const float *src[3]; int64_t ld[3]; const int *ix[3];
        for (int l = 0; l < layers; l++) { src[l] = y[l]; ld[l] = H; ix[l] = l == layers - 1 ? w.idx_id : w.idx_gshuf; }
        return gather(st, layers, src, ld, ix, H, 0, out, out_hi, out_lo);
    };
    if (c.enc_gru_layers > 3 || c.df_gru_layers > 2) return fail(DFB_ERR_UNSUPPORTED, "DeepFilterNet v1: more GRU layers than built (3 / 2)");
    if ((rc = ggru(s, w.enc_gru.data(), c.enc_gru_layers, f.emb_hi, f.emb_lo, f.y, f.y_hi, f.y_lo, f.xproj, cx ? cx->h_enc : nullptr, f.embo,
                   f.embo_hi, f.embo_lo)))
        return rc;
    if (d_lsnr && (rc = run_gl(s, f.embo, H, w.lsnr.w, w.lsnr.b, nullptr, 0, d_lsnr, 1, M, 1, H, 1, ACT_SIGMOID, c.lsnr_scale, c.lsnr_offset)))
        return rc;
    DFB_CUDA(cudaEventRecord(L.ev_fork, s));
    if (!serial) { s = L.dhi; sa = L.daux; DFB_CUDA(cudaStreamWaitEvent(s, L.ev_fork, 0)); }
    DFB_CUDA(cudaStreamWaitEvent(sa, L.ev_fork, 0));
    // ---- DF decoder, deepfilternet.py:219-229 (auxiliary stream)
    {
        if ((rc = ggru(sa, w.df_gru.data(), c.df_gru_layers, f.embo_hi, f.embo_lo, f.z, f.z_hi, f.z_lo, f.xproj2, cx ? cx->h_df : nullptr, f.dfc,
                       f.dfc_hi, f.dfc_lo)))
            return rc;
        if (d_alpha && (rc = run_gl(sa, f.dfc, H, w.df_fc_a.w, w.df_fc_a.b, nullptr, 0, d_alpha, 1, M, 1, H, 1, ACT_SIGMOID))) return rc;
        const int N = Fd * O2;
        rc = DFB_ERR_UNSUPPORTED;
        if (w.df_fc_out.w_hi) rc = launch_gemm_bf16x3(sa, f.dfc_hi, f.dfc_lo, H, w.df_fc_out.w_hi, w.df_fc_out.w_lo, w.df_fc_out.b, d_coefs, N, M, N, H);
        if (rc == DFB_ERR_UNSUPPORTED) rc = run_gl(sa, f.dfc, H, w.df_fc_out.w_t, w.df_fc_out.b, nullptr, 0, d_coefs, N, M, 1, H, N, ACT_NONE);
        if (rc) return rc;
        const long long rows = (long long)M * Fd;
        DFB_PROF("k_convp_v1", sa);
        k_convp_v1<10><<<(unsigned)((rows + 127) / 128), 128, 0, sa>>>(f.c0, w.df_convp.w, w.df_convp.b, d_coefs, rows);
        DFB_LAUNCH_CHECK();
    }
    DFB_CUDA(cudaEventRecord(L.ev_join, sa));
    // ---- ERB decoder, deepfilternet.py:179-189
    {
        if ((rc = run_gl(s, f.embo, H, w.erb_fc_emb.w, w.erb_fc_emb.b, nullptr, 0, f.dec_old, H, M, c.g_erb_in, H, H, ACT_RELU))) return rc;
        const float *src[1] = {f.dec_old}; const int64_t ld[1] = {H}; const int *ix[1] = {w.idx_dec};
        if ((rc = gather(s, 1, src, ld, ix, H, 0, f.dec, nullptr, nullptr))) return rc;
        if ((rc = block(s, w.conv3p, DW_S1, f.e3, E / 4, f.p3, E / 4, 1, 0, nullptr)) ||
            (rc = block(s, w.conv2p, DW_S1, f.e2, E / 4, f.p2, E / 4, 1, 0, nullptr)) ||
            (rc = block(s, w.conv1p, DW_S1, f.e1, E / 2, f.p1, E / 2, 1, 0, nullptr)) ||
            (rc = block(s, w.conv0p, DW_S1, f.e0, E, f.p0, E, 1, 0, nullptr)))
            return rc;
        if ((rc = block(s, w.convt3, DW_S1, f.dec, E / 4, f.d3, E / 4, kt, 0, f.p3)) ||
            (rc = block(s, w.convt2, DW_T2, f.d3, E / 4, f.d2, E / 2, kt, 0, f.p2)) ||
            (rc = block(s, w.convt1, DW_T2, f.d2, E / 2, f.d1, E, kt, 0, f.p1)))
            return rc;
        static PerDeviceOnce attr_once;
        const int smem = (kMaskWarps * 2 * (E + 2) * kMaskLd + kt * 3 * kCh) * 4;
        if (auto once_guard = attr_once.first()) {
            DFB_CUDA(cudaFuncSetAttribute(k_mask_out, cudaFuncAttributeMaxDynamicSharedMemorySize, (kMaskWarps * 2 * (64 + 2) * kMaskLd + 2 * 3 * kCh) * 4));
        }
        const int per_cta = kMaskWarps * kMaskChunk;
        dim3 grid((unsigned)((T + per_cta - 1) / per_cta), (unsigned)B);
        DFB_PROF("k_mask_out", s);
        k_mask_out<<<grid, 32 * kMaskWarps, smem, s>>>(f.p0, f.d1, w.ones, w.zeros, w.conv0_out.w, w.conv0_out.b, d_m, T, E, kt, nullptr, 0);
        DFB_LAUNCH_CHECK();
    }
    DFB_CUDA(cudaStreamWaitEvent(s, L.ev_join, 0));
    if (!serial) {
        DFB_CUDA(cudaEventRecord(L.ev_out, s));
        DFB_CUDA(cudaStreamWaitEvent(s_in, L.ev_out, 0));
    }
    return DFB_OK;
}

// Chunk pipeline of dfb_enhance / dfb_enhance_host: signals of at least 64 * chunks frames are cut into >= `chunks` time
// chunks (device-pointer / host-pointer entry point); lanes = 2 overlaps the encoder phase of chunk c + 1 with the decoder
// phase of chunk c, lanes = 1 runs the chunks back to back.  Defaults auto / 4 / 2 (DFB_DEVICE_CHUNKS, DFB_HOST_CHUNKS,
// DFB_LANES at dfb_model_create); device_chunks = 0 (auto) is 3 chunks up to 8 streams, 2 up to 256, else 1.
extern "C" int dfb_model_set_chunking(dfb_model *m, int device_chunks, int host_chunks, int lanes) {
    if (!m || device_chunks < 0 || host_chunks < 1 || lanes < 1 || lanes > 2) return fail(DFB_ERR_INVALID, "bad chunking parameters");
    m->dev_chunks = device_chunks; m->host_chunks = host_chunks; m->n_lanes = lanes;
    return DFB_OK;
}

// The workspace is sized from the model's band layout but the DSP kernels index with the state's: they must agree.
static int check_state(const dfb_model *m, const dfb_state *st) {
    if (m->device != st->device) return fail(DFB_ERR_INVALID, "model and state live on different devices");
    if (st->fft != 960 || st->hop != 480)
        return fail(DFB_ERR_UNSUPPORTED, "the model path is built for fft_size 960 / hop_size 480 (DSP state: %d / %d)", st->fft,
                    st->hop);
    if (st->tb.E != m->cfg.nb_erb)
        return fail(DFB_ERR_INVALID, "DF state has %d ERB bands, the model was built for %d", st->tb.E, m->cfg.nb_erb);
    if (!m->erb_widths.empty())
        for (int i = 0; i < m->cfg.nb_erb; i++)
            if (m->erb_widths[i] != st->erb[i])
                return fail(DFB_ERR_INVALID, "DF state's ERB band %d is %lld bins wide, the model was built for %lld", i,
                            (long long)st->erb[i], (long long)m->erb_widths[i]);
    return DFB_OK;
}

static int apply_mode(const dfb_model *m) { return m->cfg.model_kind == 3 ? 1 : 2; }   // v1 / v2 filter the masked spectrum
static void apply_options(const dfb_model *m, dfb::ApplyParams &p) {
    p.pf = m->post_filter; p.pf_beta = m->pf_beta; p.mask_only = m->mask_only;
}

// init_df(post_filter=..., mask_only=...) (df/enhance.py:101-187): the post filter of deepfilternet3.py:448-454 (beta =
// pf_beta) or, for DeepFilterNet2, Mask.pf on the ERB gains (modules.py:234-245, beta fixed at 0.02); mask_only = the
// model built with run_df = False (checkpoint.py:32): no deep filtering stage.
extern "C" int dfb_model_set_gating_mode(dfb_model *m, int mode) {
    if (!m) return fail(DFB_ERR_INVALID, "null model");
    if (mode != DFB_GATING_APPLY && mode != DFB_GATING_RUNTIME) return fail(DFB_ERR_INVALID, "gating mode %d", mode);
    m->gating_mode = mode;
    return DFB_OK;
}

extern "C" int dfb_model_set_options(dfb_model *m, int post_filter, float pf_beta, int mask_only) {
    if (!m) return fail(DFB_ERR_INVALID, "null model");
    m->post_filter = post_filter ? 1 : 0;
    m->pf_beta = pf_beta;
    m->mask_only = mask_only ? 1 : 0;
    return DFB_OK;
}

static int apply_impl(dfb_model *m, dfb_state *st, const float *d_spec, const float *d_m, const float *d_coefs, const float *d_alpha,
                      int64_t B, int64_t T, float *d_spec_e, void *stream);
extern "C" int dfb_apply(dfb_model *m, dfb_state *st, const float *d_spec, const float *d_m, const float *d_coefs,
                         int64_t B, int64_t T, float *d_spec_e, void *stream) {
    if (m && m->cfg.model_kind == 1 && !m->mask_only)
        return fail(DFB_ERR_UNSUPPORTED, "DeepFilterNet v1 blends with df_alpha: use dfb_model_forward_full / dfb_enhance");
    return apply_impl(m, st, d_spec, d_m, d_coefs, nullptr, B, T, d_spec_e, stream);
}
static int apply_impl(dfb_model *m, dfb_state *st, const float *d_spec, const float *d_m, const float *d_coefs, const float *d_alpha,
                      int64_t B, int64_t T, float *d_spec_e, void *stream) {
    if (!m || !st || !d_spec || !d_m || !d_coefs || !d_spec_e) return fail(DFB_ERR_INVALID, "null argument");
    if (int rcs = check_state(m, st)) return rcs;
    DFB_CUDA(cudaSetDevice(m->device));
    dfb::ApplyParams p{};
    p.spec = (const float2 *)d_spec; p.m = d_m; p.coefs = d_coefs; p.audio = nullptr; p.spec_out = (float2 *)d_spec_e;
    p.Tf = (int)T; p.mode = apply_mode(m); p.nb_df = m->cfg.nb_df; p.order = m->cfg.df_order; p.lookahead = m->cfg.df_lookahead;
    p.alpha = d_alpha;
    apply_options(m, p);
    return launch_apply_synthesis(st, p, B, (cudaStream_t)stream);
}

// Debug aid: one launch_apply_synthesis with every field of ApplyParams the batch and slot executors set, the tables copied
// from the host; it picks the kernel instance exactly as those executors' launches do (include/dfb200.h).
extern "C" int dfb_debug_apply_rows(dfb_model *m, dfb_state *st, const float *d_spec, int spec_T, int Tv, const float *d_m,
                                    const float *d_coefs, const float *d_alpha, const float *d_lsnr, int mc_T, int64_t B, int Tf,
                                    int t_first, int t_emit, int64_t w0, const int64_t *h_rows, const int64_t *h_first,
                                    const int32_t *h_links, int reduce, const float *h_ctl, const int64_t *h_ctl_sw,
                                    const int32_t *h_ctl_gate, float th_min, float th_erb, float th_df, float atten_lim,
                                    int64_t out_offset, int64_t out_len, float *d_audio, float *d_spec_out, void *stream) {
    if (!m || !st || !d_spec || !d_m || !d_coefs || (!d_audio && !d_spec_out)) return fail(DFB_ERR_INVALID, "null argument");
    if (int rcs = check_state(m, st)) return rcs;
    if (B <= 0 || B > 65535 || Tf <= 0 || spec_T < 0 || (spec_T && spec_T < Tf) || Tv < 0 || Tv > (spec_T ? spec_T : Tf) ||
        mc_T < 0 || (mc_T && mc_T < Tf) || t_first < 0 || t_emit < 0 || t_emit > Tf || w0 < 0 || out_len < 0)
        return fail(DFB_ERR_INVALID, "bad geometry");
    if ((m->cfg.model_kind == 1) != (d_alpha != nullptr))
        return fail(DFB_ERR_INVALID, "alpha is DeepFilterNet v1's, and v1 needs it");
    if (!h_rows && (h_first || h_links || h_ctl)) return fail(DFB_ERR_INVALID, "first, links and settings need the row table");
    if (h_ctl && (!h_ctl_sw || !h_ctl_gate)) return fail(DFB_ERR_INVALID, "settings need their switch frames and gate flags");
    std::vector<RaggedRow> rows;
    std::vector<LinkRow> links;
    std::vector<SlotCtl> ctl;
    for (int64_t b = 0; h_rows && b < B; b++) {
        const int64_t *r = h_rows + 3 * b;
        if (r[0] < 0 || r[1] < 0 || r[2] < w0 || r[2] - w0 > INT32_MAX) return fail(DFB_ERR_INVALID, "bad row %lld", (long long)b);
        rows.push_back(RaggedRow{0, 0, r[0], r[1], r[2]});
        if (h_links) {
            const int32_t f = h_links[2 * b], n = h_links[2 * b + 1];
            if (n < 1 || f < 0 || f > b || b >= (int64_t)f + n || (int64_t)f + n > B)
                return fail(DFB_ERR_INVALID, "bad link group of row %lld", (long long)b);
            links.push_back(LinkRow{f, n});
        }
        if (h_ctl) {
            const float *c = h_ctl + 7 * b;
            ctl.push_back(SlotCtl{c[0], c[1], c[2], c[3], h_ctl_sw[b], c[4], c[5], c[6], h_ctl_gate[b]});
        }
    }
    DFB_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = (cudaStream_t)stream;
    const size_t o_first = sizeof(RaggedRow) * rows.size(), o_links = o_first + (h_first ? sizeof(int64_t) * B : 0),
                 o_ctl = o_links + sizeof(LinkRow) * links.size(), total = o_ctl + sizeof(SlotCtl) * ctl.size();
    std::vector<char> slab(total);
    if (!rows.empty()) memcpy(slab.data(), rows.data(), o_first);
    if (h_first) memcpy(slab.data() + o_first, h_first, sizeof(int64_t) * B);
    if (!links.empty()) memcpy(slab.data() + o_links, links.data(), sizeof(LinkRow) * links.size());
    if (!ctl.empty()) memcpy(slab.data() + o_ctl, ctl.data(), sizeof(SlotCtl) * ctl.size());
    char *d = nullptr;
    if (total && (cudaMalloc(&d, total) != cudaSuccess || cudaMemcpyAsync(d, slab.data(), total, cudaMemcpyHostToDevice, s) != cudaSuccess)) {
        if (d) cudaFree(d);
        return fail(DFB_ERR_OOM, "debug tables");
    }
    dfb::ApplyParams p{};
    p.spec = (const float2 *)d_spec; p.m = d_m; p.coefs = d_coefs; p.audio = d_audio; p.spec_out = (float2 *)d_spec_out;
    p.out_stride = out_len; p.out_len = out_len; p.out_offset = out_offset;
    p.Tf = Tf; p.spec_T = spec_T; p.Tv = Tv; p.mc_T = mc_T; p.t_first = t_first;
    p.mode = apply_mode(m); p.nb_df = m->cfg.nb_df; p.order = m->cfg.df_order; p.lookahead = m->cfg.df_lookahead;
    p.atten_lim = atten_lim; p.alpha = d_alpha;
    apply_options(m, p);
    p.lsnr = d_lsnr; p.th_min = th_min; p.th_erb = th_erb; p.th_df = th_df;
    p.rows = h_rows ? (const RaggedRow *)d : nullptr; p.w0 = w0; p.t_emit = t_emit;
    p.first = h_first ? (const int64_t *)(d + o_first) : nullptr;
    if (h_links) { p.links = (const LinkRow *)(d + o_links); p.reduce = reduce; }
    const int rc = launch_apply_synthesis(st, p, B, s, h_ctl ? (const SlotCtl *)(d + o_ctl) : nullptr);
    cudaStreamSynchronize(s);
    if (d) cudaFree(d);
    return rc;
}

extern "C" int dfb_model_forward_full(dfb_model *m, dfb_state *st, const float *d_spec, const float *d_feat_erb,
                                      const float *d_feat_spec, int64_t B, int64_t T, float *d_spec_e, float *d_m,
                                      float *d_lsnr, float *d_coefs, float *d_alpha, void *stream) {
    if (!m || !st || !d_spec || !d_feat_erb || !d_feat_spec || !d_spec_e) return fail(DFB_ERR_INVALID, "null argument");
    if (int rcs = check_state(m, st)) return rcs;
    DFB_CUDA(cudaSetDevice(m->device));
    const int64_t M = B * T;
    const int O2 = 2 * m->cfg.df_order;
    if (B <= 0 || T <= 0) return DFB_OK;
    if (B > 65535) return fail(DFB_ERR_INVALID, "more than 65535 streams per call");
    size_t extra = ((size_t)M * m->cfg.nb_erb + (size_t)M * m->cfg.nb_df * O2 + (size_t)M) * 4 + 8192;
    int rc = m->arena.reserve(fwd_plan(m->cfg, (size_t)M, nullptr, nullptr) + extra);
    if (rc) return rc;
    m->arena.reset();
    float *mm = d_m ? d_m : m->arena.take<float>((size_t)M * m->cfg.nb_erb);
    float *cc = d_coefs ? d_coefs : m->arena.take<float>((size_t)M * m->cfg.nb_df * O2);
    float *aa = d_alpha;
    if (!aa && m->cfg.model_kind == 1) aa = m->arena.take<float>((size_t)M);
    rc = forward_impl(m, m->arena, d_feat_erb, d_feat_spec, (int)B, (int)T, mm, cc, d_lsnr, aa, (cudaStream_t)stream);
    if (rc) { m->arena.reset(); return rc; }
    rc = apply_impl(m, st, d_spec, mm, cc, m->cfg.model_kind == 1 ? aa : nullptr, B, T, d_spec_e, stream);
    m->arena.reset();
    return rc;
}

extern "C" int64_t dfb_enhance_out_len(const dfb_state *st, int64_t T, int pad) {
    if (!st) return -1;
    return pad ? T : (T / st->hop) * st->hop;
}

constexpr int kModelRate = 48000;   // the model's rate: 480-sample hops of the 960 / 480 STFT

// A stream of T samples at `rate` resampled to 48 kHz: ceil(T * 48000 / rate) samples (io.resample's length)
static int64_t len_at_48k(int64_t T, int rate) {
    const int64_t g = std::gcd(rate, kModelRate), og = rate / g, nw = kModelRate / g;
    return (T * nw + og - 1) / og;
}
static int64_t len_from_48k(int64_t T48, int rate) {
    const int64_t g = std::gcd(rate, kModelRate), og = kModelRate / g, nw = rate / g;
    return (T48 * nw + og - 1) / og;
}

extern "C" int64_t dfb_enhance_out_len_at(const dfb_state *st, int64_t T, int pad, int rate) {
    if (!st || T <= 0 || rate <= 0) return -1;
    if (rate == kModelRate) return dfb_enhance_out_len(st, T, pad);
    return len_from_48k(dfb_enhance_out_len(st, len_at_48k(T, rate), pad), rate);
}

// LSNR values of a stream in dfb_enhance_ragged: one per 10 ms hop of its 48 kHz output, ceil(out48 / hop)
extern "C" int64_t dfb_enhance_lsnr_len(const dfb_state *st, int64_t T, int pad, int rate) {
    if (!st || T <= 0 || rate <= 0) return -1;
    const int64_t o48 = dfb_enhance_out_len(st, rate == kModelRate ? T : len_at_48k(T, rate), pad);
    return (o48 + st->hop - 1) / st->hop;
}

// The taps of rated batches at `rate` (DESIGN.md section 5i): both directions of io.resample_kernel's sinc_fast taps,
// at most kMaxRateTaps floats together.  48000 registers nothing (a 48 kHz stream is never resampled).
constexpr int64_t kMaxRateTaps = int64_t(1) << 18;
extern "C" int dfb_model_add_rate(dfb_model *m, int rate, const float *up_taps, int up_og, int up_nw, int up_width,
                                  const float *down_taps, int down_og, int down_nw, int down_width) {
    if (!m) return fail(DFB_ERR_INVALID, "null model");
    if (rate == kModelRate) return DFB_OK;
    if (rate <= 0) return fail(DFB_ERR_UNSUPPORTED, "sample rate %d Hz", rate);
    const int g = std::gcd(rate, kModelRate);
    if (up_og != rate / g || up_nw != kModelRate / g || down_og != kModelRate / g || down_nw != rate / g)
        return fail(DFB_ERR_INVALID, "the taps of %d Hz are io.resample_kernel(%d, 48000) (og %d, nw %d) and (48000, %d) (og %d, nw %d)",
                    rate, rate, rate / g, kModelRate / g, rate, kModelRate / g, rate / g);
    if (up_width <= 0 || down_width <= 0 || up_width > (1 << 20) || down_width > (1 << 20))
        return fail(DFB_ERR_INVALID, "the taps of %d Hz have widths %d / %d", rate, up_width, down_width);
    const int64_t nu = (int64_t)up_nw * (2 * up_width + up_og), nd = (int64_t)down_nw * (2 * down_width + down_og);
    if (nu + nd > kMaxRateTaps)
        return fail(DFB_ERR_UNSUPPORTED, "sample rate %d Hz: its resampler taps hold %lld floats, more than 2^18", rate,
                    (long long)(nu + nd));
    if (!up_taps || !down_taps) return fail(DFB_ERR_INVALID, "null taps");
    if (std::find(m->rates.begin(), m->rates.end(), rate) != m->rates.end()) return DFB_OK;
    DFB_CUDA(cudaSetDevice(m->device));
    float *taps = nullptr;
    RateDir *dirs = nullptr;
    const size_t n = m->rates.size() + 1;
    if (cudaMalloc(&taps, sizeof(float) * (size_t)(nu + nd)) != cudaSuccess || cudaMalloc(&dirs, sizeof(RateDir) * 2 * n) != cudaSuccess) {
        if (taps) cudaFree(taps);
        return fail(DFB_ERR_OOM, "resampler taps allocation failed");
    }
    std::vector<RateDir> up = m->rate_up, down = m->rate_down, all;
    up.push_back(RateDir{taps, up_og, up_nw, 2 * up_width + up_og, up_width});
    down.push_back(RateDir{taps + nu, down_og, down_nw, 2 * down_width + down_og, down_width});
    all = up;
    all.insert(all.end(), down.begin(), down.end());
    // (synchronous: a call still running reads the old table, which is freed below)
    if (cudaMemcpy(taps, up_taps, sizeof(float) * (size_t)nu, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(taps + nu, down_taps, sizeof(float) * (size_t)nd, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(dirs, all.data(), sizeof(RateDir) * all.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaDeviceSynchronize() != cudaSuccess) {
        cudaFree(taps);
        cudaFree(dirs);
        return fail(DFB_ERR_CUDA, "resampler taps upload failed");
    }
    if (m->d_rate_dirs) cudaFree(m->d_rate_dirs);
    m->d_rate_dirs = dirs;
    m->rates.push_back(rate);
    m->rate_up.swap(up);
    m->rate_down.swap(down);
    m->rate_taps.push_back(taps);
    return DFB_OK;
}

// enhance(): df/enhance.py:206-250.  Streams are processed in groups so that the workspace stays
// below the model's workspace cap (40 GB by default; dfb_model_set_max_workspace / DFB_MAX_WORKSPACE_MB); streams
// are independent (per-channel state reset, pyDF/src/lib.rs:56-58).
extern "C" int dfb_model_set_max_workspace(dfb_model *m, int64_t bytes) {
    if (!m || bytes <= 0) return fail(DFB_ERR_INVALID, "bad workspace cap");
    m->max_workspace = (size_t)bytes;
    return DFB_OK;
}


// ============================================================== time-chunked executor ====
// enhance() (df/enhance.py:206-250) and the streaming API run the path in TIME CHUNKS with carried per-stream state
// (SURVEY.md Appendix D): memory is proportional to the chunk, not the signal; host copies of one chunk overlap the
// compute of the next; and the frame-incremental API of the reference (libDF/src/tract.rs:509-642) is the same code
// with a chunk of a few frames.  Per chunk the window [W0, d1) of DNN frames = kHalo already finished frames (their
// feed-forward activations are recomputed from the carried feature history; receptive field <= 6 frames) + the new
// frames [d0, d1); the recurrences run over the new frames only, from the carried hidden states.
struct StreamState {
    int B = 0;
    int64_t a1 = 0, d1 = 0, e1 = 0;     // frames analysed / through the DNN / emitted as audio so far (absolute)
    bool started = false, dnn_started = false;   // first analysis / first DNN chunk done (states are valid)
    float *slab = nullptr;              // one allocation holding everything below
    float *ana_mem = nullptr;           // [B][hop]       last input hop (streaming API; the batch path reads resident audio)
    float *erb_state = nullptr, *unit_state = nullptr;   // [B][E], [B][Fd]  EMA states of the feature normalisation
    float *h_enc = nullptr, *h_erb = nullptr, *h_df = nullptr;   // [layers][B][H]
    float *t_spec = nullptr, *t_fe = nullptr, *t_fs = nullptr;   // last Hf = kHalo + Lmax frames of spec / features, right aligned
    float *t_m = nullptr, *t_c = nullptr;                        // last kMcTail frames of m / coefs, right aligned
    float *t_l = nullptr;                                        // ... and of lsnr (stage gating)
    float *t_dec = nullptr;                                      // (conv_kt == 2) last kHalo frames of dec_emb
    int n_feat = 0, n_mc = 0, n_dec = 0;                         // valid frames in the tails
    // runtime gating mode (GateRun): c0 of the DF decoder's last df_pathway_kt - 1 run frames, (conv_kt == 2) dec_emb | e3 |
    // d1 | e0 of the ERB decoder's last run frame; rt_valid: the last DNN chunk kept them (else it ran in apply mode)
    float *t_c0 = nullptr, *t_run = nullptr;
    bool rt_valid = false;
};
constexpr int kMcTail = 6;   // >= df_order (DeepFilterNet2, see run_chunk)

struct ChunkGeom { int Lmax, lag, Hf; };
static ChunkGeom chunk_geom(const dfb_model_config &c) {
    ChunkGeom g;
    g.Lmax = c.conv_lookahead > c.df_lookahead ? c.conv_lookahead : c.df_lookahead;
    // DeepFilterNet2 filters the MASKED spectrum: frame t needs the masks of frames <= t + df_lookahead, so its audio
    // trails the DNN frames by df_lookahead (deepfilternet2.py:494-503)
    g.lag = c.model_kind != 3 ? c.df_lookahead : 0;
    g.Hf = kHalo + g.Lmax;
    return g;
}

// Every array of the state slab is `layers` x [B][per_row] floats; only the GRU states have more than one layer.
// Arrays 13 / 14: the runtime gating mode's decoder tails (GateRun), 0 floats for DeepFilterNet v1 (14: for conv_kt == 1).
// Arrays 15 / 16: the histories of a resampled handle's up / down resampler (dfb_stream_set_sample_rate), 0 floats otherwise.
// The resampler histories stay last: handles that resample nothing move every array but those two (k_slot_rows).
constexpr int kStateArrays = 17;
// row_off / row_floats: one stream's row of every array, packed (the scratch rows of k_slot_rows)
struct StateLayout { int64_t off[kStateArrays], row_off[kStateArrays], row_floats; int layers[kStateArrays], per_row[kStateArrays]; };
constexpr int kRsArray = kStateArrays - 2;   // the first resampler history (15: up, 16: down)

// Element e (layer-major, as row_off packs a row) of slab row `row` of array a, in a slab of Bs rows.  Every kernel that
// moves state rows addresses them here: k_slot_rows, k_sessions_pack, k_sessions_unpack.
__device__ __forceinline__ int64_t state_elem(const StateLayout &lay, int Bs, int a, int row, int64_t e) {
    const int per = lay.per_row[a];
    const int l = (int)(e / per), j = (int)(e - (int64_t)l * per);
    return lay.off[a] + ((int64_t)l * Bs + row) * per + j;
}
// element e of array a in a fresh stream's row: zeros, and the normalisation EMA states at the values launch_feat_norm
// starts from without a state (arrays 1 and 2 have one layer)
__device__ __forceinline__ float state_init(int a, int64_t e, int E, int Fd) {
    return a == 1 ? erb_norm_init((int)e, E) : a == 2 ? unit_norm_init((int)e, Fd) : 0.f;
}

static size_t state_floats(const dfb_model_config &c, const dfb_state *st, int B, size_t off[kStateArrays], StateLayout *lay = nullptr,
                           int rs_up = 0, int rs_down = 0) {
    const ChunkGeom g = chunk_geom(c);
    const int E = c.nb_erb, Fd = c.nb_df, O2 = 2 * c.df_order, F = st->tb.F, ED = E / 4 * kCh;
    size_t n = 0;
    if (lay) lay->row_floats = 0;
    auto add = [&](int i, int layers, int per_row) {
        off[i] = n;
        if (lay) {
            lay->off[i] = (int64_t)n; lay->layers[i] = layers; lay->per_row[i] = per_row;
            lay->row_off[i] = lay->row_floats;
            lay->row_floats += (int64_t)layers * per_row;
        }
        n += ((size_t)layers * B * per_row + 63) & ~size_t(63);
    };
    add(0, 1, st->hop); add(1, 1, E); add(2, 1, Fd);
    add(3, c.enc_gru_layers, c.emb_hidden); add(4, c.erb_gru_layers, c.emb_hidden); add(5, c.df_gru_layers, c.df_hidden);
    add(6, 1, g.Hf * 2 * F); add(7, 1, g.Hf * E); add(8, 1, g.Hf * 2 * Fd);
    add(9, 1, kMcTail * E); add(10, 1, kMcTail * Fd * O2);
    add(11, 1, c.conv_kt > 1 ? kHalo * ED : 0);
    add(12, 1, kMcTail);
    add(13, 1, c.model_kind != 1 ? (c.df_pathway_kt - 1) * Fd * kCh : 0);
    add(14, 1, c.model_kind != 1 && c.conv_kt > 1 ? 2 * ED + 2 * E * kCh + 1 : 0);
    add(15, 1, rs_up); add(16, 1, rs_down);
    return n;
}
static void state_bind(StreamState &S, float *base, const size_t off[kStateArrays], int B) {
    S.B = B; S.slab = base;
    S.ana_mem = base + off[0]; S.erb_state = base + off[1]; S.unit_state = base + off[2];
    S.h_enc = base + off[3]; S.h_erb = base + off[4]; S.h_df = base + off[5];
    S.t_spec = base + off[6]; S.t_fe = base + off[7]; S.t_fs = base + off[8];
    S.t_m = base + off[9]; S.t_c = base + off[10]; S.t_dec = base + off[11]; S.t_l = base + off[12];
    S.t_c0 = base + off[13]; S.t_run = base + off[14];
    S.a1 = S.d1 = S.e1 = 0; S.started = S.dnn_started = false; S.n_feat = S.n_mc = S.n_dec = 0;
    S.rt_valid = false;
}

// last n frames of buf [B][T][fe] -> tail [B][cap][fe] (right aligned), and back into frames [dst_t, dst_t + n) of a buffer
static int save_tail(cudaStream_t s, const float *buf, int T, size_t fe, int n, float *tail, int cap, int B) {
    if (n <= 0) return DFB_OK;
    DFB_CUDA(cudaMemcpy2DAsync(tail + (size_t)(cap - n) * fe, sizeof(float) * fe * cap, buf + (size_t)(T - n) * fe, sizeof(float) * fe * T,
                               sizeof(float) * fe * n, B, cudaMemcpyDeviceToDevice, s));
    return DFB_OK;
}
static int load_tail(cudaStream_t s, float *buf, int T, size_t fe, int n, const float *tail, int cap, int dst_t, int B) {
    if (n <= 0) return DFB_OK;
    DFB_CUDA(cudaMemcpy2DAsync(buf + (size_t)dst_t * fe, sizeof(float) * fe * T, tail + (size_t)(cap - n) * fe, sizeof(float) * fe * cap,
                               sizeof(float) * fe * n, B, cudaMemcpyDeviceToDevice, s));
    return DFB_OK;
}

// bytes of workspace one window of Tw DNN frames needs per stream (features hold Tw + Lmax frames)
static size_t chunk_bytes_per_stream(const dfb_model_config &c, const dfb_state *st, int Tw) {
    const ChunkGeom g = chunk_geom(c);
    const int E = c.nb_erb, Fd = c.nb_df, O2 = 2 * c.df_order, F = st->tb.F;
    return (size_t)(Tw + g.Lmax) * (2 * F + E + 2 * Fd) * 4 + (size_t)Tw * (E + (size_t)Fd * O2 + 2) * 4 + fwd_plan(c, (size_t)Tw, nullptr, nullptr) +
           16384;
}

// Where the audio of one chunk comes from and goes to.
struct ChunkIO {
    const float *audio; int64_t audio_T;   // signal the analysis reads (rows[b].in_off / len): at most T samples per row
    int64_t audio_frame0;     // absolute frame index of the signal's first frame (0: resident whole signal; a0: streaming chunk)
    const float *init_mem;    // [B][hop] samples before audio[0] (streaming) or null (zeros)
    float *out; int64_t out_stride, out_len;
    int64_t out_sample0;      // absolute synthesis sample (frame * hop + i) that lands at out[0]
    float atten_lim;
    const float *lsnr_th;     // {min_db_thresh, max_db_erb_thresh, max_db_df_thresh} (tract.rs:658-672) or null: no gating
    // per-stream input / output rows and frame counts (device table; batch: streams sorted longest first), and how many
    // of them run in this chunk (a prefix: batch streams that still have frames, a handle's live slots)
    const RaggedRow *rows = nullptr;
    int nb = 0;
    // linked channels: each stream's link group (device table in kernel batch order) and the mask reduction, or null / 0
    const LinkRow *links = nullptr;
    int reduce = 0;
    // streaming slots (dfb_stream_open_slots): rows are the handle's active slots, rows[b].Tf the end of a closing one, and
    // first[b] the absolute first frame of each; emission follows the handle's clock, clipped at each stream's end.  Or null.
    const int64_t *first = nullptr;
    // per-row attenuation limit, post-filter beta and gating thresholds (launch_apply_synthesis; streaming slots and
    // batches with a settings table), or null.  ctl_gate: some row gates, so the LSNR head runs.
    const SlotCtl *ctl = nullptr;
    bool ctl_gate = false;
    // ragged batch LSNR rows (dfb_enhance_ragged), or null: row b's value j, at lsnr_rows + lsnr_offs[b] (device table),
    // is the LSNR of the frame output hop j carries, frame j + out_sample0 / hop (k_lsnr_rows)
    float *lsnr_rows = nullptr;
    const int64_t *lsnr_offs = nullptr;
    // streaming LSNR output: lsnr_from >= 0 runs the LSNR head (as gating does) and carries its tail; lsnr_out (or null)
    // [rows][out_len / hop] receives the LSNR of every frame the apply kernel emits whose DNN step ran from lsnr_from on,
    // at the hop that carries it.  Entries of hops that carry no frame are left as they are.
    int64_t lsnr_from = -1;
    float *lsnr_out = nullptr;
    // spectral handle (dfb_stream_create_spec), or null: the caller's spectrum frames replace the audio (k_spec_ingest reads
    // rows[b].in_off / len as complex values / frames) and k_spec_emit writes the network's outputs in place of apply +
    // synthesis
    const float *spec_in = nullptr;
    int64_t spec_frames = 0;
    const struct SpecOut *spec_out = nullptr;
    // runtime gating mode (GateRun): wherever a row gates, its decoders run only on the frames its stages let through
    bool runtime = false;
    const unsigned char *rt_halo = nullptr;   // per-row GateRun::halo, or null: every row as S.rt_valid says
};

// Outputs of a spectral call (k_spec_emit): caller row c, output row j of n_out carries frame f0 + j; slot_row maps caller
// rows to the kernel's live rows, -1 for a free slot.  Any output pointer but gains may be null.
struct SpecOut {
    float *gains, *coefs, *lsnr;
    int8_t *stage;
    int Bc;
    int64_t n_out, f0;
    const int *slot_row;
    int gating;        // LSNR stage gating with th = {min, max_erb, max_df}
    float th[3];
    int mask_only;
};

// ---- spectral handle kernels (dfb_stream_create_spec)
constexpr int kSpecF = 481, kIngWarps = 4;
constexpr const char *kSpecIngestName = "k_spec_ingest", *kSpecEmitName = "k_spec_emit";
// k_spec_ingest replaces k_analysis: warp w of CTA (x, b) reads frame x * kIngWarps + w of live row b once, coalesced
// (3848 B), and writes the frame's 32 ERB band energies in dB -- |X|^2 and the in-band sums exactly as k_analysis's
// epilogue, so the same spectrum gives the same bits -- and its first Fd bins, into rows out_t0 ... of buffers holding Tbuf
// frames per stream, where k_feat_norm reads them.  Row b reads from in + rows[b].in_off (complex values), and zeros from
// frame rows[b].len on (a closing slot).
__global__ void __launch_bounds__(32 * kIngWarps) k_spec_ingest(const float2 *__restrict__ in, const RaggedRow *__restrict__ rows,
                                                                int nf, float2 *__restrict__ bins, int Fd, int64_t bins_pitch,
                                                                float *__restrict__ erb_db, int out_t0, int Tbuf, DspTables tb) {
    __shared__ float s_p[kIngWarps][kSpecF + 3];
    const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * kIngWarps + warp;
    if (t >= nf) return;
    const bool have = t < rows[b].len;
    const float2 *x = in + rows[b].in_off + (int64_t)t * kSpecF;
    const int64_t orow = (int64_t)b * Tbuf + out_t0 + t;
    float2 *brow = bins + orow * bins_pitch;
    float *P = s_p[warp];
    for (int k = lane; k < kSpecF; k += 32) {
        const float2 v = have ? __ldg(x + k) : make_float2(0.f, 0.f);
        P[k] = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
        if (k < Fd) brow[k] = v;
    }
    __syncwarp();
    // band energies: sequential sum inside each band, factor 1/width inside the sum (lib.rs:288-292), as k_analysis
    for (int band = lane; band < tb.E; band += 32) {
        const int o = tb.erb_off[band], n = tb.erb_off[band + 1] - o;
        const float kinv = tb.erb_kinv[band];
        float acc = 0.f;
        for (int j = 0; j < n; j++) acc = __fadd_rn(acc, __fmul_rn(P[o + j], kinv));
        erb_db[orow * tb.E + band] = __fmul_rn(log10f(__fadd_rn(acc, 1e-10f)), 10.f);
    }
}

static int launch_spec_ingest(const dfb_state *st, const float *in, const RaggedRow *rows, int B, int nf, float *bins, int Fd,
                              int64_t bins_pitch, float *erb_db, int out_t0, int Tbuf, cudaStream_t s) {
    if (B <= 0 || nf <= 0) return DFB_OK;
    if (st->tb.F != kSpecF || st->tb.E > 32 * 8) return fail(DFB_ERR_UNSUPPORTED, "spectral input is built for fft_size 960");
    // timed by dfb_profile_* like the enhancement path's kernels, but outside the DFB_PROF list whose per-kernel roofline
    // model bench.py keeps: a spectral handle is not on the enhancement path (bench_stream_spec.py reports its share)
    dfb::ProfScope prof_scope__(kSpecIngestName, s);
    dim3 grid((unsigned)((nf + kIngWarps - 1) / kIngWarps), (unsigned)B);
    k_spec_ingest<<<grid, 32 * kIngWarps, 0, s>>>((const float2 *)in, rows, nf, (float2 *)bins, Fd, bins_pitch, erb_db, out_t0, Tbuf,
                                                  st->tb);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

// k_spec_emit replaces apply + synthesis: CTA (j, c) writes output row j of caller row c in one pass -- the frame's ERB
// gains (reduced over its link group in registers, as the LINK apply kernel does), its coefficients and LSNR, after the
// stage rule -- or NaN / -1 where the row carries no frame.  The frame rule is k_lsnr_out's: window frame t = f0 + j - w0 is
// emitted when t_first <= t < Te, clipped at the row's end and first frame.  m [B][mcT][E], coefs [B][mcT][FO], lsnr [B][mcT].
__global__ void __launch_bounds__(128) k_spec_emit(SpecOut o, const float *__restrict__ m, const float *__restrict__ coefs,
                                                   const float *__restrict__ lsnr, int mcT, int E, int FO, int64_t w0, int t_first, int Te,
                                                   const RaggedRow *__restrict__ rows, const int64_t *__restrict__ first,
                                                   const LinkRow *__restrict__ links, int reduce) {
    const int c = blockIdx.y, tid = threadIdx.x;
    const int64_t j = blockIdx.x, q = (int64_t)c * o.n_out + j;
    const int r = o.slot_row[c];
    int64_t t = -1;
    if (r >= 0) {
        const int te = min(Te, (int)(rows[r].Tf - w0));
        const int t0 = max(t_first, stream_first(first, r, w0));
        const int64_t tt = o.f0 + j - w0;
        if (tt >= t0 && tt < te) t = tt;
    }
    if (t < 0) {
        const float nan = __int_as_float(0x7fffffff);
        for (int e = tid; e < E; e += blockDim.x) o.gains[q * E + e] = nan;
        if (o.coefs)
            for (int k = tid; k < FO; k += blockDim.x) o.coefs[q * FO + k] = nan;
        if (tid == 0) {
            if (o.lsnr) o.lsnr[q] = nan;
            if (o.stage) o.stage[q] = -1;
        }
        return;
    }
    const float l = lsnr[(int64_t)r * mcT + t];
    const int lb = links ? links[r].first : r;          // gating reads the link group's channel 0
    const float lg = lsnr[(int64_t)lb * mcT + t];
    int stage = 1;
    if (o.gating) stage = lg < o.th[0] ? 0 : lg > o.th[1] ? 3 : lg > o.th[2] ? 2 : 1;   // tract.rs:658-672
    if (stage == 1 && o.mask_only) stage = 2;
    for (int e = tid; e < E; e += blockDim.x) {
        float v = stage == 0 ? 0.f : 1.f;
        if (stage == 1 || stage == 2) {
            if (!links) {
                v = m[((int64_t)r * mcT + t) * E + e];
            } else {   // the link group's max / mean in channel order, the mean as the fp32 sum times fl32(1 / n)
                const int n = links[r].n;
                const int64_t stride = (int64_t)mcT * E;
                const float *p = m + (int64_t)lb * stride + t * E + e;
                v = p[0];
                if (reduce == kReduceMax) {
                    for (int k = 1; k < n; k++) v = fmaxf(v, p[k * stride]);
                } else {
                    for (int k = 1; k < n; k++) v += p[k * stride];
                    v = v * __frcp_rn((float)n);
                }
            }
        }
        o.gains[q * E + e] = v;
    }
    if (o.coefs) {
        const float *src = coefs + ((int64_t)r * mcT + t) * FO;
        for (int k = tid; k < FO; k += blockDim.x) o.coefs[q * FO + k] = stage == 1 ? src[k] : 0.f;
    }
    if (tid == 0) {
        if (o.lsnr) o.lsnr[q] = l;
        if (o.stage) o.stage[q] = (int8_t)stage;
    }
}

static int launch_spec_emit(const SpecOut &o, const float *m, const float *coefs, const float *lsnr, int mcT, int E, int FO, int64_t w0,
                            int t_first, int Te, const RaggedRow *rows, const int64_t *first, const LinkRow *links, int reduce,
                            cudaStream_t s) {
    if (o.Bc <= 0 || o.n_out <= 0) return DFB_OK;
    dfb::ProfScope prof_scope__(kSpecEmitName, s);   // (see launch_spec_ingest)
    k_spec_emit<<<dim3((unsigned)o.n_out, (unsigned)o.Bc), 128, 0, s>>>(o, m, coefs, lsnr, mcT, E, FO, w0, t_first, Te, rows, first, links,
                                                                        reduce);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

// LSNR of the frames the apply kernel emitted in this chunk, by the kernel's own emission rule: output hop j of row b
// carries window frame t = f0 + j - w0, which was emitted when t_first <= t < Te (Te clipped at the stream's end
// rows[b].Tf) and the stream had started (stream_first).  Frames whose DNN step ran before `from` have no LSNR.
__global__ void k_lsnr_out(const float *__restrict__ ll, int mcT, float *__restrict__ out, int64_t n_out, int64_t f0, int64_t w0,
                           int t_first, int Te, const RaggedRow *__restrict__ rows, const int64_t *__restrict__ first, int64_t from,
                           int hop) {
    const int b = blockIdx.y;
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_out) return;
    const int64_t o = rows[b].out_off / hop;
    const int te = min(Te, (int)(rows[b].Tf - w0));
    int64_t t0 = max(t_first, stream_first(first, b, w0));
    if (from - w0 > t0) t0 = from - w0;
    const int64_t t = f0 + j - w0;
    if (t >= t0 && t < te) out[o + j] = ll[(int64_t)b * mcT + t];
}

// LSNR rows of a ragged batch: every window frame t that the apply kernel emitted for row b in this chunk (t_first <= t
// < te, te the stream's own end when it ends in this window, else t_emit) goes to value (w0 + t) - f0 of the row, the
// output hop that carries it, when that hop exists: ceil(out_len / hop) values per row.
__global__ void k_lsnr_rows(const float *__restrict__ ll, int mcT, float *__restrict__ out, const int64_t *__restrict__ offs,
                            int64_t f0, int64_t w0, int t_first, int t_emit, const RaggedRow *__restrict__ rows, int hop) {
    const int b = blockIdx.y;
    const int t = t_first + blockIdx.x * blockDim.x + threadIdx.x;
    const RaggedRow r = rows[b];
    const int64_t tfb = r.Tf - w0;
    const int64_t te = tfb <= mcT ? tfb : t_emit;
    const int64_t j = w0 + t - f0, n = (r.out_len + hop - 1) / hop;
    if (t < te && j >= 0 && j < n) out[offs[b] + j] = ll[(int64_t)b * mcT + t];
}

// One chunk: analyse frames [S.a1, a1n), run the DNN over [S.d1, d1n), emit audio of frames [S.e1, e1n).
// Only the first io.nb streams run; a stream whose frame count Tf_b is <= d1n ends in this chunk: its features and
// spectrum beyond Tf_b do not exist and it emits all of its frames up to Tf_b.
// lane / pipelined: consecutive chunks of a batch call alternate between the model's two lanes (stream sets + arenas);
// chunk c starts when chunk c - 1 has finished its ENCODER phase and its decoder phase waits for chunk c - 1 to finish
// entirely, so encoder(c) overlaps decoder(c - 1).  `s` is the stream the chunk is enqueued on (the lane's main stream
// in the pipeline, the caller's stream otherwise).
static int run_chunk(dfb_model *m, dfb_state *st, StreamState &S, const ChunkIO &io, int64_t a1n, int64_t d1n, int64_t e1n,
                     cudaStream_t s, int lane = 0, bool pipelined = false) {
    Arena &arena = lane ? m->arena1 : m->arena;
    dfb_model::Lane &L = m->lanes[lane], &P = m->lanes[lane ^ 1];
    const bool have_prev = pipelined && S.started;
    if (have_prev) DFB_CUDA(cudaStreamWaitEvent(s, P.ev_fork, 0));   // previous chunk: features + encoder phase done
    const dfb_model_config &c = m->cfg;
    const ChunkGeom g = chunk_geom(c);
    const int B = io.nb, E = c.nb_erb, Fd = c.nb_df, O2 = 2 * c.df_order, F = st->tb.F, hop = st->hop;
    const int64_t W0 = S.d1 > kHalo ? S.d1 - kHalo : 0;
    const int Rc = (int)(S.d1 - W0), Tw = (int)(d1n - W0), Tsb = Tw + g.Lmax;
    const int n_hist = (int)(S.a1 - W0);                 // feature frames of the window that are already known
    const int n_new = (int)(a1n - S.a1), Tv = (int)(a1n - W0);
    if (Tw < Rc || n_hist < 0 || n_hist > S.n_feat || Tv > Tsb || Tsb <= 0)
        return fail(DFB_ERR_INVALID, "inconsistent chunk geometry");
    const bool run_dnn = d1n > S.d1;      // a short streaming call may only add look-ahead frames
    int rc;
    arena.reset();
    float *spec = arena.take<float>((size_t)B * Tsb * F * 2 + 2);
    float *fe = arena.take<float>((size_t)B * Tsb * E);
    float *fs = arena.take<float>((size_t)B * Tsb * Fd * 2);
    float *mm = arena.take<float>((size_t)B * (Tw + 1) * E);
    float *cc = arena.take<float>((size_t)B * (Tw + 1) * Fd * O2);
    float *ll = (io.lsnr_th || io.ctl_gate || io.lsnr_rows || io.lsnr_from >= 0 || io.spec_out) ? arena.take<float>((size_t)B * (Tw + 1))
                                                                                                   : nullptr;
    float *aa = c.model_kind == 1 ? arena.take<float>((size_t)B * (Tw + 1)) : nullptr;   // df_alpha (v1)
    if (!cc || (c.model_kind == 1 && !aa)) return fail(DFB_ERR_OOM, "chunk workspace exhausted");
    // ---- features: carried history, then the new frames (a spectral handle keeps no spectrum: nothing is applied)
    const bool spectral = io.spec_out != nullptr;
    if ((!spectral && (rc = load_tail(s, spec, Tsb, (size_t)2 * F, n_hist, S.t_spec, g.Hf, 0, B))) ||
        (rc = load_tail(s, fe, Tsb, E, n_hist, S.t_fe, g.Hf, 0, B)) || (rc = load_tail(s, fs, Tsb, (size_t)2 * Fd, n_hist, S.t_fs, g.Hf, 0, B)))
        return rc;
    if (n_new > 0) {
        if (spectral) {   // the ERB dB and the first Fd bins of the caller's frames, where k_feat_norm reads them
            rc = launch_spec_ingest(st, io.spec_in, io.rows, B, n_new, spec, Fd, F, fe, n_hist, Tsb, s);
        } else {
            AnaWindow w{(int)(S.a1 - io.audio_frame0), n_new, n_hist, Tsb, io.rows};
            rc = launch_analysis(st, io.audio, B, io.audio_T, spec, fe, s, io.init_mem, &w);
        }
        if (rc) return rc;
        if ((rc = launch_feat_norm(fe + (size_t)n_hist * E, E, E, spec + (size_t)n_hist * 2 * F, Fd, F, B, n_new, c.norm_alpha,
                                   S.started ? S.erb_state : nullptr, S.started ? S.unit_state : nullptr, fe + (size_t)n_hist * E,
                                   fs + (size_t)n_hist * 2 * Fd, s, Tsb, S.erb_state, S.unit_state)))
            return rc;
    }
    {   // carry the feature history right away: the next chunk may start as soon as this chunk's encoder is done
        const int nf = Tv < g.Hf ? Tv : g.Hf;
        // the feature buffers hold Tsb frames per stream of which the first Tv are valid: keep the last nf valid ones
        const size_t fes[3] = {(size_t)2 * F, (size_t)E, (size_t)2 * Fd};
        float *bufs[3] = {spec, fe, fs}, *tails[3] = {S.t_spec, S.t_fe, S.t_fs};
        for (int i = spectral ? 1 : 0; i < 3; i++)
            DFB_CUDA(cudaMemcpy2DAsync(tails[i] + (size_t)(g.Hf - nf) * fes[i], sizeof(float) * fes[i] * g.Hf,
                                       bufs[i] + (size_t)(Tv - nf) * fes[i], sizeof(float) * fes[i] * Tsb, sizeof(float) * fes[i] * nf, B,
                                       cudaMemcpyDeviceToDevice, s));
        S.n_feat = nf;
    }
    // ---- DNN over the window
    if (run_dnn) {
    ChunkCtx cx{Rc, Tsb, Tv, S.h_enc, S.h_erb, S.h_df, S.dnn_started, c.conv_kt > 1 ? S.t_dec : nullptr, S.n_dec, lane,
                have_prev ? P.ev_done : nullptr, S.B, io.rows, W0, io.first};
    // the rows gate as the apply kernel (io.ctl: each row's own entry) or k_spec_emit decides
    const bool gates = io.ctl ? io.ctl_gate : (io.lsnr_th != nullptr || (spectral && io.spec_out->gating));
    GateRun gr{io.ctl, io.links, {0.f, 0.f, 0.f}, 0, S.t_c0, S.t_run, S.rt_valid, io.rt_halo};
    if (io.runtime && gates && c.model_kind != 1) {
        const float *th = spectral ? io.spec_out->th : io.lsnr_th;
        if (!io.ctl) { gr.gate_all = 1; gr.th[0] = th[0]; gr.th[1] = th[1]; gr.th[2] = th[2]; }
        cx.gate = &gr;
    }
    if ((rc = forward_impl(m, arena, fe, fs, B, Tw, mm, cc, ll, aa, s, &cx))) return rc;
    S.rt_valid = cx.gate != nullptr;
    S.n_dec = cx.dec_tail_n;
    S.dnn_started = true;
    // the halo rows of m / coefs come from skipped recurrences: restore the last finished frames from the previous chunk
    // (the apply kernel re-synthesises frame e0 - 1 for its overlap-add tail.  DFN2's masked taps of that frame reach
    // df_order - 1 - df_lookahead frames further back, and e0 = d1 - lag with lag = df_lookahead, so they read the masks
    // of frames [d1 - df_order, d1) at any look-ahead: 5 frames at df_lookahead 2 and at 0, within kMcTail and kHalo)
    if (Rc > 0 && S.n_mc > 0 && !spectral) {
        const int n = S.n_mc < Rc ? S.n_mc : Rc;
        if ((rc = load_tail(s, mm, Tw, E, n, S.t_m, kMcTail, Rc - n, B)) || (rc = load_tail(s, cc, Tw, (size_t)Fd * O2, n, S.t_c, kMcTail, Rc - n, B)))
            return rc;
        if (ll && (rc = load_tail(s, ll, Tw, 1, n, S.t_l, kMcTail, Rc - n, B))) return rc;
    }
    }
    // ---- spectral handle: the network's outputs of frames [e0, e1n) to the caller's rows (every row, NaN where none)
    if (spectral) {
        const int t_first = (int)(S.e1 - W0), Te = run_dnn ? (int)(e1n - W0) : t_first;
        if ((rc = launch_spec_emit(*io.spec_out, mm, cc, ll, Tw, E, Fd * O2, W0, t_first, Te, io.rows, io.first, io.links, io.reduce, s)))
            return rc;
    }
    // ---- apply + synthesis of frames [e0, e1n) (ragged: a stream that ends in this chunk emits up to its end)
    else if (run_dnn && (e1n > S.e1 || !io.first)) {
        dfb::ApplyParams p{};
        p.spec = (const float2 *)spec; p.m = mm; p.coefs = cc; p.audio = io.out; p.spec_out = nullptr;
        p.out_stride = io.out_stride; p.out_len = io.out_len;
        p.out_offset = io.out_sample0 - W0 * hop;     // g = t_window * hop + i - out_offset
        p.Tf = (int)(e1n - W0); p.spec_T = Tsb; p.Tv = Tv; p.mc_T = Tw; p.t_first = (int)(S.e1 - W0);
        p.mode = apply_mode(m); p.nb_df = Fd; p.order = c.df_order; p.lookahead = c.df_lookahead;
        p.atten_lim = io.atten_lim;
        p.alpha = aa;
        apply_options(m, p);
        if (io.lsnr_th) { p.lsnr = ll; p.th_min = io.lsnr_th[0]; p.th_erb = io.lsnr_th[1]; p.th_df = io.lsnr_th[2]; }
        if (io.ctl_gate) p.lsnr = ll;   // each row's thresholds from io.ctl
        p.rows = io.rows; p.w0 = W0; p.t_emit = p.Tf; p.first = io.first;
        if (!io.first) p.Tf = Tw;   // batch: the grid covers every stream's end; slots: Te = min(end, clock)
        if (io.links) { p.links = io.links; p.reduce = io.reduce; }
        if ((rc = launch_apply_synthesis(st, p, B, s, io.ctl))) return rc;
        if (io.lsnr_out && e1n > S.e1) {
            const int64_t n_out = io.out_len / hop;
            dim3 grid((unsigned)((n_out + 127) / 128), (unsigned)B);
            k_lsnr_out<<<grid, 128, 0, s>>>(ll, Tw, io.lsnr_out, n_out, io.out_sample0 / hop, W0, p.t_first, (int)(e1n - W0), io.rows,
                                            io.first, io.lsnr_from, hop);
            DFB_LAUNCH_CHECK();
        }
        if (io.lsnr_rows && Tw > p.t_first) {
            dim3 grid((unsigned)((Tw - p.t_first + 127) / 128), (unsigned)B);
            k_lsnr_rows<<<grid, 128, 0, s>>>(ll, Tw, io.lsnr_rows, io.lsnr_offs, io.out_sample0 / hop, W0, p.t_first, p.t_emit, io.rows, hop);
            DFB_LAUNCH_CHECK();
        }
    }
    // ---- carry
    {
        if (run_dnn && !spectral) {
            const int nm = Tw < kMcTail ? Tw : kMcTail;
            if ((rc = save_tail(s, mm, Tw, E, nm, S.t_m, kMcTail, B)) || (rc = save_tail(s, cc, Tw, (size_t)Fd * O2, nm, S.t_c, kMcTail, B))) return rc;
            if (ll && (rc = save_tail(s, ll, Tw, 1, nm, S.t_l, kMcTail, B))) return rc;
            S.n_mc = nm;
        }
    }
    if (pipelined) {
        if (!run_dnn) DFB_CUDA(cudaEventRecord(L.ev_fork, s));   // no forward pass recorded it
        DFB_CUDA(cudaEventRecord(L.ev_done, s));
    }
    S.a1 = a1n; S.d1 = d1n; if (run_dnn) S.e1 = e1n;
    S.started = true;
    return DFB_OK;
}

// Chunk length (new DNN frames per chunk) for B streams under a workspace cap of `cap` bytes; 0 when not even a short
// chunk fits.
static int pick_chunk(const dfb_model *m, const dfb_state *st, int64_t B, int64_t Tf, int min_chunks, size_t cap) {
    const size_t per_frame = chunk_bytes_per_stream(m->cfg, st, 1024) / 1024 + 1;   // bytes per stream and window frame
    const ChunkGeom g = chunk_geom(m->cfg);
    int64_t tw = (int64_t)(cap / ((size_t)B * per_frame)) - g.Lmax - 8;
    int64_t tc = tw - kHalo;
    if (tc > Tf) tc = Tf;
    if (min_chunks > 1 && Tf >= (int64_t)min_chunks * 64) {
        const int64_t t2 = (Tf + min_chunks - 1) / min_chunks;
        if (t2 < tc) tc = t2;
    }
    if (m->cfg.model_kind == 1) return tw >= Tf ? (int)Tf : 0;   // DeepFilterNet v1: one window per signal (forward_v1)
    if (tc < 1) return 0;
    if (tc < Tf && tc < 32) return 0;   // a chunk this short wastes most of its window on the halo: use stream groups
    return (int)tc;
}
// Hooks around every chunk of a stream group whose buffers are staged (host batch, rated batch).  `cs` is the stream the
// chunk's compute is enqueued on (it must wait for the input / produces the output); only the first `na` streams take part
// in the chunk.  `pcie`: the hooks copy over PCIe, and the end chunks are tapered so that their copies overlap more.
struct ChunkHooks {
    bool pcie = false;
    // the chunk's analysis reads input samples [x0, x1) of every stream (as far as the stream has them)
    std::function<int(int64_t x0, int64_t x1, int64_t na, cudaStream_t cs)> before;
    // output samples [y0, y1) of every stream have been written; a stream whose frame count is <= d1 (the chunk's last DNN
    // frame) has ended in it and has written all of its output, beyond y1
    std::function<int(int64_t y0, int64_t y1, int64_t d1, int64_t na, cudaStream_t cs)> after;
};

// Per-row settings and LSNR rows of one stream group (dfb_enhance_ragged), as device tables in the group's order, or
// nulls: ctl the settings (sw = 0), gate whether any row gates, lsnr / lsnr_offs the LSNR rows (ChunkIO::lsnr_rows).
struct BatchOut {
    const SlotCtl *ctl = nullptr;
    bool gate = false;
    float *lsnr = nullptr;
    const int64_t *lsnr_offs = nullptr;
};

// Runs the chunk loop over one stream group: `rows` is its device table and `tfs` its streams' frame counts on the host,
// longest first.  The analysis reads stream b from d_x + rows[b].in_off, apply + synthesis writes it to d_out + rows[b].out_off.
static int enhance_group(dfb_model *m, dfb_state *st, const float *d_x, float *d_out, const RaggedRow *rows, const int64_t *tfs,
                         int64_t nb, int pad, float lim, int tc, bool pipelined, cudaStream_t s, const ChunkHooks *hooks,
                         const LinkRow *links, int reduce, const BatchOut &bo) {
    const dfb_model_config &c = m->cfg;
    const ChunkGeom g = chunk_geom(c);
    const int hop = st->hop, fft = st->fft;
    const int64_t Tf = tfs[0];
    size_t off[kStateArrays];
    const size_t nstate = state_floats(c, st, (int)nb, off);
    float *slab = m->aux_arena.take<float>(nstate);
    if (!slab) return fail(DFB_ERR_OOM, "stream state arena exhausted");
    StreamState S;
    state_bind(S, slab, off, (int)nb);
    int rc = DFB_OK;
    const int64_t delay = pad ? fft - hop : 0;
    if (tc >= Tf) pipelined = false;      // a single chunk
    cudaEvent_t ev_call = nullptr;
    if (pipelined) {  // both lanes start after everything the caller has enqueued so far
        DFB_CUDA(cudaEventCreateWithFlags(&ev_call, cudaEventDisableTiming));
        DFB_CUDA(cudaEventRecord(ev_call, s));
        DFB_CUDA(cudaStreamWaitEvent(m->lanes[0].main, ev_call, 0));
        DFB_CUDA(cudaStreamWaitEvent(m->lanes[1].main, ev_call, 0));
    }
    int chunk = 0, last_lane = 0;
    // Host path: the first chunk's H2D copy and the last chunk's D2H copy are the only ones nothing overlaps, so both end
    // chunks are half as long as the others (128 x 10 s in 4 chunks: 250 / 250 / 250 / 252 frames -> 125 / 250 / 250 / 250 / 127).
    const bool taper = hooks && hooks->pcie && pipelined && tc < Tf && tc >= 64;
    while (S.d1 < Tf) {
        int64_t step = tc;
        if (taper) {
            const int64_t left = Tf - S.d1;
            if (chunk == 0) step = tc / 2;
            else if (left <= tc + tc / 2 && left - tc / 2 >= tc / 4) step = left - tc / 2;   // leaves a half-length last chunk
        }
        const int64_t d1n = S.d1 + step < Tf ? S.d1 + step : Tf;
        const int64_t a1n = d1n + g.Lmax < Tf ? d1n + g.Lmax : Tf;
        const int64_t e1n = d1n == Tf ? Tf : d1n - g.lag;
        const int lane = pipelined ? (chunk & 1) : 0;
        cudaStream_t cs = pipelined ? m->lanes[lane].main : s;
        int64_t na = nb;   // streams with frames left: a prefix, since the table is sorted longest first
        while (na > 1 && tfs[na - 1] <= S.d1) na--;    // (the members of a link group share Tf: they leave together)
        if (hooks && S.a1 < a1n && (rc = hooks->before(S.a1 * hop, a1n * hop, na, cs))) break;
        const int64_t e0 = S.e1;
        ChunkIO io{d_x, Tf * hop, 0, nullptr, d_out, 0, 0, delay, lim, nullptr, rows, (int)na, links, reduce};
        io.ctl = bo.ctl; io.ctl_gate = bo.gate;
        io.lsnr_rows = bo.lsnr; io.lsnr_offs = bo.lsnr_offs;
        io.runtime = m->gating_mode == DFB_GATING_RUNTIME;
        if ((rc = run_chunk(m, st, S, io, a1n, d1n, e1n > S.e1 ? e1n : S.e1, cs, lane, pipelined))) break;
        if (hooks && (rc = hooks->after(e0 * hop > delay ? e0 * hop - delay : 0, S.e1 * hop - delay, d1n, na, cs))) break;
        // what the hook enqueued on the lane is part of the chunk: the caller's stream and the next chunk's decoder wait for it
        if (hooks && pipelined && cudaEventRecord(m->lanes[lane].ev_done, cs) != cudaSuccess) {
            rc = fail(DFB_ERR_CUDA, "chunk event record failed");
            break;
        }
        last_lane = lane;
        chunk++;
    }
    if (pipelined) {  // hand the result back to the caller's stream (the last chunk finishes after all earlier ones)
        if (chunk > 0) cudaStreamWaitEvent(s, m->lanes[last_lane].ev_done, 0);
        if (chunk > 1) cudaStreamWaitEvent(s, m->lanes[last_lane ^ 1].ev_done, 0);
        if (rc) cudaDeviceSynchronize();
        cudaEventDestroy(ev_call);
    }
    return rc;
}

// enhance(): df/enhance.py:206-250.  Time chunks (above) inside stream groups: a group is as many streams as fit the
// workspace cap with a reasonable chunk; streams are independent (per-channel state reset, pyDF/src/lib.rs:56-58).
// A stream group never splits a link group: it takes at least `min_group` streams (the largest link group), else DFB_ERR_OOM.
static int enhance_plan(dfb_model *m, dfb_state *st, int64_t B, int64_t Tf, int min_chunks, int64_t min_group, int64_t *group_out,
                        int *tc_out, bool *pipelined_out) {
    // two lanes (DFB_LANES=1 turns the chunk pipeline off): each lane's arena may take half of the workspace cap
    static const bool serial = getenv("DFB_SERIAL") && atoi(getenv("DFB_SERIAL"));
    const bool pipelined = m->n_lanes == 2 && !serial && min_chunks > 1 && Tf >= (int64_t)min_chunks * 64;
    const size_t cap = pipelined ? m->max_workspace / 2 : m->max_workspace;
    int64_t group = B > 65535 ? 65535 : B;
    int tc = 0;
    while ((tc = pick_chunk(m, st, group, Tf, min_chunks, cap)) == 0) {
        if (group == 1) return fail(DFB_ERR_OOM, "workspace cap of %zu bytes is too small for a single stream", m->max_workspace);
        if (group <= min_group)
            return fail(DFB_ERR_OOM, "workspace cap of %zu bytes is too small for a link group of %lld channels", m->max_workspace,
                        (long long)min_group);
        group = std::max((group + 1) / 2, min_group);
    }
    *group_out = group; *tc_out = tc; *pipelined_out = pipelined && tc < Tf;
    const ChunkGeom g = chunk_geom(m->cfg);
    const size_t bytes = chunk_bytes_per_stream(m->cfg, st, tc + kHalo) * (size_t)group + ((size_t)g.Lmax << 10) + (2 << 20);
    int rc = m->arena.reserve(bytes);
    if (!rc && *pipelined_out) rc = m->arena1.reserve(bytes);
    return rc;
}

// ============================================================== batch executor ====
// Every dfb_enhance* call is a batch of streams, each an input offset, a length and an output offset (RaggedRow); an
// equal-length [B][T] batch is the special case {b T, T, b out_len}.  The streams are sorted by frame count, longest first,
// and stream groups are cut from that order.  Inside a group the chunk loop above runs only the prefix of streams that
// still have frames (the others have ended: their padded frames are never computed), and the kernels that look past the
// current frame -- analysis, the input convs' feature look-ahead, apply + synthesis -- read each stream's own end from the
// group's table in the aux arena.  So every stream's output is exactly that of the stream enhanced alone, and the `pad`
// zeros of enhance() need no padded copy of the input.  Zero-padding the batch to its longest stream would NOT be
// equivalent: the padded frames would exist, with features far from zero, and change the mask and deep filter of every
// padded stream's last look-ahead frames.  DeepFilterNet v1 runs one window per signal with the end padding applied inside
// every layer (forward_v1), so its stream groups are also cut where the frame count changes: a group shares one window.

// Validates a ragged call and returns its streams in the caller's order.  Stream b is lengths[b] samples at rates[b] (rates
// null: every stream at 48 kHz; DESIGN.md section 5i).  The chunk loop runs its 48 kHz signal, ceil(lengths[b] 48000 / rate)
// samples (io.resample's length), so rows are planned from the 48 kHz lengths and sorting, stream groups, the active prefix
// and link groups work unchanged; its output is the 48 kHz output resampled back, ceil(out48 rate / 48000) samples.
// `rows` are the streams at 48 kHz (offsets the caller's, used for 48 kHz streams only), `rr` the streams at their rates
// with their directions of the model's resamplers (-1: 48 kHz).
static int batch_plan(const dfb_model *m, const dfb_state *st, int64_t in_numel, const int64_t *in_offsets, const int64_t *lengths,
                      int64_t B, int pad, int64_t out_numel, const int64_t *out_offsets, const int32_t *rates,
                      std::vector<RaggedRow> &rows, std::vector<RateRow> &rr) {
    if (!in_offsets || !lengths || !out_offsets) return fail(DFB_ERR_INVALID, "null argument");
    if (B <= 0) return fail(DFB_ERR_INVALID, "empty batch");
    rows.resize((size_t)B);
    rr.resize((size_t)B);
    for (int64_t b = 0; b < B; b++) {
        const int64_t len = lengths[b], io = in_offsets[b], oo = out_offsets[b];
        const int rate = rates ? rates[b] : kModelRate;
        int dir = -1;
        if (rate != kModelRate) {
            const auto it = std::find(m->rates.begin(), m->rates.end(), rate);
            if (it == m->rates.end())
                return fail(DFB_ERR_INVALID, "stream %lld: sample rate %d Hz is not registered (dfb_model_add_rate)", (long long)b, rate);
            dir = (int)(it - m->rates.begin());
        }
        if (len <= 0) return fail(DFB_ERR_INVALID, "stream %lld has length %lld", (long long)b, (long long)len);
        const int64_t len48 = dir < 0 ? len : len_at_48k(len, rate), tf = (pad ? len48 + st->fft : len48) / st->hop,
                      ol48 = dfb_enhance_out_len(st, len48, pad), ol = dir < 0 ? ol48 : len_from_48k(ol48, rate);
        if (tf <= 0) return fail(DFB_ERR_INVALID, "stream %lld is shorter than one hop%s", (long long)b, rates ? " at 48 kHz" : "");
        if (io < 0 || io > in_numel - len)
            return fail(DFB_ERR_INVALID, "stream %lld reaches outside the input (%lld samples)", (long long)b, (long long)in_numel);
        if (oo < 0 || oo > out_numel - ol)
            return fail(DFB_ERR_INVALID, "stream %lld reaches outside the output (%lld samples)", (long long)b, (long long)out_numel);
        rows[(size_t)b] = RaggedRow{io, len48, oo, ol48, tf};
        rr[(size_t)b] = RateRow{io, len, oo, ol, tf, dir};
    }
    return DFB_OK;
}

// Copies samples [x0, end) of each stream i < n from src + src_off + x0 to dst + dst_off + x0 (`at(i)` describes stream i).
// Consecutive streams with the same end and a constant pitch on both sides share one 2-D copy, so an equal-length batch
// (or the channels of one multi-channel entry) takes one copy per chunk and direction instead of one per stream.
struct StreamCopy { int64_t dst_off, src_off, end; };
template <class At>
static int copy_streams(float *dst, const float *src, int64_t x0, int64_t n, At at, cudaMemcpyKind kind, cudaStream_t s) {
    constexpr int64_t kMaxPitch = INT32_MAX / sizeof(float);
    for (int64_t i = 0, j; i < n; i = j) {
        const StreamCopy a = at(i);
        const int64_t w = a.end - x0;
        int64_t dp = 0, sp = 0;   // pitches of the run [i, j)
        for (j = i + 1; j < n; j++) {
            const StreamCopy b = at(j), p = at(j - 1);
            if (b.end != a.end) break;
            if (j == i + 1) {
                dp = b.dst_off - a.dst_off; sp = b.src_off - a.src_off;
                if (dp < w || sp < w || dp > kMaxPitch || sp > kMaxPitch) break;
            } else if (b.dst_off - p.dst_off != dp || b.src_off - p.src_off != sp) break;
        }
        if (w <= 0) continue;
        if (j - i == 1) DFB_CUDA(cudaMemcpyAsync(dst + a.dst_off + x0, src + a.src_off + x0, sizeof(float) * w, kind, s));
        else DFB_CUDA(cudaMemcpy2DAsync(dst + a.dst_off + x0, sizeof(float) * dp, src + a.src_off + x0, sizeof(float) * sp,
                                        sizeof(float) * w, (size_t)(j - i), kind, s));
    }
    return DFB_OK;
}

// Validates the link groups of a linked call: group g is the next group_sizes[g] streams in the caller's order (`rows` and
// `rr` from batch_plan), all of one rate and one length.  Returns each stream's group {first stream, size} in the caller's
// order, or an empty table when nothing is linked (reduce none, or every group a single stream): such a call is the unlinked
// one.
static int link_plan(const dfb_model *m, const std::vector<RaggedRow> &rows, const std::vector<RateRow> &rr,
                     const int64_t *group_sizes, int64_t n_groups, int reduce, std::vector<LinkRow> &links) {
    if (reduce != kReduceNone && reduce != kReduceMax && reduce != kReduceMean)
        return fail(DFB_ERR_INVALID, "reduce_mask %d is not 0 (none), 1 (max) or 2 (mean)", reduce);
    if (!group_sizes || n_groups <= 0) return fail(DFB_ERR_INVALID, "no link groups");
    const int64_t B = (int64_t)rows.size();
    links.assign((size_t)B, LinkRow{0, 1});
    int64_t b = 0, n_max = 0;
    for (int64_t g = 0; g < n_groups; g++) {
        const int64_t n = group_sizes[g];
        if (n <= 0 || n > B - b) return fail(DFB_ERR_INVALID, "link group sizes do not sum to the %lld streams", (long long)B);
        if (n > 65535) return fail(DFB_ERR_INVALID, "link group %lld has more than 65535 channels", (long long)g);
        for (int64_t i = b; i < b + n; i++) {
            if (rows[(size_t)i].len != rows[(size_t)b].len)
                return fail(DFB_ERR_INVALID, "link group %lld has channels of different lengths", (long long)g);
            if (rr[(size_t)i].dir != rr[(size_t)b].dir || rr[(size_t)i].in_len != rr[(size_t)b].in_len)
                return fail(DFB_ERR_INVALID, "link group %lld mixes sample rates or lengths", (long long)g);
            links[(size_t)i] = LinkRow{(int)b, (int)n};
        }
        b += n;
        n_max = std::max(n_max, n);
    }
    if (b != B) return fail(DFB_ERR_INVALID, "link group sizes do not sum to the %lld streams", (long long)B);
    if (reduce == kReduceNone || n_max == 1) {
        links.clear();
        return DFB_OK;
    }
    if (m->cfg.model_kind == 1) return fail(DFB_ERR_UNSUPPORTED, "linked channels: DeepFilterNet v1 is not supported");
    return DFB_OK;
}

// The batch executor behind every dfb_enhance* entry point; `rows` and `rates` (the caller's order, from batch_plan) are
// sorted here.  `rows` are the streams at 48 kHz, which is what the chunk loop runs, and rates[b] is stream b at its own
// rate (DESIGN.md section 5i): the caller's buffers hold that.  Device buffers: the work is enqueued on `s`, on the caller's
// buffers when every stream is at 48 kHz.  Host buffers (`host`) or a rated batch (a stream at another rate than 48 kHz):
// each stream group is staged into 48 kHz device buffers that hold its streams packed back to back (a rated host batch also
// in staging buffers at the streams' rates), chunk by chunk and each stream's range clipped to its length.  Per chunk,
// before the analysis, the up-resampler writes the 48 kHz samples it reads, and after apply + synthesis the down-resampler
// writes the outputs that became complete; 48 kHz streams are copied, never resampled.  On the host path the H2D copy of
// chunk c + 1 and the D2H copy of chunk c - 1 run on their own streams (both copy engines) while chunk c computes, and the
// call is synchronous.
// `links` (or null): each stream's link group from link_plan, sorted here along with `rows`; `reduce` the mask reduction.
// `ctl` (or null): each stream's settings (sw = 0), sorted likewise; they replace atten_lim_db and the model's DeepFilterNet3
// post filter, and `gate` says whether any of them gates.  `lsnr` (or null): each stream's LSNR row goes to
// lsnr + lsnr_offsets[b] (caller's buffer, host or device as `host` says; k_lsnr_rows).
static int enhance_rows(dfb_model *m, dfb_state *st, std::vector<RaggedRow> &rows, std::vector<RateRow> &rates, const float *src,
                        float *dst, int pad, float atten_lim_db, bool host, cudaStream_t s, std::vector<LinkRow> *links = nullptr,
                        int reduce = 0, std::vector<SlotCtl> *ctl = nullptr, bool gate = false, float *lsnr = nullptr,
                        const int64_t *lsnr_offsets = nullptr) {
    const int64_t B = (int64_t)rows.size();
    const bool rated = std::any_of(rates.begin(), rates.end(), [](const RateRow &q) { return q.dir >= 0; });
    int64_t min_group = 1;   // the largest link group: a stream group never splits one
    std::vector<int64_t> lsnr_off;   // the streams' LSNR offsets in the caller's buffer, sorted
    {
        // The members of a link group are consecutive and share their sort key (one length), so the stable sort keeps them
        // one contiguous run in their own order: nothing between them has that key.  Sorting a permutation carries each
        // stream's group along, as the new position of the group's first member, and its rate.
        std::vector<int64_t> idx((size_t)B);
        std::iota(idx.begin(), idx.end(), (int64_t)0);
        std::stable_sort(idx.begin(), idx.end(), [&](int64_t a, int64_t b) { return rows[(size_t)a].Tf > rows[(size_t)b].Tf; });
        std::vector<RaggedRow> sr((size_t)B);
        std::vector<LinkRow> sl(links ? (size_t)B : 0);
        std::vector<RateRow> sq((size_t)B);
        std::vector<SlotCtl> sc(ctl ? (size_t)B : 0);
        std::vector<int64_t> so(lsnr ? (size_t)B : 0);
        for (int64_t i = 0; i < B; i++) {
            const int64_t o = idx[(size_t)i];
            sr[(size_t)i] = rows[(size_t)o];
            sq[(size_t)i] = rates[(size_t)o];
            if (ctl) sc[(size_t)i] = (*ctl)[(size_t)o];
            if (lsnr) so[(size_t)i] = lsnr_offsets[o];
            if (links) {
                const LinkRow g = (*links)[(size_t)o];
                sl[(size_t)i] = LinkRow{(int)(i - (o - g.first)), g.n};
                min_group = std::max(min_group, (int64_t)g.n);
            }
        }
        rows.swap(sr);
        if (links) links->swap(sl);
        rates.swap(sq);
        if (ctl) ctl->swap(sc);
        lsnr_off.swap(so);
    }
    std::vector<int64_t> tfs((size_t)B);
    int64_t true_frames = 0;
    for (int64_t i = 0; i < B; i++) { tfs[i] = rows[i].Tf; true_frames += tfs[i]; }
    int min_chunks = m->host_chunks;
    if (!host) {
        // cutting a large device-resident batch into pipelined chunks can cost more (persistent kernels re-pay their
        // prologues, short grids leave partial waves) than the overlap of encoder and decoder phases gains; for a few
        // streams, where everything is latency bound, the overlap wins.  dev_chunks 0 = that policy.
        min_chunks = m->dev_chunks > 0 ? m->dev_chunks : (B <= 8 ? 3 : (B <= 256 ? 2 : 1));
        // ended streams drop out at chunk boundaries only: with a spread of lengths, shorter chunks save more padded frames
        // than they cost (DeepFilterNet3, 128 streams of 1 - 20 s on one H100 at 700 W: 2 chunks 34.6 ms, 4 chunks 30.1 ms, 8 30.3)
        if (m->dev_chunks == 0 && (double)B * tfs[0] > 1.1 * (double)true_frames && min_chunks < 4) min_chunks = 4;
    }
    int64_t group = 0;
    int tc = 0;
    bool pipelined = false;
    int rc = enhance_plan(m, st, B, tfs[0], min_chunks, min_group, &group, &tc, &pipelined);
    if (rc) return rc;
    size_t off[kStateArrays];   // the aux arena holds one group's state slab and tables
    if ((rc = m->aux_arena.reserve(state_floats(m->cfg, st, (int)group, off) * sizeof(float) +
                                   (size_t)group * (sizeof(RaggedRow) + sizeof(LinkRow) + (rated ? 2 * sizeof(RateRow) : 0) +
                                                    sizeof(SlotCtl) + sizeof(int64_t)) + 8192)))
        return rc;
    // stream groups: up to `group` streams, cut only between link groups (group >= every link group, so a cut inside one
    // moves back to its first member, past b0); DeepFilterNet v1: of one frame count
    auto group_end = [&](int64_t b0) {
        int64_t b1 = B - b0 < group ? B : b0 + group;
        if (links && b1 < B && (*links)[(size_t)b1].first < b1) b1 = (*links)[(size_t)b1].first;
        if (m->cfg.model_kind == 1)
            for (int64_t i = b0 + 1; i < b1; i++)
                if (tfs[i] != tfs[b0]) { b1 = i; break; }
        return b1;
    };
    // device link tables: each stream group indexes its own streams from 0
    std::vector<LinkRow> dlinks;
    if (links) {
        dlinks = *links;
        for (int64_t b0 = 0, b1; b0 < B; b0 = b1) {
            b1 = group_end(b0);
            for (int64_t i = b0; i < b1; i++) dlinks[(size_t)i].first -= (int)b0;
        }
    }
    // device rows: the streams themselves, or (host, rated) their places in the staging buffers, sized for the largest group.
    // A rated host batch also stages its streams at their own rates: ur / dr_ are the up / down resamplers' rows.
    const bool staged = host || rated;
    std::vector<RaggedRow> drows(rows);
    std::vector<RateRow> ur(rates), dr_(rates);
    // LSNR rows: written to the caller's device buffer, or (host) staged per stream group, packed, at dlo
    const int hop = st->hop;
    auto lsnr_n = [&](int64_t i) { return (rows[(size_t)i].out_len + hop - 1) / hop; };
    std::vector<int64_t> dlo(lsnr_off);
    float *d_in = nullptr, *d_out = nullptr, *d_rin = nullptr, *d_rout = nullptr, *d_lsnr = nullptr;
    int smem_up = 0, smem_down = 0;
    int64_t n_lsnr = 0;
    if (lsnr && host)
        for (int64_t b0 = 0, b1; b0 < B; b0 = b1) {
            b1 = group_end(b0);
            int64_t gl = 0;
            for (int64_t i = b0; i < b1; i++) { dlo[(size_t)i] = gl; gl += lsnr_n(i); }
            n_lsnr = std::max(n_lsnr, gl);
        }
    if (staged) {
        int64_t n_in = 0, n_out = 0, n_rin = 0, n_rout = 0;
        for (int64_t b0 = 0, b1; b0 < B; b0 = b1) {
            b1 = group_end(b0);
            int64_t gi = 0, go = 0, gri = 0, gro = 0;
            for (int64_t i = b0; i < b1; i++) {
                drows[i].in_off = gi; drows[i].out_off = go;
                gi += rows[i].len; go += rows[i].out_len;
                const RateRow &q = rates[(size_t)i];
                ur[i] = RateRow{q.in_off, q.in_len, drows[i].in_off, rows[i].len, q.tf, q.dir};
                dr_[i] = RateRow{drows[i].out_off, rows[i].out_len, q.out_off, q.out_len, q.tf, q.dir};
                if (q.dir < 0) continue;
                if (host) {
                    ur[i].in_off = gri; dr_[i].out_off = gro;
                    gri += q.in_len; gro += q.out_len;
                }
                const RateDir &u = m->rate_up[(size_t)q.dir], &d = m->rate_down[(size_t)q.dir];
                if (u.nw * u.K <= kRateSmemFloats) smem_up = std::max(smem_up, u.nw * u.K);
                if (d.nw * d.K <= kRateSmemFloats) smem_down = std::max(smem_down, d.nw * d.K);
            }
            n_in = std::max(n_in, gi); n_out = std::max(n_out, go);
            n_rin = std::max(n_rin, gri); n_rout = std::max(n_rout, gro);
        }
        if ((rc = st->arena.reserve(sizeof(float) * (size_t)(n_in + n_out + n_rin + n_rout + n_lsnr) + 5120))) return rc;
        st->arena.reset();
        d_in = st->arena.take<float>((size_t)n_in); d_out = st->arena.take<float>((size_t)n_out);
        if (n_rin) d_rin = st->arena.take<float>((size_t)n_rin);
        if (n_rout) d_rout = st->arena.take<float>((size_t)n_rout);
        if (n_lsnr) d_lsnr = st->arena.take<float>((size_t)n_lsnr);
    }
    if (lsnr && !host) d_lsnr = lsnr;
    // the most outputs a row of rr[0, na) writes in a resampler launch
    auto max_range = [&](bool up, const RateRow *rr, int64_t na, const RateIO &io) {
        int64_t mx = 0, o0, o1;
        for (int64_t i = 0; i < na; i++) {
            if (rr[i].dir < 0) continue;
            rate_range(up, (up ? m->rate_up : m->rate_down)[(size_t)rr[i].dir], rr[i], io, &o0, &o1);
            mx = std::max(mx, o1 - o0);
        }
        return mx;
    };
    const float lim = (atten_lim_db > 0.f) ? powf(10.f, -atten_lim_db / 20.f) : 0.f;
    cudaStream_t sc = host ? m->stream : s, sh = m->h2d, sd = m->d2h;
    std::vector<cudaEvent_t> evs;
    auto order = [&](cudaStream_t from, cudaStream_t to) -> int {   // `to` waits for what has been enqueued on `from` so far
        cudaEvent_t e = nullptr;
        DFB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        evs.push_back(e);
        DFB_CUDA(cudaEventRecord(e, from));
        DFB_CUDA(cudaStreamWaitEvent(to, e, 0));
        return DFB_OK;
    };
    for (int64_t b0 = 0, b1; b0 < B && !rc; b0 = b1) {
        b1 = group_end(b0);
        const RaggedRow *hr = rows.data() + b0, *dr = drows.data() + b0;
        const int64_t *tf = tfs.data() + b0;
        ChunkHooks hooks;
        hooks.pcie = host;
        // uh / dh the group's resampler rows, rh its streams in the caller's buffers; d_prev the DNN frames of the previous
        // chunk (which streams had ended at its down-resampler launch).  In a batch at 48 kHz only, both resampler launches
        // have no outputs and return before launching, and the copies of the staging buffers at the streams' rates are empty.
        const RateRow *uh = ur.data() + b0, *dh = dr_.data() + b0, *rh = rates.data() + b0;
        RateRow *d_ur = nullptr, *d_dr = nullptr;
        int64_t d_prev = 0;
        const RateDir *d_up = m->d_rate_dirs, *d_down = m->d_rate_dirs + m->rates.size();
        hooks.before = [&](int64_t x0, int64_t x1, int64_t na, cudaStream_t cs) -> int {
            // a 48 kHz stream is copied; a stream at another rate reads what its resampler needs for the 48 kHz samples below
            // x1, its tap look-ahead included, of which earlier chunks copied those below x0's need
            const cudaMemcpyKind kind = host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
            int r = copy_streams(d_in, src, x0, na, [&](int64_t i) {
                return StreamCopy{dr[i].in_off, hr[i].in_off, uh[i].dir < 0 ? std::min(x1, hr[i].len) : x0};
            }, kind, host ? sh : cs);
            if (!r && host)
                r = copy_streams(d_rin, src, 0, na, [&](int64_t i) {
                    if (uh[i].dir < 0) return StreamCopy{0, 0, 0};
                    const RateDir &d = m->rate_up[(size_t)uh[i].dir];
                    const int64_t a = rate_up_need(d, uh[i], x0), b = rate_up_need(d, uh[i], x1);
                    return StreamCopy{uh[i].in_off + a, rh[i].in_off + a, b - a};
                }, cudaMemcpyHostToDevice, sh);
            if (!r && host) r = order(sh, cs);
            if (r) return r;
            const RateIO io{host ? d_rin : src, d_in, x0, x1, 0, 0};
            return launch_resample_rows(cs, true, d_up, d_ur, (int)na, io, max_range(true, uh, na, io), smem_up);
        };
        hooks.after = [&](int64_t y0, int64_t y1, int64_t d1, int64_t na, cudaStream_t cs) -> int {
            const RateIO io{d_out, host ? d_rout : dst, y0, y1, d_prev, d1};
            d_prev = d1;
            int r = launch_resample_rows(cs, false, d_down, d_dr, (int)na, io, max_range(false, dh, na, io), smem_down);
            if (r || (host && (r = order(cs, sd)))) return r;
            r = copy_streams(dst, d_out, y0, na, [&](int64_t i) {   // a 48 kHz stream that has ended: all of its output
                return StreamCopy{hr[i].out_off, dr[i].out_off,
                                  dh[i].dir >= 0 ? y0 : tf[i] <= d1 ? hr[i].out_len : std::min(y1, hr[i].out_len)};
            }, host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, host ? sd : cs);
            if (r || !host) return r;
            r = copy_streams(dst, d_rout, 0, na, [&](int64_t i) {
                if (dh[i].dir < 0) return StreamCopy{0, 0, 0};
                int64_t a, b;
                rate_range(false, m->rate_down[(size_t)dh[i].dir], dh[i], io, &a, &b);
                return StreamCopy{rh[i].out_off + a, dh[i].out_off + a, b - a};
            }, cudaMemcpyDeviceToHost, sd);
            if (r || !lsnr) return r;
            // LSNR values [y0 / hop, y1 / hop) carry the frames emitted in this chunk (y = e hop - delay), all of them once
            // the stream has ended
            return copy_streams(lsnr, d_lsnr, y0 / hop, na, [&](int64_t i) {
                const int64_t n = lsnr_n(b0 + i);
                return StreamCopy{lsnr_off[(size_t)(b0 + i)], dlo[(size_t)(b0 + i)], tf[i] <= d1 ? n : std::min(y1 / hop, n)};
            }, cudaMemcpyDeviceToHost, sd);
        };
        // (host) the previous group's D2H copies read the staged output and its compute the staged input: order this
        // group's first writes after them
        if (host && ((rc = order(sd, sc)) || (rc = order(sc, sh)))) break;
        // the previous group's compute still reads the state slab and table: upload this group's table behind it
        m->aux_arena.reset();
        RaggedRow *d_rows = m->aux_arena.take<RaggedRow>((size_t)(b1 - b0));
        DFB_CUDA(cudaMemcpyAsync(d_rows, dr, sizeof(RaggedRow) * (b1 - b0), cudaMemcpyHostToDevice, sc));
        LinkRow *d_links = nullptr;
        if (links) {
            d_links = m->aux_arena.take<LinkRow>((size_t)(b1 - b0));
            if (!d_links) { rc = fail(DFB_ERR_OOM, "link table arena exhausted"); break; }
            DFB_CUDA(cudaMemcpyAsync(d_links, dlinks.data() + b0, sizeof(LinkRow) * (b1 - b0), cudaMemcpyHostToDevice, sc));
        }
        if (rated) {
            d_ur = m->aux_arena.take<RateRow>((size_t)(b1 - b0));
            d_dr = m->aux_arena.take<RateRow>((size_t)(b1 - b0));
            if (!d_ur || !d_dr) { rc = fail(DFB_ERR_OOM, "resampler table arena exhausted"); break; }
            DFB_CUDA(cudaMemcpyAsync(d_ur, uh, sizeof(RateRow) * (b1 - b0), cudaMemcpyHostToDevice, sc));
            DFB_CUDA(cudaMemcpyAsync(d_dr, dh, sizeof(RateRow) * (b1 - b0), cudaMemcpyHostToDevice, sc));
        }
        BatchOut bo;
        if (ctl) {
            SlotCtl *d_ctl = m->aux_arena.take<SlotCtl>((size_t)(b1 - b0));
            if (!d_ctl) { rc = fail(DFB_ERR_OOM, "settings table arena exhausted"); break; }
            DFB_CUDA(cudaMemcpyAsync(d_ctl, ctl->data() + b0, sizeof(SlotCtl) * (b1 - b0), cudaMemcpyHostToDevice, sc));
            bo.ctl = d_ctl;
            bo.gate = gate;
        }
        if (lsnr) {
            int64_t *d_lo = m->aux_arena.take<int64_t>((size_t)(b1 - b0));
            if (!d_lo) { rc = fail(DFB_ERR_OOM, "LSNR table arena exhausted"); break; }
            DFB_CUDA(cudaMemcpyAsync(d_lo, dlo.data() + b0, sizeof(int64_t) * (b1 - b0), cudaMemcpyHostToDevice, sc));
            bo.lsnr = d_lsnr;
            bo.lsnr_offs = d_lo;
        }
        rc = enhance_group(m, st, staged ? d_in : src, staged ? d_out : dst, d_rows, tf, b1 - b0, pad, lim, tc, pipelined, sc,
                           staged ? &hooks : nullptr, d_links, links ? reduce : 0, bo);
    }
    if (host) {
        const cudaError_t e1 = cudaStreamSynchronize(sc), e2 = cudaStreamSynchronize(sd), e3 = cudaStreamSynchronize(sh);
        const cudaError_t e = e1 != cudaSuccess ? e1 : (e2 != cudaSuccess ? e2 : e3);
        if (!rc && e != cudaSuccess) rc = fail(DFB_ERR_CUDA, "enhance_host failed: %s", cudaGetErrorString(e));
    }
    for (cudaEvent_t e : evs) cudaEventDestroy(e);
    m->arena.reset();
    m->arena1.reset();
    return rc;
}

// An equal-length batch [B][T] at 48 kHz: stream b is {b T, T, b out_len}.  pad = True appends fft zeros
// (enhance.py:230-233): Tf = (T + fft) / hop.
static int equal_rows(const dfb_state *st, int64_t B, int64_t T, int pad, std::vector<RaggedRow> &rows, std::vector<RateRow> &rr) {
    const int64_t Tf = (pad ? T + st->fft : T) / st->hop, out_len = dfb_enhance_out_len(st, T, pad);
    if (Tf <= 0) return fail(DFB_ERR_INVALID, "input shorter than one hop");
    rows.resize((size_t)B);
    rr.resize((size_t)B);
    for (int64_t b = 0; b < B; b++) {
        rows[(size_t)b] = RaggedRow{b * T, T, b * out_len, out_len, Tf};
        rr[(size_t)b] = RateRow{b * T, T, b * out_len, out_len, Tf, -1};
    }
    return DFB_OK;
}

extern "C" int dfb_enhance(dfb_model *m, dfb_state *st, const float *d_audio, int64_t B, int64_t T, int pad,
                           float atten_lim_db, float *d_out, void *stream) {
    if (!m || !st || !d_audio || !d_out) return fail(DFB_ERR_INVALID, "null argument");
    if (B <= 0 || T <= 0) return fail(DFB_ERR_INVALID, "empty input");
    if (int rcs = check_state(m, st)) return rcs;
    std::vector<RaggedRow> rows;
    std::vector<RateRow> rr;
    if (int rc = equal_rows(st, B, T, pad, rows, rr)) return rc;
    DFB_CUDA(cudaSetDevice(m->device));
    return enhance_rows(m, st, rows, rr, d_audio, d_out, pad, atten_lim_db, false, (cudaStream_t)stream);
}

extern "C" int dfb_enhance_host(dfb_model *m, dfb_state *st, const float *h_audio, int64_t B, int64_t T, int pad,
                                float atten_lim_db, float *h_out) {
    if (!m || !st || !h_audio || !h_out) return fail(DFB_ERR_INVALID, "null argument");
    if (B <= 0 || T <= 0) return fail(DFB_ERR_INVALID, "empty input");
    if (int rcs = check_state(m, st)) return rcs;
    std::vector<RaggedRow> rows;
    std::vector<RateRow> rr;
    if (int rc = equal_rows(st, B, T, pad, rows, rr)) return rc;
    DFB_CUDA(cudaSetDevice(m->device));
    return enhance_rows(m, st, rows, rr, h_audio, h_out, pad, atten_lim_db, true, nullptr);
}

// Validates the per-stream settings of dfb_enhance_ragged (n of them, one per stream in the caller's order) and returns
// them as apply-kernel rows with sw = 0 (*gate: some stream gates).  Linked streams (`links` non-empty) must agree within
// their group.  The table runs the specialised CTL apply kernel, so it follows the slot path's model rules.
static int settings_plan(const dfb_model *m, const dfb_enhance_settings *set, int64_t n, int64_t B, const std::vector<LinkRow> &links,
                         std::vector<SlotCtl> &ctl, bool *gate) {
    if (n != B) return fail(DFB_ERR_INVALID, "%lld settings for %lld streams", (long long)n, (long long)B);
    const dfb_model_config &c = m->cfg;
    if (c.model_kind == 1) return fail(DFB_ERR_UNSUPPORTED, "per-stream settings: DeepFilterNet v1 is not supported");
    if (c.df_order != 5 || c.nb_df != 96 || c.nb_erb != 32)
        return fail(DFB_ERR_UNSUPPORTED, "per-stream settings are built for df_order 5, nb_df 96 and 32 ERB bands");
    ctl.resize((size_t)B);
    *gate = false;
    for (int64_t b = 0; b < B; b++) {
        const dfb_enhance_settings &e = set[b];
        if (std::isnan(e.atten_lim_db)) return fail(DFB_ERR_INVALID, "stream %lld: attenuation limit is NaN", (long long)b);
        if (!(std::isfinite(e.post_filter_beta) && e.post_filter_beta >= 0.f))
            return fail(DFB_ERR_INVALID, "stream %lld: post-filter beta must be finite and >= 0", (long long)b);
        if (e.lsnr_gating && (std::isnan(e.min_db_thresh) || std::isnan(e.max_db_erb_thresh) || std::isnan(e.max_db_df_thresh)))
            return fail(DFB_ERR_INVALID, "stream %lld: an LSNR threshold is NaN", (long long)b);
        if (e.post_filter_beta > 0.f && c.model_kind != 3)
            return fail(DFB_ERR_UNSUPPORTED, "per-stream post-filter beta: DeepFilterNet3 topologies only (DeepFilterNet2's beta is fixed)");
        if (e.lsnr_gating && c.model_kind != 3) return fail(DFB_ERR_UNSUPPORTED, "LSNR stage gating: DeepFilterNet3 topologies only");
        const float lim = e.atten_lim_db > 0.f ? powf(10.f, -e.atten_lim_db / 20.f) : 0.f;
        SlotCtl r{lim, e.post_filter_beta, lim, e.post_filter_beta, 0};
        if (e.lsnr_gating) { r.th_min = e.min_db_thresh; r.th_erb = e.max_db_erb_thresh; r.th_df = e.max_db_df_thresh; r.gate = 1; }
        ctl[(size_t)b] = r;
        *gate |= r.gate != 0;
    }
    for (int64_t b = 0; b < (int64_t)links.size(); b++)
        if (memcmp(&ctl[(size_t)b], &ctl[(size_t)links[(size_t)b].first], sizeof(SlotCtl)))
            return fail(DFB_ERR_INVALID, "stream %lld: the streams of a link group take one setting", (long long)b);
    return DFB_OK;
}

// The body of dfb_enhance_ragged(_host): `group_sizes` null for a call without link groups, `rates` null for one whose
// streams are all at 48 kHz, `settings` null for one setting (atten_lim_db, the model's post filter, no gating) for every
// stream, `lsnr` null for no LSNR rows.
static int enhance_ragged(dfb_model *m, dfb_state *st, const float *src, int64_t in_numel, const int64_t *in_offsets,
                          const int64_t *lengths, int64_t B, int pad, float atten_lim_db, float *dst, int64_t out_numel,
                          const int64_t *out_offsets, const int64_t *group_sizes, int64_t n_groups, int reduce_mask,
                          const int32_t *rates, const dfb_enhance_settings *settings, int64_t n_settings, float *lsnr,
                          int64_t lsnr_numel, const int64_t *lsnr_offsets, bool host, cudaStream_t s) {
    if (!m || !st || !src || !dst) return fail(DFB_ERR_INVALID, "null argument");
    if (int rcs = check_state(m, st)) return rcs;
    std::vector<RaggedRow> rows;
    std::vector<RateRow> rr;
    std::vector<LinkRow> links;
    std::vector<SlotCtl> ctl;
    bool gate = false;
    if (int rc = batch_plan(m, st, in_numel, in_offsets, lengths, B, pad, out_numel, out_offsets, rates, rows, rr)) return rc;
    if (group_sizes)
        if (int rc = link_plan(m, rows, rr, group_sizes, n_groups, reduce_mask, links)) return rc;
    if (settings)
        if (int rc = settings_plan(m, settings, n_settings, B, links, ctl, &gate)) return rc;
    if (lsnr) {
        if (!lsnr_offsets) return fail(DFB_ERR_INVALID, "LSNR output without offsets");
        if (m->cfg.model_kind == 1) return fail(DFB_ERR_UNSUPPORTED, "LSNR rows: DeepFilterNet v1 is not supported");
        for (int64_t b = 0; b < B; b++) {
            const int64_t o = lsnr_offsets[b], n = (rows[(size_t)b].out_len + st->hop - 1) / st->hop;
            if (o < 0 || o > lsnr_numel - n)
                return fail(DFB_ERR_INVALID, "stream %lld's LSNR row reaches outside the LSNR output (%lld values)", (long long)b,
                            (long long)lsnr_numel);
        }
    }
    DFB_CUDA(cudaSetDevice(m->device));
    return enhance_rows(m, st, rows, rr, src, dst, pad, atten_lim_db, host, s, links.empty() ? nullptr : &links, reduce_mask,
                        settings ? &ctl : nullptr, gate, lsnr, lsnr_offsets);
}

extern "C" int dfb_enhance_ragged(dfb_model *m, dfb_state *st, const float *d_audio, int64_t in_numel, const int64_t *in_offsets,
                                  const int64_t *lengths, int64_t B, int pad, float atten_lim_db, float *d_out, int64_t out_numel,
                                  const int64_t *out_offsets, const int64_t *group_sizes, int64_t n_groups, int reduce_mask,
                                  const int32_t *rates, const dfb_enhance_settings *settings, int64_t n_settings, float *d_lsnr,
                                  int64_t lsnr_numel, const int64_t *lsnr_offsets, void *stream) {
    return enhance_ragged(m, st, d_audio, in_numel, in_offsets, lengths, B, pad, atten_lim_db, d_out, out_numel, out_offsets,
                          group_sizes, n_groups, reduce_mask, rates, settings, n_settings, d_lsnr, lsnr_numel, lsnr_offsets, false,
                          (cudaStream_t)stream);
}

extern "C" int dfb_enhance_ragged_host(dfb_model *m, dfb_state *st, const float *h_audio, int64_t in_numel, const int64_t *in_offsets,
                                       const int64_t *lengths, int64_t B, int pad, float atten_lim_db, float *h_out, int64_t out_numel,
                                       const int64_t *out_offsets, const int64_t *group_sizes, int64_t n_groups, int reduce_mask,
                                       const int32_t *rates, const dfb_enhance_settings *settings, int64_t n_settings, float *h_lsnr,
                                       int64_t lsnr_numel, const int64_t *lsnr_offsets) {
    return enhance_ragged(m, st, h_audio, in_numel, in_offsets, lengths, B, pad, atten_lim_db, h_out, out_numel, out_offsets,
                          group_sizes, n_groups, reduce_mask, rates, settings, n_settings, h_lsnr, lsnr_numel, lsnr_offsets, true,
                          nullptr);
}

// Debug aid: one of the model's offline resamplers alone over a ragged batch, in the launches the chunk loop would make
extern "C" int dfb_debug_resample_rows(int up, const dfb_model *m, const float *d_in, const int64_t *in_offsets,
                                       const int64_t *in_lengths, const int32_t *rates, int64_t B, float *d_out,
                                       const int64_t *out_offsets, const int64_t *h_bounds, int64_t n_bounds, void *stream) {
    if (!m || !d_in || !in_offsets || !in_lengths || !rates || !d_out || !out_offsets || !h_bounds || n_bounds <= 0 || B <= 0 ||
        B > 65535)
        return fail(DFB_ERR_INVALID, "bad argument");
    std::vector<RateRow> rows((size_t)B);
    int smem = 0;
    for (int64_t b = 0; b < B; b++) {
        const auto it = std::find(m->rates.begin(), m->rates.end(), (int)rates[b]);
        if (it == m->rates.end()) return fail(DFB_ERR_INVALID, "row %lld: sample rate %d Hz is not registered", (long long)b, rates[b]);
        if (in_lengths[b] <= 0) return fail(DFB_ERR_INVALID, "row %lld has length %lld", (long long)b, (long long)in_lengths[b]);
        const int dir = (int)(it - m->rates.begin());
        const RateDir &d = (up ? m->rate_up : m->rate_down)[(size_t)dir];
        const int64_t n = up ? len_at_48k(in_lengths[b], rates[b]) : len_from_48k(in_lengths[b], rates[b]);
        rows[(size_t)b] = RateRow{in_offsets[b], in_lengths[b], out_offsets[b], n, INT64_MAX, dir};
        if (d.nw * d.K <= kRateSmemFloats) smem = std::max(smem, d.nw * d.K);
    }
    for (int64_t i = 0; i < n_bounds; i++)
        if (h_bounds[i] <= (i ? h_bounds[i - 1] : 0)) return fail(DFB_ERR_INVALID, "chunk bounds must increase from > 0");
    if (int rc = use_device(m->device)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const RateDir *dirs = m->d_rate_dirs + (up ? 0 : m->rates.size());
    RateRow *d_rows = nullptr;
    int rc = DFB_OK;
    if (cudaMalloc(&d_rows, sizeof(RateRow) * B) != cudaSuccess ||
        cudaMemcpyAsync(d_rows, rows.data(), sizeof(RateRow) * B, cudaMemcpyHostToDevice, s) != cudaSuccess)
        rc = fail(DFB_ERR_OOM, "debug buffers");
    // up: launch c writes the 48 kHz outputs [bounds[c - 1], bounds[c]); down: the outputs complete once the 48 kHz input is
    // known up to bounds[c]
    for (int64_t i = 0; i < n_bounds && !rc; i++) {
        const RateIO io{d_in, d_out, i ? h_bounds[i - 1] : 0, h_bounds[i], 0, 0};
        int64_t mx = 0, o0, o1;
        for (const RateRow &r : rows) {
            rate_range(up != 0, (up ? m->rate_up : m->rate_down)[(size_t)r.dir], r, io, &o0, &o1);
            mx = std::max(mx, o1 - o0);
        }
        rc = launch_resample_rows(s, up != 0, dirs, d_rows, (int)B, io, mx, smem);
    }
    cudaStreamSynchronize(s);
    if (d_rows) cudaFree(d_rows);
    return rc;
}

// ============================================================== streaming API ====
// Frame-incremental processing with carried state: the batched counterpart of the reference's single-stream runtime
// (libDF/src/tract.rs:509-642 `DfTract::process`, C ABI libDF/src/capi.rs:83-253 df_create / df_process_frame / df_free).
// Every call feeds n >= 1 hops per stream and returns n hops; the output trails the input by `latency` frames
// (max(conv_lookahead, df_lookahead), + df_lookahead for DeepFilterNet2) on top of the STFT's own fft - hop samples,
// i.e. the concatenated output equals enhance(pad=False) of the concatenated input delayed by latency * hop samples.
// Streaming slots (dfb_stream_open_slots / dfb_stream_close_slots; DESIGN.md section 5c).  Each of the handle's B slots
// opens and closes on its own under the handle's single clock: a slot opened at analysis frame a starts a fresh stream
// whose frame 0 is a (its state-slab row is initialised, the kernels that look back in time read padding before a), and a
// closed slot's stream ends at the frame its input had reached (rows[b].Tf, as a ragged stream's end), then emits its
// look-ahead tail over the next `latency` hops and becomes free.  Open and closing slots are the prefix [0, n_act) of the
// state slab, so every kernel runs over B = n_act rows only; free slots are not computed and return zeros.
enum { kSlotFree = 0, kSlotOpen = 1, kSlotClosing = 2 };
constexpr int64_t kOpenEnd = 0x7fffffff;   // rows[b].Tf of an open slot: kernels take Tf - w0 as int

// The state-slab rows of one call: ops[i] = {dst, src} sets row dst of every array to row src as the last call left it, or
// (src < 0) to the initial state of a fresh stream: zeros, and the normalisation EMA states at the values launch_feat_norm
// starts from without a state.  Sources and destinations overlap when rows close up behind a freed slot, so the moves come
// first in `ops` and pass 0 copies their sources to scratch rows [i][lay.row_floats]; pass 1 writes every destination.
// Two launches whatever the number of rows.  grid (x, ops of the pass, kStateArrays).
__global__ void k_slot_rows(float *__restrict__ slab, StateLayout lay, int Bs, const int2 *__restrict__ ops, float *__restrict__ scratch,
                            int pass, int E, int Fd) {
    const int i = blockIdx.y, a = blockIdx.z;
    const int2 op = ops[i];
    const int64_t n = (int64_t)lay.layers[a] * lay.per_row[a];
    float *sc = scratch + (int64_t)i * lay.row_floats + lay.row_off[a];
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        if (pass == 0) {
            sc[e] = slab[state_elem(lay, Bs, a, op.y, e)];
            continue;
        }
        slab[state_elem(lay, Bs, a, op.x, e)] = op.y >= 0 ? sc[e] : state_init(a, e, E, Fd);
    }
}

// carried analysis memory: row b's last input hop, read where rows[b] says its input row is
__global__ void k_carry_hop(float *__restrict__ ana_mem, const float *__restrict__ in, const RaggedRow *__restrict__ rows, int64_t last,
                            int hop) {
    const int b = blockIdx.x;
    for (int i = threadIdx.x; i < hop; i += blockDim.x) ana_mem[(int64_t)b * hop + i] = in[rows[b].in_off + last + i];
}

struct dfb_stream {
    dfb_model *m;
    dfb_state *st;
    int device;                                        // the model's, kept so that freeing never reads the model
    int B;
    float lim;
    StreamState S;
    float *slab = nullptr;
    bool gating = false;
    float th[3] = {-10.f, 30.f, 20.f};                 // tract.rs:180-185 defaults
    int gating_mode = -1;                              // dfb_stream_set_gating_mode, -1: the model's
    float *stage_in = nullptr, *stage_out = nullptr;   // device staging of the *_host entry point
    size_t stage_in_cap = 0, stage_out_cap = 0;
    bool fed = false;                                  // a frame has been processed since create / reset
    bool slot_ops = false;                             // a slot operation, setter or flush since create / reset
    // streaming slots (slots_init: every slot open from frame 0 in row b = slot b)
    std::vector<int> slot_state, slot_row, row_slot;   // kSlot*; slot -> row of the active prefix (-1 free); row -> slot
    std::vector<int64_t> slot_first, slot_end;         // absolute first frame; end frame of a closing slot
    int n_act = 0;
    std::vector<int> row_src;                          // per row: its state-slab row at the last call, or -1: a fresh stream
    // held sessions (dfb_stream_hold_slots; DESIGN.md section 5p): live rows [n_act, n_live) that no call computes
    std::vector<char> slot_held;
    std::vector<int64_t> slot_held_frames;             // per slot: frames held since the LSNR head started (its LSNR start)
    int n_live = 0;
    int64_t rows_moved = 0;                            // rows k_slot_rows wrote at the last call (dfb_debug_stream_rows_moved)
    // runtime gating: per slot, whether its decoder tails were kept by its own last DNN call (S.rt_valid of that call)
    std::vector<char> slot_rt;
    unsigned char *d_halo = nullptr;                   // per row: take the tails from the halo (GateRun::halo)
    // slot groups (dfb_stream_open_linked, or the fixed channel groups of dfb_stream_set_mask_reduce): per slot the slot of
    // its group's channel 0 (-1 free) and the group's channel count.  A group's rows are contiguous in the active prefix,
    // in channel order.
    std::vector<int> slot_grp, slot_nch;
    int group_reduce = 0;                              // mask reduction of the groups (dfb_stream_set_mask_reduce)
    int fixed_nch = 1;                                 // channels of the fixed groups (dfb_stream_set_mask_reduce), 1: none
    bool tab_dirty = true;                             // rows / first frames / link groups to re-upload
    int64_t tab_n = -1;                                // ... for calls of this many input hops
    bool tab_linked = false;                           // the uploaded table has a linked group of more than one channel
    RaggedRow *d_rows = nullptr;
    int64_t *d_first = nullptr;
    LinkRow *d_grp = nullptr;
    // per-slot settings (dfb_stream_set_atten_lim / _post_filter_beta).  ctl_on: a setter has run since create / reset, so
    // the per-row table goes to the apply kernel.
    bool ctl_on = false;
    std::vector<float> slot_lim, slot_beta;            // per slot: own limit (linear, 0 off) / beta, or NaN: the handle's
    std::vector<signed char> slot_gate;                // per slot: own LSNR gating (0 off, 1 on with slot_th), or -1: the handle's
    std::vector<float> slot_th;                        // per slot: own thresholds [3]
    bool ctl_gate = false;                             // a row of the uploaded table gates
    std::vector<char> slot_fresh;                      // per slot: opened since the last call (no previous setting)
    std::vector<SlotCtl> slot_ctl;                     // per slot: the settings of the last call and the one before
    std::vector<SlotCtl> ctl_up;                       // per row: the table on the device
    SlotCtl *d_ctl = nullptr;
    float beta_run = 0.f;                              // the handle's default beta at the last call
    // LSNR output: computed for DNN frames >= lsnr_from, the first one after the first request since create / reset
    int64_t lsnr_from = -1;
    float *stage_lsnr = nullptr;                       // device staging of dfb_stream_process_host_lsnr
    size_t stage_lsnr_cap = 0;
    // spectral handle (dfb_stream_create_spec): spectrum frames in, the network's outputs out; runs the LSNR head always
    bool spectral = false;
    int *d_slotmap = nullptr;                          // per slot its row of the active prefix, -1 free
    float *spec_stage_in = nullptr, *spec_stage_out = nullptr;   // device staging of dfb_stream_process_spec_host
    size_t spec_in_cap = 0, spec_out_cap = 0;
    // sample rate (dfb_stream_set_sample_rate): 0 runs at the model's 48 kHz; else the caller's rate, resampled up into the
    // unchanged 48 kHz slot path and back down.  A mixed-rate handle (dfb_stream_add_slot_rate) stays at 48 kHz and runs
    // each slot in its own direction of the resamplers: the identity at 48 kHz, or one of its registered rates.  The
    // histories are arrays 13 / 14 of the state slab, as wide as the directions' largest S.
    int rate = 0;
    std::vector<int> rs_rates;                         // per direction its rate: {rate}, {48000, registered ...} or none
    ResampleDirs rs_up{}, rs_down{};
    std::vector<float *> rs_taps;                      // the directions' taps on the device
    std::vector<int> slot_dir;                         // per slot: its session's direction
    float *rs_in = nullptr, *rs_out = nullptr;         // the slot path's 48 kHz input / output [B][n * 480]
    size_t rs_in_cap = 0, rs_out_cap = 0;
    float *rs_lsnr = nullptr;                          // flush: the LSNR of its two passes
    size_t rs_lsnr_cap = 0;
    float *sess_stage = nullptr;                       // device staging of dfb_stream_export / import_sessions_host
    size_t sess_stage_cap = 0;
    std::vector<ResampleRow> rs_rows;                  // the live rows' table on the device
    ResampleRow *d_rs = nullptr;
};

// a handle that runs the resamplers: at another rate than 48 kHz, or mixed-rate
static bool resampled(const dfb_stream *h) { return !h->rs_rates.empty(); }
static bool mixed_rate(const dfb_stream *h) { return !h->rate && resampled(h); }
// per-row floats of one resampler's histories: its directions' largest S (0 without resamplers)
static int rs_hist(const dfb_stream *h, const ResampleDirs &d) {
    int S = 0;
    for (size_t i = 0; i < h->rs_rates.size(); i++) S = std::max(S, d.d[i].S);
    return S;
}
static size_t stream_state_floats(const dfb_stream *h, size_t off[kStateArrays], StateLayout *lay = nullptr) {
    return state_floats(h->m->cfg, h->st, h->B, off, lay, rs_hist(h, h->rs_up), rs_hist(h, h->rs_down));
}

// the handle's default post-filter beta: the model's option (0 = off) for DeepFilterNet3; per-row beta is not used for
// DeepFilterNet2, whose post filter acts on the ERB gains with a fixed beta
static float default_beta(const dfb_model *m) { return (m->cfg.model_kind == 3 && m->post_filter) ? m->pf_beta : 0.f; }

// The slot tables of a new or reset handle: every slot open, its stream started at frame 0 in row b = slot b, with the
// handle's settings, and the fixed channel groups of dfb_stream_set_mask_reduce (one group per slot without them).
// Device rows follow at the next call.
static void slots_init(dfb_stream *h) {
    const size_t B = (size_t)h->B;
    h->slot_state.assign(B, kSlotOpen);
    h->slot_row.resize(B); h->row_slot.resize(B); h->row_src.resize(B); h->slot_grp.resize(B);
    std::iota(h->slot_row.begin(), h->slot_row.end(), 0);
    std::iota(h->row_slot.begin(), h->row_slot.end(), 0);
    std::iota(h->row_src.begin(), h->row_src.end(), 0);
    for (int b = 0; b < h->B; b++) h->slot_grp[(size_t)b] = b - b % h->fixed_nch;
    h->slot_nch.assign(B, h->fixed_nch);
    h->slot_first.assign(B, 0);
    h->slot_end.assign(B, kOpenEnd);
    h->slot_dir.assign(B, 0);
    h->n_act = h->n_live = h->B;
    h->slot_held.assign(B, 0);
    h->slot_held_frames.assign(B, 0);
    h->slot_rt.assign(B, 0);
    h->tab_dirty = true;
    h->slot_lim.assign(B, NAN);
    h->slot_beta.assign(B, NAN);
    h->slot_gate.assign(B, -1);
    h->slot_th.assign(3 * B, 0.f);
    h->slot_fresh.assign(B, 0);
    h->slot_ctl.assign(B, SlotCtl{});
    h->ctl_on = false;
    h->slot_ops = false;
}

static int stream_new(dfb_stream **out, dfb_model *m, dfb_state *st, int64_t B, float atten_lim_db, bool spectral) {
    if (!out || !m || !st || B <= 0 || B > 65535) return fail(DFB_ERR_INVALID, "bad argument");
    *out = nullptr;
    if (int rcs = check_state(m, st)) return rcs;
    if (m->cfg.model_kind == 1)
        return fail(DFB_ERR_UNSUPPORTED, "DeepFilterNet v1 runs as one window per signal (forward_v1): no frame-incremental API");
    DFB_CUDA(cudaSetDevice(m->device));
    dfb_stream *h = new dfb_stream();
    h->m = m; h->st = st; h->device = m->device; h->B = (int)B;
    h->lim = (atten_lim_db > 0.f) ? powf(10.f, -atten_lim_db / 20.f) : 0.f;
    h->spectral = spectral;
    if (spectral) h->lsnr_from = 0;
    size_t off[kStateArrays];
    const size_t n = state_floats(m->cfg, st, (int)B, off);
    auto dev = [](auto **p, size_t bytes) {
        if (cudaMalloc(p, bytes) == cudaSuccess) return true;
        *p = nullptr;
        return false;
    };
    if (!dev(&h->slab, n * sizeof(float)) || !dev(&h->d_rows, sizeof(RaggedRow) * B) || !dev(&h->d_first, sizeof(int64_t) * B) ||
        !dev(&h->d_grp, sizeof(LinkRow) * B)) {
        dfb_stream_free(h);
        return fail(DFB_ERR_OOM, "stream state allocation failed");
    }
    cudaMemset(h->slab, 0, n * sizeof(float));
    state_bind(h->S, h->slab, off, (int)B);
    slots_init(h);
    h->beta_run = default_beta(m);
    *out = h;
    return DFB_OK;
}

extern "C" int dfb_stream_create(dfb_stream **out, dfb_model *m, dfb_state *st, int64_t B, float atten_lim_db) {
    return stream_new(out, m, st, B, atten_lim_db, false);
}
// df_process_frame_raw's handle: spectrum frames in, gains / coefs / LSNR / stage out (no STFT, nothing applied)
extern "C" int dfb_stream_create_spec(dfb_stream **out, dfb_model *m, dfb_state *st, int64_t B) {
    return stream_new(out, m, st, B, 0.f, true);
}

extern "C" void dfb_stream_free(dfb_stream *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->slab) cudaFree(h->slab);
    if (h->stage_in) cudaFree(h->stage_in);
    if (h->stage_out) cudaFree(h->stage_out);
    if (h->d_rows) cudaFree(h->d_rows);
    if (h->d_first) cudaFree(h->d_first);
    if (h->d_grp) cudaFree(h->d_grp);
    if (h->d_ctl) cudaFree(h->d_ctl);
    if (h->d_halo) cudaFree(h->d_halo);
    if (h->stage_lsnr) cudaFree(h->stage_lsnr);
    if (h->d_slotmap) cudaFree(h->d_slotmap);
    if (h->spec_stage_in) cudaFree(h->spec_stage_in);
    if (h->spec_stage_out) cudaFree(h->spec_stage_out);
    for (float *p : {h->rs_in, h->rs_out, h->rs_lsnr, h->sess_stage})
        if (p) cudaFree(p);
    for (float *p : h->rs_taps) cudaFree(p);
    if (h->d_rs) cudaFree(h->d_rs);
    delete h;
}

extern "C" int dfb_stream_reset(dfb_stream *h) {
    if (!h) return fail(DFB_ERR_INVALID, "null stream");
    size_t off[kStateArrays];
    stream_state_floats(h, off);
    state_bind(h->S, h->slab, off, h->B);
    h->fed = false;
    slots_init(h);
    h->lsnr_from = h->spectral ? 0 : -1;
    return DFB_OK;
}

// Linked channels on a stream handle: streams g * channels + c (c < channels) are the channels of recording g and share one
// ERB mask (reduce_mask max / mean, as dfb_enhance_ragged's link groups): fixed slot groups, which survive a reset and take no
// slot operations.  Only before the first frame of a new or reset handle: the frame re-synthesised for the overlap-add
// tail at the next call would otherwise mix the two settings.  channels = 1 records the reduction of the slot groups
// opened later (dfb_stream_open_linked).
extern "C" int dfb_stream_set_mask_reduce(dfb_stream *h, int channels, int reduce_mask) {
    if (!h) return fail(DFB_ERR_INVALID, "null stream");
    if (h->fed) return fail(DFB_ERR_INVALID, "mask reduction set after the first frame: reset the stream first");
    if (h->slot_ops) return fail(DFB_ERR_UNSUPPORTED, "mask reduction set after slot operations: reset the stream first");
    if (reduce_mask != kReduceNone && reduce_mask != kReduceMax && reduce_mask != kReduceMean)
        return fail(DFB_ERR_INVALID, "reduce_mask %d is not 0 (none), 1 (max) or 2 (mean)", reduce_mask);
    if (channels <= 0 || h->B % channels) return fail(DFB_ERR_INVALID, "%d streams are not groups of %d channels", h->B, channels);
    h->group_reduce = reduce_mask;
    h->fixed_nch = reduce_mask == kReduceNone ? 1 : channels;
    slots_init(h);
    return DFB_OK;
}

// LSNR stage gating of the Rust runtime (libDF/src/tract.rs:658-672; thresholds tract.rs:180-185, DfParams of
// deep-filter / capi.rs).  Off by default: the Python path this library mirrors does not gate.  DeepFilterNet3 only on
// audio handles (the apply kernel gates mode 1); a spectral handle gates in k_spec_emit, for DeepFilterNet2 too.
extern "C" int dfb_stream_set_gating_mode(dfb_stream *h, int mode) {
    if (!h) return fail(DFB_ERR_INVALID, "null stream");
    if (mode != -1 && mode != DFB_GATING_APPLY && mode != DFB_GATING_RUNTIME) return fail(DFB_ERR_INVALID, "gating mode %d", mode);
    h->gating_mode = mode;
    return DFB_OK;
}

extern "C" int dfb_stream_set_lsnr_thresholds(dfb_stream *h, int enable, float min_db_thresh, float max_db_erb_thresh,
                                              float max_db_df_thresh) {
    if (!h) return fail(DFB_ERR_INVALID, "null stream");
    if (enable && h->m->cfg.model_kind != 3 && !h->spectral)
        return fail(DFB_ERR_UNSUPPORTED, "LSNR stage gating: DeepFilterNet3 topologies only");
    h->gating = enable != 0;
    h->th[0] = min_db_thresh; h->th[1] = max_db_erb_thresh; h->th[2] = max_db_df_thresh;
    return DFB_OK;
}

// hops the 48 kHz slot path's output trails its input by
static int64_t path_latency(const dfb_stream *h) {
    if (h->spectral) return h->m->cfg.conv_lookahead;   // the outputs wait for the encoder's look-ahead only
    const ChunkGeom g = chunk_geom(h->m->cfg);
    return g.Lmax + g.lag;
}
// a resampled session ends one hop later in the slot path (its zero extension fills the resamplers' look-ahead); a
// mixed-rate handle's flush returns its longest drain
extern "C" int64_t dfb_stream_latency_frames(const dfb_stream *h) { return h ? path_latency(h) + (resampled(h) ? 1 : 0) : -1; }
extern "C" int64_t dfb_stream_frame_length(const dfb_stream *h) {   // capi.rs df_get_frame_length
    return h ? (h->rate ? h->rate / 100 : h->st->hop) : -1;
}
// a resampled handle's signal delay on top of the 48 kHz handle's, in samples of its rate: D r / 48000 + E
extern "C" int64_t dfb_stream_latency_samples(const dfb_stream *h) {
    if (!h) return -1;
    const ResampleDir &u = h->rs_up.d[0];
    return h->rate ? (int64_t)u.Z / u.nw * u.og + h->rs_down.d[0].Z : 0;
}

// ---- streaming slots: host bookkeeping.  Device rows follow at the next call (stream_step moves them first, by row_src).
// the slot becomes free (and not held); its row stays among the live rows until rows_layout
static void slot_release(dfb_stream *h, int slot) {
    h->slot_row[(size_t)slot] = -1;
    h->slot_grp[(size_t)slot] = -1;
    h->slot_nch[(size_t)slot] = 0;
    h->slot_state[(size_t)slot] = kSlotFree;
    h->slot_held[(size_t)slot] = 0;
}

// The live rows' layout: the advancing groups (open or closing, not held) are the prefix [0, n_act), the held groups the
// rows [n_act, n_live) behind it, each group contiguous and in channel order; the rows of freed slots leave.  A group
// that lies inside its region keeps its row; the others fill the holes first fit, so a row that leaves the prefix is
// replaced by one from its end instead of the prefix closing up (the region falls back to packing its groups in order
// when linked groups fragment the holes).  A row that moves carries its source row (row_src) along: the next call moves
// the state-slab rows in one pass (k_slot_rows), however many rows moved.
static void rows_layout(dfb_stream *h) {
    struct Grp { int row, n; bool held; };
    std::vector<Grp> grps;
    int n_adv = 0, n_live = 0;
    for (int r = 0; r < h->n_live;) {
        const int b = h->row_slot[(size_t)r];
        if (h->slot_state[(size_t)b] == kSlotFree) { r++; continue; }
        const int n = h->slot_nch[(size_t)b];   // r holds the group's channel 0
        const bool held = h->slot_held[(size_t)b] != 0;
        grps.push_back(Grp{r, n, held});
        if (!held) n_adv += n;
        n_live += n;
        r += n;
    }
    std::vector<int> to(grps.size(), -1);   // per group its new first row
    for (int region = 0; region < 2; region++) {
        const bool held = region == 1;
        const int lo = held ? n_adv : 0, hi = held ? n_live : n_adv;
        std::vector<char> taken((size_t)(hi - lo), 0);
        for (size_t k = 0; k < grps.size(); k++) {
            const Grp &g = grps[k];
            if (g.held != held || g.row < lo || g.row + g.n > hi) continue;
            to[k] = g.row;
            std::fill(taken.begin() + (g.row - lo), taken.begin() + (g.row - lo + g.n), (char)1);
        }
        bool fits = true;
        for (size_t k = 0; k < grps.size() && fits; k++) {
            if (grps[k].held != held || to[k] >= 0) continue;
            const int n = grps[k].n;
            int at = -1;
            for (int q = 0, run = 0; q < hi - lo && at < 0; q++) {
                run = taken[(size_t)q] ? 0 : run + 1;
                if (run == n) at = q - n + 1;
            }
            if (at < 0) { fits = false; break; }
            to[k] = lo + at;
            std::fill(taken.begin() + at, taken.begin() + at + n, (char)1);
        }
        if (!fits)
            for (size_t k = 0, q = (size_t)lo; k < grps.size(); k++)
                if (grps[k].held == held) { to[k] = (int)q; q += (size_t)grps[k].n; }
    }
    const std::vector<int> slot_of(h->row_slot), src_of(h->row_src);
    bool moved = n_live != h->n_live || n_adv != h->n_act;
    for (size_t k = 0; k < grps.size(); k++)
        for (int c = 0; c < grps[k].n; c++) {
            const int from = grps[k].row + c, r = to[k] + c, b = slot_of[(size_t)from];
            moved |= r != from;
            h->row_slot[(size_t)r] = b;
            h->row_src[(size_t)r] = src_of[(size_t)from];
            h->slot_row[(size_t)b] = r;
        }
    if (moved) h->tab_dirty = true;
    h->n_act = n_adv;
    h->n_live = n_live;
}

// closing slots whose last frame has been output become free: `out_end` is the frame after the last output hop so far
// (a1 - latency after a process call, a1 after a flush).  The members of a group share their end frame: they leave together.
static void slots_retire(dfb_stream *h, int64_t out_end) {
    bool freed = false;
    for (int b = 0; b < h->B; b++)
        if (h->slot_state[(size_t)b] == kSlotClosing && h->slot_end[(size_t)b] <= out_end) {
            slot_release(h, b);
            freed = true;
        }
    if (freed) rows_layout(h);   // (no row leaves: the layout stands)
}

static void slot_close(dfb_stream *h, int slot) {
    if (h->slot_state[(size_t)slot] != kSlotOpen) return;
    h->slot_state[(size_t)slot] = kSlotClosing;
    // the stream ends after the input it has been fed; a resampled session one hop later, the hop its zero extension fills
    h->slot_end[(size_t)slot] = h->S.a1 + (resampled(h) ? h->rs_up.d[h->slot_dir[(size_t)slot]].ext : 0);
    h->tab_dirty = true;
}

static void holds_lift_all(dfb_stream *h);

// After a flush every stream has ended: all slots are free once their tails are out.  Without look-ahead a flush computes
// nothing and only closes the slots.
static void slots_close_all(dfb_stream *h) {
    holds_lift_all(h);
    for (int b = 0; b < h->B; b++) slot_close(h, b);
    slots_retire(h, h->S.a1 - path_latency(h));
    h->slot_ops = true;
}

// Valid slot indices, each listed once; a live group of more than one channel is listed with all of its members or not at
// all (groups open, close and take settings as a unit).
static int slot_list_check(const dfb_stream *h, const int64_t *slots, int64_t n) {
    if (!h || n < 0 || (n > 0 && !slots)) return fail(DFB_ERR_INVALID, "bad argument");
    if (h->fixed_nch > 1) return fail(DFB_ERR_UNSUPPORTED, "slot operations on a handle with linked channels");
    std::vector<int> seen((size_t)h->B, 0);
    for (int64_t i = 0; i < n; i++) {
        const int64_t b = slots[i];
        if (b < 0 || b >= h->B) return fail(DFB_ERR_INVALID, "slot %lld outside [0, %d)", (long long)b, h->B);
        if (seen[(size_t)b]) return fail(DFB_ERR_INVALID, "slot %lld listed twice", (long long)b);
        seen[(size_t)b] = 1;
    }
    std::vector<int> listed((size_t)h->B, 0);   // per group (by its channel-0 slot): members listed
    for (int64_t i = 0; i < n; i++)
        if (h->slot_grp[(size_t)slots[i]] >= 0) listed[(size_t)h->slot_grp[(size_t)slots[i]]]++;
    for (int64_t i = 0; i < n; i++) {
        const int f = h->slot_grp[(size_t)slots[i]];
        if (f >= 0 && listed[(size_t)f] != h->slot_nch[(size_t)f])
            return fail(DFB_ERR_INVALID, "slot %lld belongs to a group of %d channels (slot %d is channel 0): list all of them",
                        (long long)slots[i], h->slot_nch[(size_t)f], f);
    }
    return DFB_OK;
}

static int slot_list(dfb_stream *h, const int64_t *slots, int64_t n) {
    if (int rc = slot_list_check(h, slots, n)) return rc;
    h->slot_ops = true;
    return DFB_OK;
}

// Opens one group per `nch` consecutive listed slots (channel c of a group in its c-th slot), each a fresh stream in rows
// of the active prefix.  The listed slots' old streams (whole groups, by slot_list_check) are dropped without
// their tails first.  dir: the sessions' direction of the resamplers (0: the handle's rate, 48 kHz on a mixed-rate handle).
static int slots_open(dfb_stream *h, const int64_t *slots, int64_t n, int64_t nch, int dir = 0) {
    if (int rc = slot_list(h, slots, n)) return rc;
    for (int64_t i = 0; i < n; i++)
        if (h->slot_state[(size_t)slots[i]] != kSlotFree) slot_release(h, (int)slots[i]);
    rows_layout(h);
    for (int64_t i = 0; i < n; i++) {
        const int b = (int)slots[i], r = h->n_live++;
        h->slot_row[(size_t)b] = r;
        h->row_slot[(size_t)r] = b;
        h->row_src[(size_t)r] = -1;
        h->slot_grp[(size_t)b] = (int)slots[i - i % nch];
        h->slot_nch[(size_t)b] = (int)nch;
        h->slot_state[(size_t)b] = kSlotOpen;
        h->slot_first[(size_t)b] = h->S.a1;
        h->slot_end[(size_t)b] = kOpenEnd;
        h->slot_dir[(size_t)b] = dir;
        h->slot_lim[(size_t)b] = h->slot_beta[(size_t)b] = NAN;   // back to the handle's settings
        h->slot_gate[(size_t)b] = -1;
        h->slot_fresh[(size_t)b] = 1;
        h->slot_rt[(size_t)b] = h->S.rt_valid;
        h->slot_held_frames[(size_t)b] = 0;
    }
    rows_layout(h);
    h->tab_dirty = true;
    return DFB_OK;
}

extern "C" int dfb_stream_open_slots(dfb_stream *h, const int64_t *slots, int64_t n) { return slots_open(h, slots, n, 1); }

extern "C" int dfb_stream_open_linked(dfb_stream *h, const int64_t *slots, int64_t n) {
    if (h && n == 0) return fail(DFB_ERR_INVALID, "a group of no channels");
    return slots_open(h, slots, n, n);
}

// the rates a streaming handle resamples to and from 48 kHz (dfb_stream_set_sample_rate / dfb_stream_add_slot_rate)
static bool stream_rate(int rate) {
    return rate == 8000 || rate == 12000 || rate == 16000 || rate == 24000 || rate == 32000 || rate == 44100;
}

// the direction of a mixed-rate handle's sessions at `rate`
static int rate_dir(const dfb_stream *h, int rate, int *dir) {
    if (rate != kModelRate && !stream_rate(rate))
        return fail(DFB_ERR_UNSUPPORTED, "sample rate %d: 8000, 12000, 16000, 24000, 32000, 44100 or 48000", rate);
    if (!mixed_rate(h)) return fail(DFB_ERR_INVALID, "slots open at their own rates on a handle with slot rates only (dfb_stream_add_slot_rate)");
    for (size_t i = 0; i < h->rs_rates.size(); i++)
        if (h->rs_rates[i] == rate) {
            *dir = (int)i;
            return DFB_OK;
        }
    return fail(DFB_ERR_INVALID, "sample rate %d is not registered on this handle (dfb_stream_add_slot_rate)", rate);
}

extern "C" int dfb_stream_open_slots_at(dfb_stream *h, const int64_t *slots, int64_t n, int rate) {
    int dir = 0;
    if (!h) return fail(DFB_ERR_INVALID, "null stream");
    if (int rc = rate_dir(h, rate, &dir)) return rc;
    return slots_open(h, slots, n, 1, dir);
}

extern "C" int dfb_stream_open_linked_at(dfb_stream *h, const int64_t *slots, int64_t n, int rate) {
    int dir = 0;
    if (!h) return fail(DFB_ERR_INVALID, "null stream");
    if (n == 0) return fail(DFB_ERR_INVALID, "a group of no channels");
    if (int rc = rate_dir(h, rate, &dir)) return rc;
    return slots_open(h, slots, n, n, dir);
}

extern "C" int dfb_stream_close_slots(dfb_stream *h, const int64_t *slots, int64_t n) {
    if (int rc = slot_list(h, slots, n)) return rc;
    for (int64_t i = 0; i < n; i++) slot_close(h, (int)slots[i]);
    slots_retire(h, h->S.a1 - path_latency(h));   // without look-ahead (latency 0) a closed slot is free at once
    return DFB_OK;
}

// ---- held sessions (DESIGN.md section 5p).  A held session sits in a live row behind the active prefix, which no call
// computes or writes; after every call its bookkeeping moves forward by the frames the clock advanced (holds_rebase), so
// that, relative to the clock, its state is what its last advancing call left.
extern "C" int dfb_stream_hold_slots(dfb_stream *h, const int64_t *slots, int64_t n, int hold) {
    if (int rc = slot_list_check(h, slots, n)) return rc;
    for (int64_t i = 0; i < n; i++)
        if (h->slot_state[(size_t)slots[i]] == kSlotFree) return fail(DFB_ERR_INVALID, "slot %lld is free", (long long)slots[i]);
    h->slot_ops = true;
    for (int64_t i = 0; i < n; i++) {
        const size_t b = (size_t)slots[i];
        h->slot_held[b] = hold ? 1 : 0;
        // before a handle's first frame its rows start from a state the first call implies (S.started): a row that sits
        // that call out gets it written instead, as a freshly opened row
        if (hold && !h->S.started) h->row_src[(size_t)h->slot_row[b]] = -1;
    }
    rows_layout(h);
    return DFB_OK;
}

extern "C" int dfb_stream_held_slots(const dfb_stream *h, int8_t *h_held) {
    if (!h || !h_held) return fail(DFB_ERR_INVALID, "null argument");
    for (int b = 0; b < h->B; b++) h_held[b] = h->slot_held[(size_t)b] ? 1 : 0;
    return DFB_OK;
}

// every hold lifted (a flush ends every session, held ones included)
static void holds_lift_all(dfb_stream *h) {
    if (h->n_live == h->n_act) return;
    std::fill(h->slot_held.begin(), h->slot_held.end(), (char)0);
    rows_layout(h);
}

// after a call that moved the clock d frames on: the held sessions' first frame, end frame and settings switch with it
static void holds_rebase(dfb_stream *h, int64_t d) {
    if (d == 0 || h->n_live == h->n_act) return;
    for (int r = h->n_act; r < h->n_live; r++) {
        const size_t b = (size_t)h->row_slot[(size_t)r];
        h->slot_first[b] += d;
        h->slot_held_frames[b] += d;
        if (h->slot_state[b] == kSlotClosing) h->slot_end[b] += d;
        h->slot_ctl[b].sw += d;
    }
}

// ---- per-slot settings.  A setting is stored per slot; each call resolves every live slot's setting (its own, or the
// handle's default at that call) and, when it differs from the one of the slot's last call, switches at the call's first
// output frame f0: frame f0 - 1, which the apply kernel re-synthesises for its overlap-add tail, keeps the previous one.
// The checks every per-slot setter makes before the value's own: a spectral handle, the slot list, the model shape.
static int ctl_check(const dfb_stream *h, const int64_t *slots, int64_t n) {
    if (h && h->spectral)
        return fail(DFB_ERR_UNSUPPORTED, "per-slot settings are apply-stage settings: a spectral handle applies nothing");
    if (int rc = slot_list_check(h, slots, n)) return rc;
    const dfb_model_config &c = h->m->cfg;
    if (c.df_order != 5 || c.nb_df != 96 || c.nb_erb != 32)
        return fail(DFB_ERR_UNSUPPORTED, "per-slot settings are built for df_order 5, nb_df 96 and 32 ERB bands");
    return DFB_OK;
}

// The per-row settings table from now on (the device table allocated once).
static int ctl_enable(dfb_stream *h) {
    if (h->ctl_on) return DFB_OK;
    if (!h->d_ctl) {
        DFB_CUDA(cudaSetDevice(h->m->device));
        if (cudaMalloc(&h->d_ctl, sizeof(SlotCtl) * (size_t)h->B) != cudaSuccess) {
            h->d_ctl = nullptr;
            return fail(DFB_ERR_OOM, "slot settings allocation failed");
        }
    }
    // every slot has run with the handle's settings so far
    for (int b = 0; b < h->B; b++) h->slot_ctl[(size_t)b] = SlotCtl{h->lim, h->beta_run, h->lim, h->beta_run, 0};
    std::fill(h->slot_fresh.begin(), h->slot_fresh.end(), (char)0);
    h->ctl_up.clear();
    h->ctl_on = true;
    return DFB_OK;
}

// After the value's checks: naming a free slot is refused; otherwise the per-row table is on from now on.
static int ctl_begin(dfb_stream *h, const int64_t *slots, int64_t n) {
    for (int64_t i = 0; i < n; i++)
        if (h->slot_state[(size_t)slots[i]] == kSlotFree) return fail(DFB_ERR_INVALID, "slot %lld is free", (long long)slots[i]);
    if (n == 0) return DFB_OK;
    h->slot_ops = true;
    return ctl_enable(h);
}

static int ctl_set(dfb_stream *h, const int64_t *slots, int64_t n, bool beta, float v) {
    if (int rc = ctl_check(h, slots, n)) return rc;
    if (beta && h->m->cfg.model_kind != 3)
        return fail(DFB_ERR_UNSUPPORTED, "per-slot post-filter beta: DeepFilterNet3 topologies only (DeepFilterNet2's beta is fixed)");
    if (std::isnan(v) || (beta && !(v >= 0.f && std::isfinite(v))))
        return fail(DFB_ERR_INVALID, beta ? "post-filter beta must be finite and >= 0" : "attenuation limit is NaN");
    if (int rc = ctl_begin(h, slots, n)) return rc;
    std::vector<float> &dst = beta ? h->slot_beta : h->slot_lim;
    for (int64_t i = 0; i < n; i++) dst[(size_t)slots[i]] = v;
    return DFB_OK;
}

// Per-slot LSNR stage gating (the LADSPA plugin's per-instance thresholds): the listed slots gate with their own thresholds,
// or not at all (enable == 0), from the next call on, every frame of that call included.
extern "C" int dfb_stream_set_lsnr_thresholds_slots(dfb_stream *h, const int64_t *slots, int64_t n, int enable, float min_db_thresh,
                                                    float max_db_erb_thresh, float max_db_df_thresh) {
    if (int rc = ctl_check(h, slots, n)) return rc;
    if (enable && h->m->cfg.model_kind != 3) return fail(DFB_ERR_UNSUPPORTED, "LSNR stage gating: DeepFilterNet3 topologies only");
    if (enable && (std::isnan(min_db_thresh) || std::isnan(max_db_erb_thresh) || std::isnan(max_db_df_thresh)))
        return fail(DFB_ERR_INVALID, "an LSNR threshold is NaN");
    if (int rc = ctl_begin(h, slots, n)) return rc;
    for (int64_t i = 0; i < n; i++) {
        const size_t b = (size_t)slots[i];
        h->slot_gate[b] = enable ? 1 : 0;
        h->slot_th[3 * b] = min_db_thresh; h->slot_th[3 * b + 1] = max_db_erb_thresh; h->slot_th[3 * b + 2] = max_db_df_thresh;
    }
    return DFB_OK;
}

extern "C" int dfb_stream_set_atten_lim(dfb_stream *h, const int64_t *slots, int64_t n, float atten_lim_db) {
    const float lim = std::isnan(atten_lim_db) ? NAN : (atten_lim_db > 0.f ? powf(10.f, -atten_lim_db / 20.f) : 0.f);
    return ctl_set(h, slots, n, false, lim);
}

extern "C" int dfb_stream_set_post_filter_beta(dfb_stream *h, const int64_t *slots, int64_t n, float beta) {
    return ctl_set(h, slots, n, true, beta);
}

// the per-row settings of a call whose first output hop carries frame f0; uploaded when they differ from the last upload
static int ctl_rows(dfb_stream *h, int64_t f0, cudaStream_t s) {
    const float beta_def = default_beta(h->m);
    std::vector<SlotCtl> rows((size_t)h->n_act);
    h->ctl_gate = false;
    for (int r = 0; r < h->n_act; r++) {
        const size_t b = (size_t)h->row_slot[(size_t)r];
        const float lim = std::isnan(h->slot_lim[b]) ? h->lim : h->slot_lim[b];
        const float beta = std::isnan(h->slot_beta[b]) ? beta_def : h->slot_beta[b];
        SlotCtl &c = h->slot_ctl[b];
        if (h->slot_fresh[b]) { c = SlotCtl{lim, beta, lim, beta, f0}; h->slot_fresh[b] = 0; }
        else if (lim != c.lim || beta != c.beta) c = SlotCtl{lim, beta, c.lim, c.beta, f0};
        // gating: the slot's own, or the handle's (dfb_stream_set_lsnr_thresholds)
        const bool own = h->slot_gate[b] >= 0;
        const float *th = own ? &h->slot_th[3 * b] : h->th;
        c.gate = own ? h->slot_gate[b] : (h->gating ? 1 : 0);
        c.th_min = th[0]; c.th_erb = th[1]; c.th_df = th[2];
        h->ctl_gate |= c.gate != 0;
        rows[(size_t)r] = c;
    }
    if (rows.size() != h->ctl_up.size() || memcmp(rows.data(), h->ctl_up.data(), sizeof(SlotCtl) * rows.size())) {
        if (!rows.empty())
            DFB_CUDA(cudaMemcpyAsync(h->d_ctl, rows.data(), sizeof(SlotCtl) * rows.size(), cudaMemcpyHostToDevice, s));
        h->ctl_up.swap(rows);
    }
    return DFB_OK;
}

extern "C" int dfb_stream_slot_states(const dfb_stream *h, int32_t *h_states) {
    if (!h || !h_states) return fail(DFB_ERR_INVALID, "null argument");
    for (int b = 0; b < h->B; b++) h_states[b] = h->slot_state[(size_t)b];
    return DFB_OK;
}

extern "C" int dfb_stream_slot_rates(const dfb_stream *h, int32_t *h_rates) {
    if (!h || !h_rates) return fail(DFB_ERR_INVALID, "null argument");
    if (h->spectral) return fail(DFB_ERR_INVALID, "a spectral handle takes spectra, which have no sample rate");
    for (int b = 0; b < h->B; b++)
        h_rates[b] = h->slot_state[(size_t)b] == kSlotFree ? 0
                     : resampled(h)                         ? h->rs_rates[(size_t)h->slot_dir[(size_t)b]]
                                                            : kModelRate;
    return DFB_OK;
}

extern "C" int dfb_stream_slot_groups(const dfb_stream *h, int64_t *h_first) {
    if (!h || !h_first) return fail(DFB_ERR_INVALID, "null argument");
    for (int b = 0; b < h->B; b++) h_first[b] = h->slot_grp[(size_t)b];
    return DFB_OK;
}

// Row moves of a call: live row r (held rows included) takes its state from row_src[r] as the last call left it, or starts
// fresh (-1).  Two launches of k_slot_rows whatever the number of rows, the scratch rows in the model arena (the chunk
// that follows reuses it in stream order).
static int slots_move_rows(dfb_stream *h, cudaStream_t s) {
    std::vector<int2> ops;
    int n_mv = 0;
    for (int pass = 0; pass < 2; pass++)   // the moves first, then the fresh rows
        for (int r = 0; r < h->n_live; r++) {
            const int src = h->row_src[(size_t)r];
            if (src != r && (src >= 0) == (pass == 0)) ops.push_back(make_int2(r, src));
        }
    for (const int2 &op : ops) n_mv += op.y >= 0;
    for (int r = 0; r < h->n_live; r++) h->row_src[(size_t)r] = r;
    h->rows_moved = (int64_t)ops.size();
    if (ops.empty()) return DFB_OK;
    dfb_model *m = h->m;
    size_t off[kStateArrays];
    StateLayout lay;
    stream_state_floats(h, off, &lay);
    if (int rc = m->arena.reserve(sizeof(int2) * ops.size() + sizeof(float) * (size_t)lay.row_floats * n_mv + 1024)) return rc;
    m->arena.reset();
    int2 *d_ops = m->arena.take<int2>(ops.size());
    float *scratch = m->arena.take<float>((size_t)lay.row_floats * n_mv + 1);
    DFB_CUDA(cudaMemcpyAsync(d_ops, ops.data(), sizeof(int2) * ops.size(), cudaMemcpyHostToDevice, s));
    for (int pass = n_mv ? 0 : 1; pass < 2; pass++) {
        k_slot_rows<<<dim3(4, pass ? (unsigned)ops.size() : (unsigned)n_mv, resampled(h) ? kStateArrays : kStateArrays - 2), 256, 0, s>>>(
            h->slab, lay, h->B, d_ops, scratch, pass, m->cfg.nb_erb, m->cfg.nb_df);
        DFB_LAUNCH_CHECK();
    }
    m->arena.reset();
    return DFB_OK;
}

// The spectral side of a call's ChunkIO: input frames [B][n][F] where the row table says, outputs to `so` with n_out rows
// per caller row from frame f0 on, the LSNR head always on
static void spec_io(const dfb_stream *h, ChunkIO &io, SpecOut *so, const float *d_in, int64_t n, int64_t n_out, int64_t f0) {
    so->Bc = h->B; so->n_out = n_out; so->f0 = f0; so->slot_row = h->d_slotmap;
    so->gating = h->gating; so->th[0] = h->th[0]; so->th[1] = h->th[1]; so->th[2] = h->th[2];
    so->mask_only = h->m->mask_only;
    io.spec_in = d_in; io.spec_frames = n; io.spec_out = so;
    io.lsnr_from = 0; io.lsnr_out = nullptr;
}
// a spectral call with no live row: every output row carries no frame (NaN, stage -1)
static int spec_fill_empty(const SpecOut &so, const dfb_model_config &c, int64_t rows, cudaStream_t s) {
    DFB_CUDA(cudaMemsetAsync(so.gains, 0xff, sizeof(float) * rows * c.nb_erb, s));
    if (so.coefs) DFB_CUDA(cudaMemsetAsync(so.coefs, 0xff, sizeof(float) * rows * c.nb_df * 2 * c.df_order, s));
    if (so.lsnr) DFB_CUDA(cudaMemsetAsync(so.lsnr, 0xff, sizeof(float) * rows, s));
    if (so.stage) DFB_CUDA(cudaMemsetAsync(so.stage, 0xff, rows, s));
    return DFB_OK;
}

// The slot tables of a call of n input hops: closes every open slot first on a flush, moves the state-slab rows of slots
// that opened or closed up (slots_move_rows) and uploads the row tables when they changed.
static int stream_tables(dfb_stream *h, int64_t n, bool flush, bool spec, cudaStream_t s) {
    const int hop = h->st->hop, B = h->B;
    const int64_t n_out = flush ? path_latency(h) : n, a0 = h->S.a1;
    if (flush) slots_close_all(h);
    if (int rc = slots_move_rows(h, s)) return rc;
    if (h->tab_dirty || h->tab_n != n) {
        std::vector<RaggedRow> rows((size_t)h->n_act);
        std::vector<int64_t> first((size_t)h->n_act);
        std::vector<LinkRow> grp((size_t)h->n_act);
        bool linked = false;   // the link table goes to the kernels only while a group of more than one channel is linked
        bool pending = false;  // a closing row reads input in this call
        const int64_t unit = spec ? kSpecF : hop, per = spec ? 1 : hop;   // input offsets in complex values / samples, lengths in frames / samples
        for (int r = 0; r < h->n_act; r++) {
            const int b = h->row_slot[(size_t)r];
            const bool open = h->slot_state[(size_t)b] == kSlotOpen;
            // a closing row reads no input, but for the hops before its end frame (a resampled session's last hop)
            const int64_t tail = std::min(n, std::max<int64_t>(0, h->slot_end[(size_t)b] - a0));
            rows[(size_t)r] = RaggedRow{b * n * unit, (open ? n : tail) * per, b * n_out * hop, n_out * hop, h->slot_end[(size_t)b]};
            pending |= !open && tail > 0;
            first[(size_t)r] = h->slot_first[(size_t)b];
            grp[(size_t)r] = LinkRow{h->slot_row[(size_t)h->slot_grp[(size_t)b]], h->slot_nch[(size_t)b]};
            linked |= grp[(size_t)r].n > 1 && h->group_reduce != kReduceNone;
        }
        if (h->n_act > 0) {
            DFB_CUDA(cudaMemcpyAsync(h->d_rows, rows.data(), sizeof(RaggedRow) * rows.size(), cudaMemcpyHostToDevice, s));
            DFB_CUDA(cudaMemcpyAsync(h->d_first, first.data(), sizeof(int64_t) * first.size(), cudaMemcpyHostToDevice, s));
            if (linked) DFB_CUDA(cudaMemcpyAsync(h->d_grp, grp.data(), sizeof(LinkRow) * grp.size(), cudaMemcpyHostToDevice, s));
        }
        if (spec) {   // k_spec_emit covers every caller row: free slots get NaN / -1
            if (!h->d_slotmap && cudaMalloc(&h->d_slotmap, sizeof(int) * (size_t)B) != cudaSuccess) {
                h->d_slotmap = nullptr;
                return fail(DFB_ERR_OOM, "slot table allocation failed");
            }
            std::vector<int> map(h->slot_row);   // held rows carry no frame
            for (int &r : map) r = r < h->n_act ? r : -1;
            DFB_CUDA(cudaMemcpyAsync(h->d_slotmap, map.data(), sizeof(int) * (size_t)B, cudaMemcpyHostToDevice, s));
        }
        h->tab_dirty = pending;   // such a row reads nothing from the next call on
        h->tab_n = n;
        h->tab_linked = linked;
    }
    return DFB_OK;
}

// One call: rows [0, n_act) of the slab, the row table for calls of n input hops.
// Spectral handle (so != null): d_in is [B][n][F] complex, the outputs go to so's buffers, d_out / d_lsnr are null.
static int stream_step(dfb_stream *h, const float *d_in, int64_t n, bool flush, float *d_out, float *d_lsnr, cudaStream_t s,
                       SpecOut *so = nullptr) {
    if (d_lsnr && h->lsnr_from < 0) {   // from now on every call runs the LSNR head
        h->lsnr_from = h->S.d1;
        // a session's LSNR start is relative to its frames as of now: only the frames it is held from here on shift it
        std::fill(h->slot_held_frames.begin(), h->slot_held_frames.end(), (int64_t)0);
    }
    dfb_model *m = h->m;
    dfb_state *st = h->st;
    StreamState &S = h->S;
    const ChunkGeom g = chunk_geom(m->cfg);
    const int hop = st->hop, B = h->B;
    const int64_t Ltot = path_latency(h), n_out = flush ? Ltot : n;
    const int64_t lag = so ? 0 : g.lag, la = Ltot - lag;   // feature look-ahead of the DNN frames; their outputs' further lag
    const int64_t a0 = S.a1, a1n = a0 + (flush ? 0 : n);
    if (a1n >= kOpenEnd - 1) return fail(DFB_ERR_UNSUPPORTED, "stream clock beyond 2^31 - 2 frames: reset the stream");
    int rc = DFB_OK;
    int64_t d1n = flush ? a1n : a1n - la, e1n = flush ? a1n : d1n - lag;
    if (d1n < S.d1) d1n = S.d1;
    if (e1n < S.e1) e1n = S.e1;
    if ((rc = stream_tables(h, n, flush, so != nullptr, s))) return rc;
    const int64_t f0 = a0 - Ltot;   // output hop j carries frame a0 - Ltot + j (flush: a1 = a0)
    // The apply kernel writes every hop that carries a frame of its row.  The others are zero: those of free slots, of
    // frames before 0, before a row's first frame or from a closing row's end on, and all of them when no frame is emitted.
    bool gaps = h->n_act < B || f0 < 0 || e1n <= S.e1;
    for (int r = 0; r < h->n_act && !gaps; r++) {
        const size_t b = (size_t)h->row_slot[(size_t)r];
        gaps = h->slot_first[b] > f0 || h->slot_end[b] < f0 + n_out;
    }
    if (gaps && n_out > 0 && !so) DFB_CUDA(cudaMemsetAsync(d_out, 0, sizeof(float) * B * n_out * hop, s));
    if (d_lsnr && n_out > 0) DFB_CUDA(cudaMemsetAsync(d_lsnr, 0xff, sizeof(float) * B * n_out, s));   // NaN: hops without a frame
    if (h->ctl_on && (rc = ctl_rows(h, f0, s))) return rc;
    h->beta_run = default_beta(m);
    h->fed = true;
    if (h->n_act == 0) {   // nothing to compute: the clock moves on (a slot opened later starts from zeroed tails)
        if (so && n_out > 0 && (rc = spec_fill_empty(*so, m->cfg, B * n_out, s))) return rc;
        S.a1 = a1n; S.d1 = d1n; S.e1 = e1n;
        if (a1n > 0) S.started = true;
        if (d1n > 0) S.dnn_started = true;
        S.n_feat = g.Hf; S.n_mc = kMcTail; S.n_dec = kHalo;
        holds_rebase(h, a1n - a0);
        slots_retire(h, flush ? a1n : a1n - Ltot);
        return DFB_OK;
    }
    ChunkIO io{so ? nullptr : d_in, n * hop, a0, nullptr, d_out, n_out * hop, n_out * hop, f0 * hop, h->lim,
               h->gating && !so ? h->th : nullptr, h->d_rows, h->n_act};
    io.first = h->d_first;
    if (so) spec_io(h, io, so, d_in, n, n_out, f0);
    if (h->tab_linked) { io.links = h->d_grp; io.reduce = h->group_reduce; }
    if (h->ctl_on) { io.ctl = h->d_ctl; io.ctl_gate = h->ctl_gate; }
    io.lsnr_from = h->lsnr_from;
    io.lsnr_out = d_lsnr;
    io.runtime = (h->gating_mode >= 0 ? h->gating_mode : m->gating_mode) == DFB_GATING_RUNTIME;
    // a row whose own tails' validity differs from the last DNN call's (a session held since another mode's call) switches
    // alone: per-row halo flags
    if (io.runtime) {
        std::vector<unsigned char> halo((size_t)h->n_act);
        bool mixed = false;
        for (int r = 0; r < h->n_act; r++) {
            const bool v = h->slot_rt[(size_t)h->row_slot[(size_t)r]] != 0;
            halo[(size_t)r] = v ? 0 : 1;
            mixed |= v != S.rt_valid;
        }
        if (mixed) {
            if (!h->d_halo && cudaMalloc(&h->d_halo, (size_t)B) != cudaSuccess) {
                h->d_halo = nullptr;
                return fail(DFB_ERR_OOM, "gating table allocation failed");
            }
            DFB_CUDA(cudaMemcpyAsync(h->d_halo, halo.data(), halo.size(), cudaMemcpyHostToDevice, s));
            io.rt_halo = h->d_halo;
        }
    }
    rc = m->arena.reserve(chunk_bytes_per_stream(m->cfg, st, (int)(d1n - (S.d1 > kHalo ? S.d1 - kHalo : 0)) + 1) * (size_t)h->n_act +
                              (2 << 20));
    if (rc) return rc;
    if (!flush && a1n > a0 && !so) {
        if (!S.started) DFB_CUDA(cudaMemsetAsync(S.ana_mem, 0, sizeof(float) * h->n_act * hop, s));
        io.init_mem = S.ana_mem;
    }
    const int64_t d1_was = S.d1;
    if ((rc = run_chunk(m, st, S, io, a1n, d1n, e1n, s))) return rc;
    if (!flush && !so) {
        k_carry_hop<<<h->n_act, 128, 0, s>>>(S.ana_mem, d_in, h->d_rows, (n - 1) * hop, hop);
        DFB_LAUNCH_CHECK();
    }
    m->arena.reset();
    if (S.d1 > d1_was)   // a DNN chunk ran: the advancing rows' tails are as it left them
        for (int r = 0; r < h->n_act; r++) h->slot_rt[(size_t)h->row_slot[(size_t)r]] = S.rt_valid;
    holds_rebase(h, a1n - a0);
    slots_retire(h, flush ? a1n : a1n - Ltot);
    return DFB_OK;
}

// ---- handles at another sample rate (dfb_stream_set_sample_rate; DESIGN.md section 5g) and mixed-rate handles
// (dfb_stream_add_slot_rate; section 5h).  Each call runs the unchanged 48 kHz slot path between two resamplers:
// k_resample_up turns the call's input into the 48 kHz hops the path reads, k_resample_down turns the path's output back
// into the caller's hops, each row in its session's direction.  Their histories are rows of the state slab, so they move
// with the rows and start from zero with every session.

// the per-direction geometry of `rate` from io.resample_kernel's (og, nw, width); DFB_ERR_UNSUPPORTED for a rate outside
// the list, DFB_ERR_INVALID for taps of other rates or a history longer than a hop
static int rs_geometry(int rate, bool up, const float *taps, int og, int nw, int width, ResampleDir *d) {
    if (!stream_rate(rate))
        return fail(DFB_ERR_UNSUPPORTED, "sample rate %d: 8000, 12000, 16000, 24000, 32000, 44100 or 48000", rate);
    const int g = std::gcd(rate, kModelRate), from = up ? rate : kModelRate, to = up ? kModelRate : rate;
    if (!taps || og != from / g || nw != to / g || width <= 0 || width > 4096)
        return fail(DFB_ERR_INVALID, "the %s taps of %d Hz are io.resample_kernel(%d, %d): og %d, nw %d", up ? "up" : "down", rate,
                    from, to, from / g, to / g);
    const int mz = (width + og - 1) / og;
    *d = ResampleDir{taps, og, nw, 2 * width + og, mz * og + width, mz * nw, from / 100, to / 100, 1};
    if (d->S > d->hop_in) return fail(DFB_ERR_INVALID, "resampler history of %d samples is longer than a hop", d->S);
    return DFB_OK;
}

// Both directions of `rate` from the caller's taps, uploaded: *buf holds them on the device (the caller owns it).
static int rs_directions(int rate, const float *up_taps, int up_og, int up_nw, int up_width, const float *down_taps, int down_og,
                         int down_nw, int down_width, ResampleDir *up, ResampleDir *down, float **buf) {
    int rc;
    if ((rc = rs_geometry(rate, true, up_taps, up_og, up_nw, up_width, up)) ||
        (rc = rs_geometry(rate, false, down_taps, down_og, down_nw, down_width, down)))
        return rc;
    const size_t nu = (size_t)up->nw * up->K, nd = (size_t)down->nw * down->K;
    float *taps = nullptr;
    if (cudaMalloc(&taps, sizeof(float) * (nu + nd)) != cudaSuccess) return fail(DFB_ERR_OOM, "resampler taps allocation failed");
    if (cudaMemcpy(taps, up_taps, sizeof(float) * nu, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(taps + nu, down_taps, sizeof(float) * nd, cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaFree(taps);
        return fail(DFB_ERR_CUDA, "resampler taps upload failed");
    }
    up->taps = taps; down->taps = taps + nu;
    *buf = taps;
    return DFB_OK;
}

static int stage_grow(float **p, size_t *cap, size_t bytes);

// the live rows' table of the resamplers, uploaded when it changed
static int rs_table(dfb_stream *h, cudaStream_t s) {
    std::vector<ResampleRow> rows((size_t)h->n_act);
    for (int r = 0; r < h->n_act; r++) {
        const size_t b = (size_t)h->row_slot[(size_t)r];
        rows[(size_t)r] = ResampleRow{(int64_t)b, h->slot_first[b], h->slot_end[b], h->slot_dir[b]};
    }
    if (rows.size() != h->rs_rows.size() || memcmp(rows.data(), h->rs_rows.data(), sizeof(ResampleRow) * rows.size())) {
        if (!rows.empty())
            DFB_CUDA(cudaMemcpyAsync(h->d_rs, rows.data(), sizeof(ResampleRow) * rows.size(), cudaMemcpyHostToDevice, s));
        h->rs_rows.swap(rows);
    }
    return DFB_OK;
}

// One pass through the slot path: n hops of input (d_in null: none, the sessions' zero extension), or its flush; the
// output hops go to d_out [B][pitch] from hop `col` of each row on, in the row's own samples, and its LSNR to d_lsnr
// [B][n_out].  Input rows are [B][n * frame_length]: a row reads the first n hops at its own rate.
static int rate_pass(dfb_stream *h, const float *d_in, int64_t n, bool flush, float *d_out, int64_t pitch, int64_t col,
                     float *d_lsnr, cudaStream_t s) {
    const int64_t L = path_latency(h), n_out = flush ? L : n, hop = h->st->hop, wide = dfb_stream_frame_length(h), B = h->B,
                  a0 = h->S.a1;
    int rc;
    if ((rc = stream_tables(h, n, flush, false, s)) || (rc = rs_table(h, s))) return rc;
    if ((!flush && (rc = stage_grow(&h->rs_in, &h->rs_in_cap, sizeof(float) * B * n * hop))) ||
        (rc = stage_grow(&h->rs_out, &h->rs_out_cap, sizeof(float) * B * std::max<int64_t>(n_out, 1) * hop)))
        return rc;
    const int nb = h->n_act, nd = (int)h->rs_rates.size();
    // Free rows are zeroed over their whole width by a call's first pass.  A row live in it fills its own row past its
    // samples with zeros, and only such rows turn free before the call's next pass.
    if (nb < B && n_out > 0 && col == 0) DFB_CUDA(cudaMemset2DAsync(d_out, sizeof(float) * pitch, 0, sizeof(float) * pitch, B, s));
    size_t off[kStateArrays];
    stream_state_floats(h, off);
    const ResampleIO up{d_in, h->rs_in, h->slab + off[15], n * wide, n * hop, n * hop, rs_hist(h, h->rs_up), 0, 0, n, a0, 0};
    if (!flush && (rc = launch_resample_stream(s, true, h->rs_up, nd, h->d_rs, nb, up))) return rc;
    if ((rc = stream_step(h, flush ? nullptr : h->rs_in, n, flush, h->rs_out, d_lsnr, s))) return rc;
    const ResampleIO down{h->rs_out, d_out, h->slab + off[16], n_out * hop, pitch, pitch, rs_hist(h, h->rs_down), 0, col, n_out, a0, L};
    return launch_resample_stream(s, false, h->rs_down, nd, h->d_rs, nb, down);
}

// A call of a resampled or mixed-rate handle.  A flush ends every open session (a resampled session's input one hop
// before its end frame), runs that hop of zero extension through the slot path and then flushes it: L + 1 output hops.
static int rate_step(dfb_stream *h, const float *d_in, int64_t n, bool flush, float *d_out, float *d_lsnr, cudaStream_t s) {
    const int64_t wide = dfb_stream_frame_length(h), B = h->B;
    if (!flush) return rate_pass(h, d_in, n, false, d_out, n * wide, 0, d_lsnr, s);
    const int64_t L = path_latency(h), w = L + 1;
    holds_lift_all(h);
    for (int b = 0; b < h->B; b++) slot_close(h, b);
    h->slot_ops = true;
    int rc;
    float *l1 = nullptr, *l2 = nullptr;
    if (d_lsnr) {
        if ((rc = stage_grow(&h->rs_lsnr, &h->rs_lsnr_cap, sizeof(float) * B * w))) return rc;
        l1 = h->rs_lsnr; l2 = l1 + B;
    }
    if ((rc = rate_pass(h, nullptr, 1, false, d_out, w * wide, 0, l1, s))) return rc;
    if (L > 0 && (rc = rate_pass(h, nullptr, 0, true, d_out, w * wide, 1, l2, s))) return rc;
    if (d_lsnr) {
        DFB_CUDA(cudaMemcpy2DAsync(d_lsnr, sizeof(float) * w, l1, sizeof(float), sizeof(float), B, cudaMemcpyDeviceToDevice, s));
        if (L > 0)
            DFB_CUDA(cudaMemcpy2DAsync(d_lsnr + 1, sizeof(float) * w, l2, sizeof(float) * L, sizeof(float) * L, B, cudaMemcpyDeviceToDevice, s));
    }
    return DFB_OK;
}

// the calls of an audio handle, at 48 kHz or resampled
static int audio_step(dfb_stream *h, const float *d_in, int64_t n, bool flush, float *d_out, float *d_lsnr, cudaStream_t s) {
    return resampled(h) ? rate_step(h, d_in, n, flush, d_out, d_lsnr, s) : stream_step(h, d_in, n, flush, d_out, d_lsnr, s);
}

// (Re)allocates the state slab of a new or reset handle for its current directions, zeroed.
static int stream_slab(dfb_stream *h) {
    size_t off[kStateArrays];
    const size_t n = stream_state_floats(h, off);
    float *p = nullptr;
    if (cudaMalloc(&p, n * sizeof(float)) != cudaSuccess) return fail(DFB_ERR_OOM, "stream state allocation failed");
    if (h->slab) cudaFree(h->slab);
    h->slab = p;
    DFB_CUDA(cudaMemset(h->slab, 0, n * sizeof(float)));
    state_bind(h->S, h->slab, off, h->B);
    return DFB_OK;
}

// The rules both rate setters share: an audio handle, new or reset, before its first frame and any slot operation.
static int rate_setter(dfb_stream *h) {
    if (!h) return fail(DFB_ERR_INVALID, "null stream");
    if (h->spectral) return fail(DFB_ERR_INVALID, "a spectral handle takes spectra, which have no sample rate");
    if (h->fed || h->slot_ops)
        return fail(DFB_ERR_INVALID, "sample rate set after the first frame or a slot operation: reset the stream first");
    DFB_CUDA(cudaSetDevice(h->m->device));
    if (!h->d_rs && cudaMalloc(&h->d_rs, sizeof(ResampleRow) * (size_t)h->B) != cudaSuccess) {
        h->d_rs = nullptr;
        return fail(DFB_ERR_OOM, "resampler table allocation failed");
    }
    return DFB_OK;
}

// Installs the directions `rates` / up / down with the new tap buffers `added` (owned from here on, freed on failure):
// the slab is reallocated for their histories and every slot starts afresh.
static int rs_install(dfb_stream *h, int rate, std::vector<int> rates, const ResampleDirs &up, const ResampleDirs &down,
                      const std::vector<float *> &added, bool replace) {
    const int old_rate = h->rate;
    std::vector<int> old_rates = h->rs_rates;
    const ResampleDirs old_up = h->rs_up, old_down = h->rs_down;
    h->rate = rate; h->rs_rates = std::move(rates); h->rs_up = up; h->rs_down = down;
    if (int rc = stream_slab(h)) {   // the old slab stays
        h->rate = old_rate; h->rs_rates = std::move(old_rates); h->rs_up = old_up; h->rs_down = old_down;
        for (float *p : added) cudaFree(p);
        return rc;
    }
    if (replace) {
        for (float *p : h->rs_taps) cudaFree(p);
        h->rs_taps.clear();
    }
    h->rs_taps.insert(h->rs_taps.end(), added.begin(), added.end());
    h->rs_rows.clear();
    slots_init(h);
    return DFB_OK;
}

extern "C" int dfb_stream_set_sample_rate(dfb_stream *h, int rate, const float *up_taps, int up_og, int up_nw, int up_width,
                                          const float *down_taps, int down_og, int down_nw, int down_width) {
    if (int rc = rate_setter(h)) return rc;
    if (mixed_rate(h))   // already at 48 kHz, with its registered slot rates
        return rate == kModelRate ? DFB_OK : fail(DFB_ERR_INVALID, "a handle with slot rates runs at 48000 Hz: its slots open at their rates");
    ResampleDirs up{}, down{};
    float *taps = nullptr;
    if (rate != kModelRate) {
        if (int rc = rs_directions(rate, up_taps, up_og, up_nw, up_width, down_taps, down_og, down_nw, down_width, &up.d[0],
                                   &down.d[0], &taps))
            return rc;
        return rs_install(h, rate, {rate}, up, down, {taps}, true);
    }
    return rs_install(h, 0, {}, up, down, {}, true);
}

// A rate of a mixed-rate handle's slots: one more direction of both resamplers, the first registration also adds the
// identity (48 kHz) direction 0.
extern "C" int dfb_stream_add_slot_rate(dfb_stream *h, int rate, const float *up_taps, int up_og, int up_nw, int up_width,
                                        const float *down_taps, int down_og, int down_nw, int down_width) {
    if (h && !h->spectral && h->rate)
        return fail(DFB_ERR_INVALID, "slot rates are registered on a 48 kHz handle: this one runs at %d Hz", h->rate);
    if (int rc = rate_setter(h)) return rc;
    ResampleDir up{}, down{};
    for (int i = 0; i < 2; i++)   // the arguments' checks first, the upload once the rate is known to be new
        if (int rc = rs_geometry(rate, i == 0, i ? down_taps : up_taps, i ? down_og : up_og, i ? down_nw : up_nw,
                                 i ? down_width : up_width, i ? &down : &up))
            return rc;
    if (std::find(h->rs_rates.begin(), h->rs_rates.end(), rate) != h->rs_rates.end()) return DFB_OK;
    std::vector<int> rates = h->rs_rates;
    ResampleDirs ups = h->rs_up, downs = h->rs_down;
    std::vector<float *> added;
    if (rates.empty()) {
        static const float one = 1.f;
        float *d_one = nullptr;
        if (cudaMalloc(&d_one, sizeof(float)) != cudaSuccess) return fail(DFB_ERR_OOM, "resampler taps allocation failed");
        if (cudaMemcpy(d_one, &one, sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
            cudaFree(d_one);
            return fail(DFB_ERR_CUDA, "resampler taps upload failed");
        }
        added.push_back(d_one);
        const int hop = h->st->hop;
        ups.d[0] = downs.d[0] = ResampleDir{d_one, 1, 1, 1, 0, 0, hop, hop, 0};
        rates.push_back(kModelRate);
    }
    float *taps = nullptr;
    const size_t k = rates.size();
    if (int rc = rs_directions(rate, up_taps, up_og, up_nw, up_width, down_taps, down_og, down_nw, down_width, &ups.d[k],
                               &downs.d[k], &taps)) {
        for (float *p : added) cudaFree(p);
        return rc;
    }
    added.push_back(taps);
    rates.push_back(rate);
    return rs_install(h, 0, std::move(rates), ups, downs, added, false);
}

// Debug aid: the resamplers of a handle on their own over a list of call sizes, every row one session from hop 0 in the
// direction of its rate
extern "C" int dfb_debug_resample_slots(int up, const dfb_stream *h, const int32_t *h_rates, const float *d_in, int64_t C,
                                        const int64_t *h_calls, int64_t n_calls, float *d_out, void *stream) {
    if (!h || !h_rates || !d_in || !d_out || C <= 0 || C > 65535 || !h_calls || n_calls <= 0)
        return fail(DFB_ERR_INVALID, "bad argument");
    std::vector<ResampleRow> rows((size_t)C);
    for (int64_t c = 0; c < C; c++) {
        const auto it = std::find(h->rs_rates.begin(), h->rs_rates.end(), (int)h_rates[c]);
        if (it == h->rs_rates.end()) return fail(DFB_ERR_INVALID, "row %lld: the handle has no direction at %d Hz", (long long)c, h_rates[c]);
        rows[(size_t)c] = ResampleRow{c, 0, kOpenEnd, it - h->rs_rates.begin()};
    }
    int64_t H = 0;
    for (int64_t i = 0; i < n_calls; i++) {
        if (h_calls[i] <= 0) return fail(DFB_ERR_INVALID, "call %lld has %lld hops", (long long)i, (long long)h_calls[i]);
        H += h_calls[i];
    }
    if (int rc = use_device(h->m->device)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const ResampleDirs &dirs = up ? h->rs_up : h->rs_down;
    const int64_t hp = rs_hist(h, dirs), W = H * h->st->hop;
    ResampleRow *d_rows = nullptr;
    float *hist = nullptr;
    int rc = DFB_OK;
    if (cudaMalloc(&d_rows, sizeof(ResampleRow) * C) != cudaSuccess || cudaMalloc(&hist, sizeof(float) * (C * hp + 1)) != cudaSuccess ||
        cudaMemcpyAsync(d_rows, rows.data(), sizeof(ResampleRow) * C, cudaMemcpyHostToDevice, s) != cudaSuccess ||
        cudaMemsetAsync(hist, 0, sizeof(float) * (C * hp + 1), s) != cudaSuccess)
        rc = fail(DFB_ERR_OOM, "debug buffers");
    for (int64_t i = 0, a0 = 0; i < n_calls && !rc; a0 += h_calls[i++])
        rc = launch_resample_stream(s, up != 0, dirs, (int)h->rs_rates.size(), d_rows, (int)C,
                                    ResampleIO{d_in, d_out, hist, W, W, i == n_calls - 1 ? W : 0, hp, a0, a0, h_calls[i], a0,
                                               kOpenEnd});   // the last call fills each row's end with zeros
    cudaStreamSynchronize(s);
    if (d_rows) cudaFree(d_rows);
    if (hist) cudaFree(hist);
    return rc;
}

// Debug aid: one resampler on its own over a list of call sizes, every row one session from hop 0
extern "C" int dfb_debug_resample_stream(int up, int rate, const float *d_taps, int og, int nw, int width, const float *d_in, int64_t C,
                                         const int64_t *h_calls, int64_t n_calls, float *d_out, void *stream) {
    ResampleDirs dirs{};
    ResampleDir &d = dirs.d[0];
    if (int rc = rs_geometry(rate, up != 0, d_taps, og, nw, width, &d)) return rc;
    if (!d_in || !d_out || C <= 0 || C > 65535 || !h_calls || n_calls <= 0) return fail(DFB_ERR_INVALID, "bad argument");
    int64_t H = 0;
    for (int64_t i = 0; i < n_calls; i++) {
        if (h_calls[i] <= 0) return fail(DFB_ERR_INVALID, "call %lld has %lld hops", (long long)i, (long long)h_calls[i]);
        H += h_calls[i];
    }
    int dev = 0;
    DFB_CUDA(cudaGetDevice(&dev));
    if (int rc = use_device(dev)) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    std::vector<ResampleRow> rows((size_t)C);
    for (int64_t c = 0; c < C; c++) rows[(size_t)c] = ResampleRow{c, 0, kOpenEnd, 0};
    ResampleRow *d_rows = nullptr;
    float *hist = nullptr;
    int rc = DFB_OK;
    if (cudaMalloc(&d_rows, sizeof(ResampleRow) * C) != cudaSuccess || cudaMalloc(&hist, sizeof(float) * C * d.S) != cudaSuccess ||
        cudaMemcpyAsync(d_rows, rows.data(), sizeof(ResampleRow) * C, cudaMemcpyHostToDevice, s) != cudaSuccess ||
        cudaMemsetAsync(hist, 0, sizeof(float) * C * d.S, s) != cudaSuccess)
        rc = fail(DFB_ERR_OOM, "debug buffers");
    for (int64_t i = 0, a0 = 0; i < n_calls && !rc; a0 += h_calls[i++])
        rc = launch_resample_stream(s, up != 0, dirs, 1, d_rows, (int)C,
                                    ResampleIO{d_in, d_out, hist, H * d.hop_in, H * d.hop_out, 0, d.S, a0, a0, h_calls[i], a0,
                                               kOpenEnd});
    cudaStreamSynchronize(s);
    if (d_rows) cudaFree(d_rows);
    if (hist) cudaFree(hist);
    return rc;
}

// d_in [B][n_frames * hop] -> d_out [B][n_frames * hop] (device pointers, asynchronous on `stream`); d_lsnr (or null)
// [B][n_frames]: the LSNR of the frame each output hop carries, NaN where it carries none
static int audio_only(const dfb_stream *h) {
    return h && h->spectral ? fail(DFB_ERR_INVALID, "a spectral handle takes spectrum frames: dfb_stream_process_spec / flush_spec") : DFB_OK;
}
extern "C" int dfb_stream_process_lsnr(dfb_stream *h, const float *d_in, int64_t n_frames, float *d_out, float *d_lsnr, void *stream) {
    if (int rc = audio_only(h)) return rc;
    if (!h || !d_in || !d_out || n_frames <= 0) return fail(DFB_ERR_INVALID, "bad argument");
    DFB_CUDA(cudaSetDevice(h->m->device));
    return audio_step(h, d_in, n_frames, false, d_out, d_lsnr, (cudaStream_t)stream);
}
extern "C" int dfb_stream_process(dfb_stream *h, const float *d_in, int64_t n_frames, float *d_out, void *stream) {
    return dfb_stream_process_lsnr(h, d_in, n_frames, d_out, nullptr, stream);
}

// End of the stream: the `latency` frames still in flight, computed with zero look-ahead exactly like the end of a
// batch enhance(); d_out [B][latency * hop].  Closes every open slot.  d_lsnr (or null) [B][latency]: the LSNR of the tail
// frames.
extern "C" int dfb_stream_flush_lsnr(dfb_stream *h, float *d_out, float *d_lsnr, void *stream) {
    if (int rc = audio_only(h)) return rc;
    if (!h || !d_out) return fail(DFB_ERR_INVALID, "bad argument");
    DFB_CUDA(cudaSetDevice(h->m->device));
    int rc = DFB_OK;
    if (dfb_stream_latency_frames(h) > 0) rc = audio_step(h, nullptr, 0, true, d_out, d_lsnr, (cudaStream_t)stream);
    if (!rc) slots_close_all(h);
    return rc;
}
extern "C" int dfb_stream_flush(dfb_stream *h, float *d_out, void *stream) { return dfb_stream_flush_lsnr(h, d_out, nullptr, stream); }

static int stage_grow(float **p, size_t *cap, size_t bytes) {
    if (bytes <= *cap) return DFB_OK;
    if (*p) cudaFree(*p);
    *p = nullptr; *cap = 0;
    if (cudaMalloc(p, bytes) != cudaSuccess) { *p = nullptr; return fail(DFB_ERR_OOM, "stream staging allocation failed"); }
    *cap = bytes;
    return DFB_OK;
}
// host-pointer variant (synchronous): h_in / h_out [B][n_frames * hop]; h_in == NULL flushes into h_out [B][latency * hop];
// h_lsnr (or null) [B][n_frames] / [B][latency] as dfb_stream_process_lsnr
extern "C" int dfb_stream_process_host_lsnr(dfb_stream *h, const float *h_in, int64_t n_frames, float *h_out, float *h_lsnr) {
    if (int rc = audio_only(h)) return rc;
    if (!h || (h_in && n_frames <= 0)) return fail(DFB_ERR_INVALID, "bad argument");
    DFB_CUDA(cudaSetDevice(h->m->device));
    const bool flush = h_in == nullptr;
    const int64_t nf = flush ? dfb_stream_latency_frames(h) : n_frames;
    if (nf == 0) {   // a flush without look-ahead has no output: it only closes the slots
        slots_close_all(h);
        return DFB_OK;
    }
    if (!h_out) return fail(DFB_ERR_INVALID, "bad argument");
    const size_t bytes = sizeof(float) * (size_t)h->B * nf * dfb_stream_frame_length(h), lbytes = sizeof(float) * (size_t)h->B * nf;
    int rc;
    if ((!flush && (rc = stage_grow(&h->stage_in, &h->stage_in_cap, bytes))) || (rc = stage_grow(&h->stage_out, &h->stage_out_cap, bytes)) ||
        (h_lsnr && (rc = stage_grow(&h->stage_lsnr, &h->stage_lsnr_cap, lbytes))))
        return rc;
    cudaStream_t s = h->m->stream;
    if (!flush) DFB_CUDA(cudaMemcpyAsync(h->stage_in, h_in, bytes, cudaMemcpyHostToDevice, s));
    if ((rc = audio_step(h, h->stage_in, nf, flush, h->stage_out, h_lsnr ? h->stage_lsnr : nullptr, s))) return rc;
    DFB_CUDA(cudaMemcpyAsync(h_out, h->stage_out, bytes, cudaMemcpyDeviceToHost, s));
    if (h_lsnr) DFB_CUDA(cudaMemcpyAsync(h_lsnr, h->stage_lsnr, lbytes, cudaMemcpyDeviceToHost, s));
    DFB_CUDA(cudaStreamSynchronize(s));
    if (flush) slots_close_all(h);
    return DFB_OK;
}
extern "C" int dfb_stream_process_host(dfb_stream *h, const float *h_in, int64_t n_frames, float *h_out) {
    return dfb_stream_process_host_lsnr(h, h_in, n_frames, h_out, nullptr);
}

// ---- session export / import (dfb_stream_export_sessions / dfb_stream_import_sessions; DESIGN.md section 5o).  A session
// is its rows of the 17 state arrays plus the host bookkeeping of its slots; its outputs depend on the handle only through
// the handle's clock, which the blob replaces by the session's age.  The rows move in one kernel launch per direction.
constexpr uint32_t kBlobMagic = 0x53424644u;   // "DFBS", little-endian
constexpr uint32_t kBlobVersion = 1;
constexpr int64_t kNoLsnr = INT64_MIN;         // BlobSession::lsnr_start of a session whose LSNR head never ran
struct BlobHeader {
    uint32_t magic, version;
    uint64_t fingerprint;
    int32_t sr, fft_size, hop_size, nb_erb;
    int32_t gating_mode, gate_tails, n_sessions, n_rows;
    int64_t total_bytes;
    int64_t row_floats[kStateArrays];
};
struct BlobSession {
    int64_t age, lsnr_start, ctl_switch;
    int32_t rate, channels, reduce, reserved;
    float lim, beta;
    int32_t gate;
    float th[3];
    float last_lim, last_beta, prev_lim, prev_beta;
    int32_t last_gate;
    float last_th[3];
    int32_t up_hist, down_hist;
    int64_t data_offset;
};
static_assert(sizeof(BlobHeader) == 192 && sizeof(BlobSession) == 112, "the blob layout of include/dfb200.h");

// One row (channel) of a blob: its slab row (-1 on export: a fresh stream's initial state), its floats' offset in the
// data area, its session's own resampler history widths and (import) the leading entries of its LSNR tail read as NaN.
struct SessionRow { int64_t blob; int slab, up, down, nan_l; };

// Offset of array a in a blob row: arrays 0 .. 14 as the slab's row_off packs them, then the row's own histories.
__device__ __forceinline__ int64_t blob_elem0(const StateLayout &lay, const SessionRow &r, int a) {
    return r.blob + (a < kRsArray ? lay.row_off[a] : lay.row_off[kRsArray] + (a > kRsArray ? r.up : 0));
}

// Every listed row of every state array into the blob, read where the row's state lives at the last call (a pending
// move's source) or as a fresh stream's initial state.  grid (x, rows, kStateArrays).
__global__ void k_sessions_pack(const float *__restrict__ slab, StateLayout lay, int Bs, const SessionRow *__restrict__ rows,
                                float *__restrict__ blob, int E, int Fd) {
    const int a = blockIdx.z;
    const SessionRow r = rows[blockIdx.y];
    const int64_t n = a < kRsArray ? (int64_t)lay.layers[a] * lay.per_row[a] : a == kRsArray ? r.up : r.down;
    float *dst = blob + blob_elem0(lay, r, a);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        dst[e] = r.slab >= 0 ? slab[state_elem(lay, Bs, a, r.slab, e)] : state_init(a, e, E, Fd);
}

// The blob's rows into slab rows: a resampler history padded with zeros to the handle's width, the first nan_l entries
// of the LSNR tail (array 12) NaN.  grid (x, rows, kStateArrays).
__global__ void k_sessions_unpack(float *__restrict__ slab, StateLayout lay, int Bs, const SessionRow *__restrict__ rows,
                                  const float *__restrict__ blob) {
    const int a = blockIdx.z;
    const SessionRow r = rows[blockIdx.y];
    const int64_t n = (int64_t)lay.layers[a] * lay.per_row[a], own = a < kRsArray ? n : a == kRsArray ? r.up : r.down;
    const float *src = blob + blob_elem0(lay, r, a);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        float v = e < own ? src[e] : 0.f;
        if (a == 12 && e < r.nan_l) v = __int_as_float(0x7fffffff);
        slab[state_elem(lay, Bs, a, r.slab, e)] = v;
    }
}

// One launch of the pack (export) or unpack kernel over the rows, their table in the model arena.
static int sessions_launch(dfb_stream *h, bool pack, const std::vector<SessionRow> &rows, float *blob_data, cudaStream_t s) {
    if (rows.empty()) return DFB_OK;
    dfb_model *m = h->m;
    size_t off[kStateArrays];
    StateLayout lay;
    stream_state_floats(h, off, &lay);
    if (int rc = m->arena.reserve(sizeof(SessionRow) * rows.size() + 1024)) return rc;
    m->arena.reset();
    SessionRow *d_rows = m->arena.take<SessionRow>(rows.size());
    DFB_CUDA(cudaMemcpyAsync(d_rows, rows.data(), sizeof(SessionRow) * rows.size(), cudaMemcpyHostToDevice, s));
    const dim3 grid(4, (unsigned)rows.size(), kStateArrays);
    if (pack)
        k_sessions_pack<<<grid, 256, 0, s>>>(h->slab, lay, h->B, d_rows, blob_data, m->cfg.nb_erb, m->cfg.nb_df);
    else
        k_sessions_unpack<<<grid, 256, 0, s>>>(h->slab, lay, h->B, d_rows, blob_data);
    DFB_LAUNCH_CHECK();
    m->arena.reset();
    return DFB_OK;
}

// what session export and import refuse on any handle
static int sessions_handle(const dfb_stream *h) {
    if (!h) return fail(DFB_ERR_INVALID, "null stream");
    if (h->spectral) return fail(DFB_ERR_UNSUPPORTED, "session export / import: audio handles only (a spectral handle's sessions do not move)");
    if (h->m->cfg.model_kind == 1) return fail(DFB_ERR_UNSUPPORTED, "DeepFilterNet v1 has no streaming sessions");
    return DFB_OK;
}
static int eff_gating_mode(const dfb_stream *h) { return h->gating_mode >= 0 ? h->gating_mode : h->m->gating_mode; }
static int slot_rate_of(const dfb_stream *h, int b) { return resampled(h) ? h->rs_rates[(size_t)h->slot_dir[(size_t)b]] : kModelRate; }
static int rs_own(const dfb_stream *h, int dir, bool up) { return resampled(h) ? (up ? h->rs_up : h->rs_down).d[dir].S : 0; }
static bool ctl_shape(const dfb_model_config &c) { return c.df_order == 5 && c.nb_df == 96 && c.nb_erb == 32; }

// A handle whose clock has settled: its DNN and output frames trail the input by the model's look-ahead and lag, a full
// halo lies behind them and every tail is full.  A session's state means the same in every such handle.
static bool clock_settled(const dfb_stream *h) {
    const StreamState &S = h->S;
    const dfb_model_config &c = h->m->cfg;
    const ChunkGeom g = chunk_geom(c);
    return S.started && S.dnn_started && S.d1 == S.a1 - g.Lmax && S.e1 == S.d1 - g.lag && S.d1 >= kHalo && S.n_feat == g.Hf &&
           S.n_mc == kMcTail && (c.conv_kt == 1 || S.n_dec == kHalo);
}
// An idle handle (no live row) moves its clock to the first settled frame, as a call with nothing to compute would.
static void clock_settle(dfb_stream *h) {
    StreamState &S = h->S;
    const ChunkGeom g = chunk_geom(h->m->cfg);
    S.a1 = std::max<int64_t>(S.a1, kHalo + g.Lmax);
    S.d1 = S.a1 - g.Lmax; S.e1 = S.d1 - g.lag;
    S.started = S.dnn_started = true;
    S.n_feat = g.Hf; S.n_mc = kMcTail; S.n_dec = kHalo;
}

// An export's slots: open, each linked group whole, from its channel 0 and in channel order.  The blob's header, its
// session records and the rows to pack.
static int export_plan(const dfb_stream *h, const int32_t *slots, int n, BlobHeader *hd, std::vector<BlobSession> *ses,
                       std::vector<SessionRow> *rows) {
    if (int rc = sessions_handle(h)) return rc;
    if (n <= 0 || !slots) return fail(DFB_ERR_INVALID, "bad argument");
    std::vector<int64_t> s64(slots, slots + n);
    if (int rc = slot_list_check(h, s64.data(), n)) return rc;
    for (int i = 0; i < n; i++)
        if (h->slot_state[(size_t)slots[i]] != kSlotOpen)
            return fail(DFB_ERR_INVALID, "slot %d is %s: only open sessions are exported", slots[i],
                        h->slot_state[(size_t)slots[i]] == kSlotFree ? "free" : "closing");
    // runtime gating: the sessions' own decoder tails (a held session keeps those of its last advancing call)
    const bool tails = h->slot_rt[(size_t)slots[0]] != 0;
    for (int i = 1; i < n; i++)
        if (eff_gating_mode(h) == DFB_GATING_RUNTIME && (h->slot_rt[(size_t)slots[i]] != 0) != tails)
            return fail(DFB_ERR_INVALID, "runtime gating: the decoder tails of slot %d %s kept by its last call, those of slot %d %s: "
                        "export them apart", slots[0], tails ? "were" : "were not", slots[i], tails ? "were not" : "were");
    size_t off[kStateArrays];
    StateLayout lay;
    stream_state_floats(h, off, &lay);
    *hd = BlobHeader{kBlobMagic, kBlobVersion, h->m->fingerprint, h->st->sr, h->st->fft, h->st->hop, h->st->nb_erb,
                     eff_gating_mode(h), eff_gating_mode(h) == DFB_GATING_RUNTIME && tails ? 1 : 0, 0, n, 0, {}};
    for (int a = 0; a < kStateArrays; a++) hd->row_floats[a] = (int64_t)lay.layers[a] * lay.per_row[a];
    ses->clear(); rows->clear();
    int64_t data = 0;   // floats
    for (int i = 0; i < n;) {
        const int b = slots[i], g = h->slot_grp[(size_t)b], nch = h->slot_nch[(size_t)b], dir = h->slot_dir[(size_t)b];
        if (b != g)
            return fail(DFB_ERR_INVALID, "slot %d is a channel of the group of slot %d: list a group from its channel 0, in channel order", b, g);
        for (int c = 0; c < nch; c++)
            if (i + c >= n || h->slot_row[(size_t)slots[i + c]] != h->slot_row[(size_t)g] + c)
                return fail(DFB_ERR_INVALID, "the group of slot %d: list its %d channels in channel order", g, nch);
        const size_t sb = (size_t)b;
        const int64_t first = h->slot_first[sb];
        BlobSession r{};
        r.age = h->S.a1 - first;
        // relative to the session's own frames: lsnr_from is on the handle's clock, which has moved on by the frames the
        // session was held since then
        r.lsnr_start = h->lsnr_from >= 0 ? h->lsnr_from - (first - h->slot_held_frames[sb]) : kNoLsnr;
        r.rate = slot_rate_of(h, b); r.channels = nch; r.reduce = nch > 1 ? h->group_reduce : kReduceNone;
        // the settings the session's next call resolves, pinned: its own, or the handle's at this time
        r.lim = std::isnan(h->slot_lim[sb]) ? h->lim : h->slot_lim[sb];
        r.beta = std::isnan(h->slot_beta[sb]) ? default_beta(h->m) : h->slot_beta[sb];
        const bool own = h->slot_gate[sb] >= 0;
        r.gate = own ? h->slot_gate[sb] : (h->gating ? 1 : 0);
        for (int k = 0; k < 3; k++) r.th[k] = own ? h->slot_th[3 * sb + k] : h->th[k];
        // the last call's settings and the switch to them; without a per-row table (or before its first call) the
        // session has one setting for all of its frames
        if (h->ctl_on && !h->slot_fresh[sb]) {
            const SlotCtl &c = h->slot_ctl[sb];
            r.last_lim = c.lim; r.last_beta = c.beta; r.prev_lim = c.lim0; r.prev_beta = c.beta0; r.ctl_switch = c.sw - first;
            r.last_gate = c.gate; r.last_th[0] = c.th_min; r.last_th[1] = c.th_erb; r.last_th[2] = c.th_df;
        } else {
            r.last_lim = r.prev_lim = r.lim; r.last_beta = r.prev_beta = r.beta; r.ctl_switch = 0;
            r.last_gate = r.gate; for (int k = 0; k < 3; k++) r.last_th[k] = r.th[k];
        }
        r.up_hist = rs_own(h, dir, true); r.down_hist = rs_own(h, dir, false);
        r.data_offset = data;   // floats into the data area for now
        const int64_t per = lay.row_off[kRsArray] + r.up_hist + r.down_hist;
        for (int c = 0; c < nch; c++, data += per)
            rows->push_back(SessionRow{data, h->row_src[(size_t)h->slot_row[(size_t)slots[i + c]]], r.up_hist, r.down_hist, 0});
        ses->push_back(r);
        i += nch;
    }
    hd->n_sessions = (int32_t)ses->size();
    const int64_t data0 = (int64_t)sizeof(BlobHeader) + (int64_t)sizeof(BlobSession) * (int64_t)ses->size();
    for (BlobSession &r : *ses) r.data_offset = data0 + r.data_offset * (int64_t)sizeof(float);
    hd->total_bytes = data0 + data * (int64_t)sizeof(float);
    return DFB_OK;
}

static void header_bytes(const BlobHeader &hd, const std::vector<BlobSession> &ses, unsigned char *dst) {
    memcpy(dst, &hd, sizeof hd);
    if (!ses.empty()) memcpy(dst + sizeof hd, ses.data(), sizeof(BlobSession) * ses.size());
}

// A released export frees its slots at once, without a tail: the sessions live only in the blob.
static void export_release(dfb_stream *h, const int32_t *slots, int n) {
    for (int i = 0; i < n; i++) slot_release(h, slots[i]);
    rows_layout(h);
    h->slot_ops = true;
}

extern "C" int dfb_stream_session_bytes(const dfb_stream *h, const int32_t *slots, int n, int64_t *bytes) {
    if (!bytes) return fail(DFB_ERR_INVALID, "bad argument");
    BlobHeader hd;
    std::vector<BlobSession> ses;
    std::vector<SessionRow> rows;
    if (int rc = export_plan(h, slots, n, &hd, &ses, &rows)) return rc;
    *bytes = hd.total_bytes;
    return DFB_OK;
}

// a device blob: its rows are read and written as floats
static int blob_pointer(const void *d_blob) {
    if (!d_blob) return fail(DFB_ERR_INVALID, "bad argument");
    if ((uintptr_t)d_blob % alignof(float)) return fail(DFB_ERR_INVALID, "a device session blob must be 4-byte aligned");
    return DFB_OK;
}

extern "C" int dfb_stream_export_sessions(dfb_stream *h, const int32_t *slots, int n, int release, void *d_blob, void *stream) {
    BlobHeader hd;
    std::vector<BlobSession> ses;
    std::vector<SessionRow> rows;
    if (int rc = export_plan(h, slots, n, &hd, &ses, &rows)) return rc;
    if (int rc = blob_pointer(d_blob)) return rc;
    DFB_CUDA(cudaSetDevice(h->m->device));
    cudaStream_t s = (cudaStream_t)stream;
    const size_t head = sizeof(BlobHeader) + sizeof(BlobSession) * ses.size();
    std::vector<unsigned char> hb(head);
    header_bytes(hd, ses, hb.data());
    DFB_CUDA(cudaMemcpyAsync(d_blob, hb.data(), head, cudaMemcpyHostToDevice, s));
    if (int rc = sessions_launch(h, true, rows, (float *)((char *)d_blob + head), s)) return rc;
    // the pack has read the slab rows (a released session's may be reused by the next call on any stream) and the blob is
    // complete when this returns; the kernel's row table in the model arena is free again
    DFB_CUDA(cudaStreamSynchronize(s));
    if (release) export_release(h, slots, n);
    return DFB_OK;
}

extern "C" int dfb_stream_export_sessions_host(dfb_stream *h, const int32_t *slots, int n, int release, void *h_blob) {
    BlobHeader hd;
    std::vector<BlobSession> ses;
    std::vector<SessionRow> rows;
    if (int rc = export_plan(h, slots, n, &hd, &ses, &rows)) return rc;
    if (!h_blob) return fail(DFB_ERR_INVALID, "bad argument");
    DFB_CUDA(cudaSetDevice(h->m->device));
    const size_t head = sizeof(BlobHeader) + sizeof(BlobSession) * ses.size(), data = (size_t)hd.total_bytes - head;
    if (int rc = stage_grow(&h->sess_stage, &h->sess_stage_cap, data)) return rc;
    cudaStream_t s = h->m->stream;
    if (int rc = sessions_launch(h, true, rows, h->sess_stage, s)) return rc;
    DFB_CUDA(cudaMemcpyAsync((char *)h_blob + head, h->sess_stage, data, cudaMemcpyDeviceToHost, s));
    header_bytes(hd, ses, (unsigned char *)h_blob);
    DFB_CUDA(cudaStreamSynchronize(s));
    if (release) export_release(h, slots, n);
    return DFB_OK;
}

// The header of a blob, checked on its own: magic, version, counts against the n listed slots, and a size that holds its
// records (read only after this check).
static int import_header(const BlobHeader &hd, int n) {
    if (hd.magic != kBlobMagic) return fail(DFB_ERR_INVALID, "not a session blob (magic 0x%08x)", hd.magic);
    if (hd.version != kBlobVersion) return fail(DFB_ERR_INVALID, "session blob version %u (this library reads %u)", hd.version, kBlobVersion);
    if (hd.n_sessions < 1 || hd.n_rows < hd.n_sessions || hd.n_rows > 65535)
        return fail(DFB_ERR_INVALID, "session blob with %d sessions in %d rows", hd.n_sessions, hd.n_rows);
    if (hd.n_rows != n) return fail(DFB_ERR_INVALID, "the blob holds %d channels: list %d slots, not %d", hd.n_rows, hd.n_rows, n);
    if (hd.total_bytes < (int64_t)sizeof(BlobHeader) + (int64_t)sizeof(BlobSession) * hd.n_sessions)
        return fail(DFB_ERR_INVALID, "session blob of %lld bytes: shorter than its %d session records", (long long)hd.total_bytes,
                    hd.n_sessions);
    return DFB_OK;
}

// Everything an import checks before it changes anything, and its plan: per blob row its slot and session, the slab
// rows it lands in and its table row for the unpack kernel.
struct ImportPlan {
    std::vector<int> dir;            // per session: its direction in this handle
    std::vector<SessionRow> rows;    // per blob row
    bool idle = false;               // the handle has no live row: its clock settles and it takes the blob's gating tails
};
static int import_plan(dfb_stream *h, const int32_t *slots, int n, const BlobHeader &hd, const std::vector<BlobSession> &ses,
                       ImportPlan *p) {
    const dfb_model_config &c = h->m->cfg;
    size_t off[kStateArrays];
    StateLayout lay;
    stream_state_floats(h, off, &lay);
    // the blob's own consistency: its records and size
    int64_t data = (int64_t)sizeof(BlobHeader) + (int64_t)sizeof(BlobSession) * hd.n_sessions, rows = 0;
    for (int k = 0; k < kRsArray; k++)
        if (hd.row_floats[k] != (int64_t)lay.layers[k] * lay.per_row[k])
            return fail(DFB_ERR_INVALID, "state array %d: the blob's rows hold %lld floats, this handle's %lld", k,
                        (long long)hd.row_floats[k], (long long)lay.layers[k] * lay.per_row[k]);
    for (const BlobSession &r : ses) {
        if (r.channels < 1 || r.up_hist < 0 || r.down_hist < 0 || r.up_hist > 4096 || r.down_hist > 4096 || r.age < 0 ||
            r.age > kOpenEnd || r.data_offset != data)
            return fail(DFB_ERR_INVALID, "session blob: a malformed session record");
        data += (int64_t)r.channels * (lay.row_off[kRsArray] + r.up_hist + r.down_hist) * (int64_t)sizeof(float);
        rows += r.channels;
    }
    if (rows != hd.n_rows || data != hd.total_bytes)
        return fail(DFB_ERR_INVALID, "session blob: its records describe %lld bytes in %lld rows, its header %lld in %d",
                    (long long)data, (long long)rows, (long long)hd.total_bytes, hd.n_rows);
    // compatibility with this handle
    if (hd.fingerprint != h->m->fingerprint)
        return fail(DFB_ERR_INVALID, "the sessions ran another model (fingerprint %016llx, this handle's model %016llx)",
                    (unsigned long long)hd.fingerprint, (unsigned long long)h->m->fingerprint);
    if (hd.sr != h->st->sr || hd.fft_size != h->st->fft || hd.hop_size != h->st->hop || hd.nb_erb != h->st->nb_erb)
        return fail(DFB_ERR_INVALID, "the sessions ran another DSP state (sr %d, fft %d, hop %d, %d ERB bands; this handle's: %d, %d, %d, %d)",
                    hd.sr, hd.fft_size, hd.hop_size, hd.nb_erb, h->st->sr, h->st->fft, h->st->hop, h->st->nb_erb);
    if (hd.gating_mode != eff_gating_mode(h))
        return fail(DFB_ERR_INVALID, "the sessions ran in gating mode %d, this handle runs %d", hd.gating_mode, eff_gating_mode(h));
    std::vector<int64_t> s64(slots, slots + n);
    if (int rc = slot_list_check(h, s64.data(), n)) return rc;
    for (int i = 0; i < n; i++)
        if (h->slot_state[(size_t)slots[i]] != kSlotFree) return fail(DFB_ERR_INVALID, "slot %d is not free", slots[i]);
    p->idle = h->n_live == 0;
    if (!p->idle && !clock_settled(h))
        return fail(DFB_ERR_INVALID, "this handle's clock has not settled since its start or flush: it settles after %d frames "
                    "of calls (8 of halo, %d of look-ahead); import into it then, or into a handle with no live session",
                    kHalo + chunk_geom(c).Lmax, chunk_geom(c).Lmax);
    if (!p->idle && hd.gating_mode == DFB_GATING_RUNTIME && (hd.gate_tails != 0) != h->S.rt_valid)
        return fail(DFB_ERR_INVALID, "runtime gating: the sessions' decoder tails %s kept by their last call, this handle's live "
                    "sessions' %s: import into a handle whose last call gated %s, or into one with no live session",
                    hd.gate_tails ? "were" : "were not", h->S.rt_valid ? "were" : "were not", hd.gate_tails ? "too" : "nothing either");
    const bool ctl = ctl_shape(c);
    p->dir.clear();
    for (const BlobSession &r : ses) {
        int dir = -1;
        if (mixed_rate(h)) {
            for (size_t k = 0; k < h->rs_rates.size(); k++)
                if (h->rs_rates[k] == r.rate) dir = (int)k;
        } else if (r.rate == (h->rate ? h->rate : kModelRate)) {
            dir = 0;
        }
        if (dir < 0) {
            std::string runs = mixed_rate(h) ? "" : std::to_string(h->rate ? h->rate : kModelRate);
            for (int rr : mixed_rate(h) ? h->rs_rates : std::vector<int>{}) runs += (runs.empty() ? "" : ", ") + std::to_string(rr);
            return fail(DFB_ERR_INVALID, "a session at %d Hz: this handle runs %s", r.rate, runs.c_str());
        }
        if (r.up_hist != rs_own(h, dir, true) || r.down_hist != rs_own(h, dir, false))
            return fail(DFB_ERR_INVALID, "a session at %d Hz with resampler histories of %d / %d samples: this handle's are %d / %d",
                        r.rate, r.up_hist, r.down_hist, rs_own(h, dir, true), rs_own(h, dir, false));
        if (r.channels > 1 && r.reduce != h->group_reduce)
            return fail(DFB_ERR_INVALID, "a group of %d channels with mask reduction %d: this handle's groups reduce by %d",
                        r.channels, r.reduce, h->group_reduce);
        if (!ctl && (r.lim != h->lim || r.beta != default_beta(h->m) || r.gate != (h->gating ? 1 : 0) ||
                     (r.gate && memcmp(r.th, h->th, sizeof r.th))))
            return fail(DFB_ERR_UNSUPPORTED, "per-session settings are built for df_order 5, nb_df 96 and 32 ERB bands: the "
                        "sessions' settings differ from this handle's");
        p->dir.push_back(dir);
    }
    // slab rows: a new row lands in its own slab row unless a pending move still reads that one
    std::vector<char> used((size_t)h->B, 0);
    for (int r = 0; r < h->n_live; r++)
        if (h->row_src[(size_t)r] >= 0) used[(size_t)h->row_src[(size_t)r]] = 1;
    const ChunkGeom g = chunk_geom(c);
    p->rows.clear();
    int next = 0;
    int64_t boff = 0;
    for (const BlobSession &r : ses) {
        // DeepFilterNet2's output trails its DNN: the LSNR tail's frames [d1 - kMcTail, d1) may still be output, and the
        // ones before the session's LSNR start have none
        int nan_l = 0;
        if (g.lag > 0) {
            const int64_t t0 = r.age - g.Lmax - kMcTail;   // the session's frame of tail entry 0
            nan_l = r.lsnr_start == kNoLsnr ? kMcTail : (int)std::min<int64_t>(kMcTail, std::max<int64_t>(0, r.lsnr_start - t0));
        }
        for (int ch = 0; ch < r.channels; ch++) {
            const int row = h->n_live + (int)p->rows.size();
            int q = row;
            if (used[(size_t)q]) {
                while (used[(size_t)next]) next++;
                q = next;
            }
            used[(size_t)q] = 1;
            p->rows.push_back(SessionRow{boff, q, r.up_hist, r.down_hist, nan_l});
            boff += lay.row_off[kRsArray] + r.up_hist + r.down_hist;
        }
    }
    return ctl ? ctl_enable(h) : DFB_OK;   // the sessions' own settings go to the per-row table (it changes no output)
}

// The blob's sessions in the listed slots, as the source left them: rebased onto this handle's clock, settings pinned.
static void import_slots(dfb_stream *h, const int32_t *slots, const BlobHeader &hd, const std::vector<BlobSession> &ses,
                         const ImportPlan &p) {
    if (p.idle) {
        clock_settle(h);
        h->S.rt_valid = hd.gate_tails != 0;
    }
    const bool ctl = h->ctl_on;
    int i = 0;
    for (size_t k = 0; k < ses.size(); k++) {
        const BlobSession &r = ses[k];
        const int64_t first = h->S.a1 - r.age;
        if (p.idle && r.lsnr_start != kNoLsnr) h->lsnr_from = std::max<int64_t>(0, std::min(h->S.d1, first + r.lsnr_start));
        for (int ch = 0; ch < r.channels; ch++, i++) {
            const size_t b = (size_t)slots[i];
            const int row = h->n_live++;
            h->slot_row[b] = row;
            h->row_slot[(size_t)row] = (int)b;
            h->row_src[(size_t)row] = p.rows[(size_t)i].slab;
            h->slot_grp[b] = slots[i - ch];
            h->slot_nch[b] = r.channels;
            h->slot_state[b] = kSlotOpen;
            h->slot_first[b] = first;
            h->slot_end[b] = kOpenEnd;
            h->slot_dir[b] = p.dir[k];
            h->slot_rt[b] = hd.gate_tails != 0;
            h->slot_held_frames[b] = 0;
            if (ctl) {
                h->slot_lim[b] = r.lim; h->slot_beta[b] = r.beta;
                h->slot_gate[b] = (signed char)(r.gate ? 1 : 0);
                for (int j = 0; j < 3; j++) h->slot_th[3 * b + j] = r.th[j];
                h->slot_fresh[b] = 0;
                h->slot_ctl[b] = SlotCtl{r.last_lim, r.last_beta, r.prev_lim, r.prev_beta, first + r.ctl_switch, r.last_th[0],
                                         r.last_th[1], r.last_th[2], r.last_gate};
            } else {   // the handle's settings, which the plan found equal to the session's
                h->slot_lim[b] = h->slot_beta[b] = NAN;
                h->slot_gate[b] = -1;
                h->slot_fresh[b] = 1;
            }
        }
    }
    // clock_settle moves d1 back to a1 - Lmax on a handle that was flushed (a flush leaves d1 = a1), and an LSNR request
    // after the flush set lsnr_from to that d1: the LSNR head must start no later than the imported sessions' next frame
    if (p.idle && ses.size() && ses[0].lsnr_start == kNoLsnr && h->lsnr_from > h->S.d1) h->lsnr_from = h->S.d1;
    rows_layout(h);   // behind held rows, the new rows move into the active prefix
    h->tab_dirty = true;
    h->slot_ops = true;
}

// the header and session records of a host blob
static int host_records(const void *h_blob, int n, BlobHeader *hd, std::vector<BlobSession> *ses) {
    if (!h_blob) return fail(DFB_ERR_INVALID, "bad argument");
    memcpy(hd, h_blob, sizeof *hd);
    if (int rc = import_header(*hd, n)) return rc;
    ses->resize((size_t)hd->n_sessions);
    memcpy(ses->data(), (const char *)h_blob + sizeof *hd, sizeof(BlobSession) * ses->size());
    return DFB_OK;
}

extern "C" int dfb_stream_import_sessions(dfb_stream *h, const int32_t *slots, int n, const void *d_blob, void *stream) {
    if (int rc = sessions_handle(h)) return rc;
    if (n <= 0 || !slots) return fail(DFB_ERR_INVALID, "bad argument");
    if (int rc = blob_pointer(d_blob)) return rc;
    DFB_CUDA(cudaSetDevice(h->m->device));
    cudaStream_t s = (cudaStream_t)stream;
    // the header first; its records only once the header says the blob holds them
    BlobHeader hd;
    DFB_CUDA(cudaMemcpyAsync(&hd, d_blob, sizeof hd, cudaMemcpyDeviceToHost, s));
    DFB_CUDA(cudaStreamSynchronize(s));
    if (int rc = import_header(hd, n)) return rc;
    std::vector<BlobSession> ses((size_t)hd.n_sessions);
    DFB_CUDA(cudaMemcpyAsync(ses.data(), (const char *)d_blob + sizeof hd, sizeof(BlobSession) * ses.size(), cudaMemcpyDeviceToHost, s));
    DFB_CUDA(cudaStreamSynchronize(s));
    ImportPlan p;
    if (int rc = import_plan(h, slots, n, hd, ses, &p)) return rc;
    const size_t head = sizeof(BlobHeader) + sizeof(BlobSession) * ses.size();
    if (int rc = sessions_launch(h, false, p.rows, (float *)((const char *)d_blob + head), s)) return rc;
    // the rows are in place, and the kernel's row table in the model arena is free again, before the handle's next call
    // on any stream
    DFB_CUDA(cudaStreamSynchronize(s));
    import_slots(h, slots, hd, ses, p);
    return DFB_OK;
}

extern "C" int dfb_stream_import_sessions_host(dfb_stream *h, const int32_t *slots, int n, const void *h_blob) {
    if (int rc = sessions_handle(h)) return rc;
    if (n <= 0 || !slots) return fail(DFB_ERR_INVALID, "bad argument");
    BlobHeader hd;
    std::vector<BlobSession> ses;
    if (int rc = host_records(h_blob, n, &hd, &ses)) return rc;
    DFB_CUDA(cudaSetDevice(h->m->device));
    ImportPlan p;
    if (int rc = import_plan(h, slots, n, hd, ses, &p)) return rc;
    const size_t head = sizeof(BlobHeader) + sizeof(BlobSession) * ses.size(), data = (size_t)hd.total_bytes - head;
    if (int rc = stage_grow(&h->sess_stage, &h->sess_stage_cap, data)) return rc;
    cudaStream_t s = h->m->stream;
    DFB_CUDA(cudaMemcpyAsync(h->sess_stage, (const char *)h_blob + head, data, cudaMemcpyHostToDevice, s));
    if (int rc = sessions_launch(h, false, p.rows, h->sess_stage, s)) return rc;
    DFB_CUDA(cudaStreamSynchronize(s));
    import_slots(h, slots, hd, ses, p);
    return DFB_OK;
}

// ---- spectral handle (dfb_stream_create_spec): capi.rs df_process_frame_raw, batched and for n_frames frames at once.
// d_spec [B][n_frames][F] complex -> [B][n_frames] rows of gains / coefs / LSNR / stage (device pointers, asynchronous).
static int spec_only(const dfb_stream *h) {
    if (!h) return fail(DFB_ERR_INVALID, "null stream");
    return h->spectral ? DFB_OK : fail(DFB_ERR_INVALID, "an audio handle takes audio: dfb_stream_create_spec makes a spectral one");
}
extern "C" int dfb_stream_process_spec(dfb_stream *h, const float *d_spec, int64_t n_frames, float *d_gains, float *d_coefs,
                                       float *d_lsnr, int8_t *d_stage, void *stream) {
    if (int rc = spec_only(h)) return rc;
    if (!d_spec || !d_gains || n_frames <= 0) return fail(DFB_ERR_INVALID, "bad argument");
    DFB_CUDA(cudaSetDevice(h->m->device));
    SpecOut so{d_gains, d_coefs, d_lsnr, d_stage};
    return stream_step(h, d_spec, n_frames, false, nullptr, nullptr, (cudaStream_t)stream, &so);
}
// end of stream: the last `latency` frames, computed with zero look-ahead features; closes every open slot
extern "C" int dfb_stream_flush_spec(dfb_stream *h, float *d_gains, float *d_coefs, float *d_lsnr, int8_t *d_stage, void *stream) {
    if (int rc = spec_only(h)) return rc;
    const int64_t L = dfb_stream_latency_frames(h);
    if (L > 0 && !d_gains) return fail(DFB_ERR_INVALID, "bad argument");
    DFB_CUDA(cudaSetDevice(h->m->device));
    int rc = DFB_OK;
    SpecOut so{d_gains, d_coefs, d_lsnr, d_stage};
    if (L > 0) rc = stream_step(h, nullptr, 0, true, nullptr, nullptr, (cudaStream_t)stream, &so);
    if (!rc) slots_close_all(h);
    return rc;
}
// host-pointer variant (synchronous): h_spec == NULL flushes into [B][latency] rows
extern "C" int dfb_stream_process_spec_host(dfb_stream *h, const float *h_spec, int64_t n_frames, float *h_gains, float *h_coefs,
                                            float *h_lsnr, int8_t *h_stage) {
    if (int rc = spec_only(h)) return rc;
    if (h_spec && n_frames <= 0) return fail(DFB_ERR_INVALID, "bad argument");
    DFB_CUDA(cudaSetDevice(h->m->device));
    const bool flush = h_spec == nullptr;
    const int64_t nf = flush ? dfb_stream_latency_frames(h) : n_frames;
    if (nf == 0) {   // a flush without look-ahead has no output: it only closes the slots
        slots_close_all(h);
        return DFB_OK;
    }
    if (!h_gains) return fail(DFB_ERR_INVALID, "bad argument");
    const dfb_model_config &c = h->m->cfg;
    const size_t rows = (size_t)h->B * nf, ng = rows * c.nb_erb, nc = rows * c.nb_df * 2 * c.df_order;
    const size_t in_bytes = sizeof(float) * rows * 2 * h->st->tb.F, out_bytes = sizeof(float) * (ng + nc + rows) + rows;
    int rc;
    if ((!flush && (rc = stage_grow(&h->spec_stage_in, &h->spec_in_cap, in_bytes))) ||
        (rc = stage_grow(&h->spec_stage_out, &h->spec_out_cap, out_bytes)))
        return rc;
    float *g = h->spec_stage_out, *cf = g + ng, *l = cf + nc;
    int8_t *sg = (int8_t *)(l + rows);
    cudaStream_t s = h->m->stream;
    if (!flush) DFB_CUDA(cudaMemcpyAsync(h->spec_stage_in, h_spec, in_bytes, cudaMemcpyHostToDevice, s));
    SpecOut so{g, h_coefs ? cf : nullptr, h_lsnr ? l : nullptr, h_stage ? sg : nullptr};
    if ((rc = stream_step(h, h->spec_stage_in, nf, flush, nullptr, nullptr, s, &so))) return rc;
    DFB_CUDA(cudaMemcpyAsync(h_gains, g, sizeof(float) * ng, cudaMemcpyDeviceToHost, s));
    if (h_coefs) DFB_CUDA(cudaMemcpyAsync(h_coefs, cf, sizeof(float) * nc, cudaMemcpyDeviceToHost, s));
    if (h_lsnr) DFB_CUDA(cudaMemcpyAsync(h_lsnr, l, sizeof(float) * rows, cudaMemcpyDeviceToHost, s));
    if (h_stage) DFB_CUDA(cudaMemcpyAsync(h_stage, sg, rows, cudaMemcpyDeviceToHost, s));
    DFB_CUDA(cudaStreamSynchronize(s));
    if (flush) slots_close_all(h);
    return DFB_OK;
}

// debug aid: the state-slab rows k_slot_rows wrote at the handle's last call (moved or started fresh)
extern "C" int dfb_debug_stream_rows_moved(const dfb_stream *h, int64_t *n) {
    if (!h || !n) return fail(DFB_ERR_INVALID, "null argument");
    *n = h->rows_moved;
    return DFB_OK;
}

// ---- debug aids of the spectral input kernel (tests): the analysis with its ERB epilogue, and k_spec_ingest on its own.
// Both run the row-table kernels the streaming executor runs, the table on the device until the launch has run.
static int with_rows(const std::vector<RaggedRow> &rows, cudaStream_t s, const std::function<int(const RaggedRow *)> &launch) {
    RaggedRow *d_rows = nullptr;
    DFB_CUDA(cudaMalloc(&d_rows, sizeof(RaggedRow) * rows.size()));
    const int rc = cudaMemcpyAsync(d_rows, rows.data(), sizeof(RaggedRow) * rows.size(), cudaMemcpyHostToDevice, s) == cudaSuccess
                       ? launch(d_rows)
                       : fail(DFB_ERR_CUDA, "row table upload failed");
    cudaStreamSynchronize(s);
    cudaFree(d_rows);
    return rc;
}
extern "C" int dfb_debug_analysis_erb(dfb_state *st, const float *d_audio, int64_t C, int64_t T, float *d_spec, float *d_erb_db,
                                      void *stream) {
    if (!st || !d_audio || !d_spec || !d_erb_db || C <= 0 || C > 65535 || T <= 0) return fail(DFB_ERR_INVALID, "bad argument");
    if (st->fft != 960 || st->hop != 480) return fail(DFB_ERR_UNSUPPORTED, "fft_size 960 / hop_size 480 only");
    DFB_CUDA(cudaSetDevice(st->device));
    const int64_t Tf = T / st->hop;
    if (Tf <= 0 || Tf > INT32_MAX) return fail(DFB_ERR_INVALID, "bad frame count");
    std::vector<RaggedRow> rows((size_t)C);
    for (int64_t b = 0; b < C; b++) rows[(size_t)b] = RaggedRow{b * T, T, 0, 0, 0};
    cudaStream_t s = (cudaStream_t)stream;
    return with_rows(rows, s, [&](const RaggedRow *d_rows) {
        AnaWindow w{0, (int)Tf, 0, (int)Tf, d_rows};
        return launch_analysis(st, d_audio, C, T, d_spec, d_erb_db, s, nullptr, &w);
    });
}
extern "C" int dfb_debug_spec_ingest(dfb_state *st, const float *d_spec, int64_t n, const int64_t *h_src, const int64_t *h_len,
                                     int64_t nb, int nb_df, float *d_erb_db, float *d_bins, void *stream) {
    if (!st || !d_spec || !d_erb_db || !d_bins || n <= 0 || n > INT32_MAX || nb <= 0 || nb > 65535 || nb_df <= 0 ||
        nb_df > st->tb.F || (!h_src) != (!h_len))
        return fail(DFB_ERR_INVALID, "bad argument");
    if (st->fft != 960 || st->hop != 480) return fail(DFB_ERR_UNSUPPORTED, "fft_size 960 / hop_size 480 only");
    DFB_CUDA(cudaSetDevice(st->device));
    std::vector<RaggedRow> rows((size_t)nb);
    for (int64_t b = 0; b < nb; b++) {
        const int64_t src = h_src ? h_src[b] : b, len = h_len ? h_len[b] : n;
        if (src < 0 || len < 0) return fail(DFB_ERR_INVALID, "bad row %lld", (long long)b);
        rows[(size_t)b] = RaggedRow{src * n * st->tb.F, len, 0, 0, 0};
    }
    cudaStream_t s = (cudaStream_t)stream;
    return with_rows(rows, s, [&](const RaggedRow *d_rows) {
        return launch_spec_ingest(st, d_spec, d_rows, (int)nb, (int)n, d_bins, nb_df, nb_df, d_erb_db, 0, (int)n, s);
    });
}
