// dfb_dwpw.cuh -- shared pieces of the fused "depthwise (+pathway) -> 1x1 -> ReLU" kernels
// (FFMA version in dfb_model.cu, tensor-core version in dfb_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dfb {

constexpr int kCh = 64;  // conv_ch of every shipped model

// fp32 pair FMA: d = a * b + c on both halves of a packed pair, as two FFMAs (Hopper has no packed fp32 FMA; the
// packing moves are register renames and cost no instruction).
__device__ __forceinline__ unsigned long long f2_pack(float lo, float hi) {
    unsigned long long r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void f2_unpack(unsigned long long v, float &lo, float &hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ unsigned long long f2_fma(unsigned long long a, unsigned long long b, unsigned long long c) {
    float a0, a1, b0, b1, c0, c1;
    f2_unpack(a, a0, a1);
    f2_unpack(b, b0, b1);
    f2_unpack(c, c0, c1);
    return f2_pack(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}

enum DwMode { DW_S1 = 0, DW_S2 = 1, DW_T2 = 2 };
constexpr int kLdA = kCh + 4;  // padded row stride of the A tile (floats)

struct DwPwParams {
    const float *in;      // [B,T,Fin,64]
    const float *path;    // optional [B,T,Fin,64]
    const float *ps, *pb; // pathway scale / bias [64]
    const float *dw;      // [kt][3][64]
    const float *pw;      // [64][64]
    const float *bias;    // [64]
    float *out;           // [B,T,Fout,64] (may be null when only the BF16 planes are wanted)
    unsigned short *out_hi, *out_lo;  // optional BF16 hi / lo planes of `out` (same indexing): operand of a tensor-core consumer
    int64_t in_fs, path_fs, out_fs;  // frame strides (floats)
    int T, Fin, Fout, kt, NF, lookahead;
    int fo_magic;         // ceil(65536 / Fout): r / Fout == (r * fo_magic) >> 16 for r < 128 (tensor-core kernel)
    // fused ERB mask head (tensor-core kernel, last decoder block, kt = 1): m = sigmoid(conv0_out(conv0p(e0) + out))
    const float *mk_e0;   // [B,T,Fout,64] or null
    const float *mk_ps, *mk_pb;  // conv0p affine [64]
    const float *mk_w;    // conv0_out taps [3][64]
    const float *mk_bias; // [1]
    float *mk_out;        // m [B,T,Fout]
    // streaming slots (tensor-core kernel, kt = 2): first frame of each stream (stream_first) and the window's frame 0,
    // or null: the previous-frame tap reads padding before it
    const int64_t *first;
    int64_t w0;
};


// Depthwise taps of this thread's channel quad (zero padded to 3 x 3) and pathway affine.
struct DwTaps {
    float4 wd[9];
    float4 ps4, pb4;
};

__device__ __forceinline__ void dw_load_taps(const DwPwParams &p, int cq, DwTaps &tp) {
#pragma unroll
    for (int i = 0; i < 9; i++) tp.wd[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 9; i++)
        if (i >= (3 - p.kt) * 3) tp.wd[i] = *reinterpret_cast<const float4 *>(p.dw + (i - (3 - p.kt) * 3) * kCh + cq * 4);
    tp.ps4 = make_float4(0.f, 0.f, 0.f, 0.f);
    tp.pb4 = tp.ps4;
    if (p.path) {
        tp.ps4 = *reinterpret_cast<const float4 *>(p.ps + cq * 4);
        tp.pb4 = *reinterpret_cast<const float4 *>(p.pb + cq * 4);
    }
}

// A[(t, fo)][4 cq .. 4 cq + 3] of the prologue (see the kernel comment in dfb_model.cu)
template <int MODE>
__device__ __forceinline__ float4 dw_prologue(const DwPwParams &p, const DwTaps &tp, int b, int t, int fo, int cq) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int dt = 0; dt < 3; dt++) {
        if (dt < 3 - p.kt) continue;
        // causal: taps at t-(kt-1) .. t; p.lookahead shifts them forward (DeepFilterNet v1 pads (kt-1-la, la), modules.py:151-154)
        const int tq = t - (2 - dt) + p.lookahead;
        if (tq < 0 || tq >= p.T) continue;
#pragma unroll
        for (int df = 0; df < 3; df++) {
            int fi;
            float4 wv;
            if (MODE == DW_S1) { fi = fo + df - 1; wv = tp.wd[dt * 3 + df]; }
            else if (MODE == DW_S2) { fi = 2 * fo + df - 1; wv = tp.wd[dt * 3 + df]; }
            else {  // DW_T2: df enumerates the (at most two) contributing taps
                if (df == 2) continue;
                if ((fo & 1) == 0) { if (df == 1) continue; fi = fo >> 1; wv = tp.wd[dt * 3 + 1]; }
                else if (df == 0) { fi = fo >> 1; wv = tp.wd[dt * 3 + 2]; }
                else { fi = (fo >> 1) + 1; wv = tp.wd[dt * 3 + 0]; }
            }
            if (fi < 0 || fi >= p.Fin) continue;
            const int64_t o = ((int64_t)b * p.T + tq);
            float4 x = *reinterpret_cast<const float4 *>(p.in + o * p.in_fs + fi * kCh + cq * 4);
            if (p.path) {
                float4 e = *reinterpret_cast<const float4 *>(p.path + o * p.path_fs + fi * kCh + cq * 4);
                x.x += fmaxf(e.x * tp.ps4.x + tp.pb4.x, 0.f);
                x.y += fmaxf(e.y * tp.ps4.y + tp.pb4.y, 0.f);
                x.z += fmaxf(e.z * tp.ps4.z + tp.pb4.z, 0.f);
                x.w += fmaxf(e.w * tp.ps4.w + tp.pb4.w, 0.f);
            }
            acc.x += x.x * wv.x; acc.y += x.y * wv.y; acc.z += x.z * wv.z; acc.w += x.w * wv.w;
        }
    }
    return acc;
}

}  // namespace dfb
