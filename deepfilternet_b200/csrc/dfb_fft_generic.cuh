// dfb_fft_generic.cuh -- fp32 real FFT of any length 2 <= N <= 8192 for the STFT / ISTFT kernels of DSP states other
// than fft 960 / hop 480 (sm_90a).
//
// Same transform as dfb_fft.cuh (the unnormalised real DFT of realfft / rustfft and its inverse), built from a per-state
// plan instead of compile-time sizes:
//   even N: M = N / 2-point complex transform of z[n] = x[2n] + i x[2n+1], then the split step (rfft_split) for the
//           forward and the merge step (irfft_merge) before the inverse;
//   odd N:  M = N-point complex transform of the real input (imaginary parts zero), the upper half by symmetry.
// The M-point transform is a Stockham autosort FFT (natural order in and out, ping-pong between two buffers): stage s
// of radix R with Ns = R_0 ... R_{s-1} reads butterfly j from src[j + r M / R], twiddles it by w_{Ns R}^{r (j mod Ns)},
// runs a DFT of length R and writes dst[(j - j mod Ns) R + j mod Ns + r Ns].  Radix 2, 3, 4, 5 and 7 butterflies are
// hard-coded (in registers, literal constants); any other prime factor p runs as a direct length-p DFT out of the
// source buffer, for correctness only (O(M p) per stage, no Bluestein).
//
// Twiddles: one table tw[k] = e^{-2 pi i k / N}, k in [0, N), computed in double and rounded to fp32; w_M^x = tw[x N / M]
// and the split / merge twiddles w_N^k are entries of the same table.
//
// The butterflies and the host plan are __host__ __device__ / host code so that tests/host/fft_generic_host_test.cu can
// run the stages sequentially on the CPU and check the index algebra against a double-precision DFT.
#pragma once
#include <cmath>
#include <vector>

#include "dfb_fft.cuh"

namespace dfb {

constexpr int kGenMaxN = 8192;      // largest fft_size of a DSP state
constexpr int kGenMaxStages = 16;   // M <= 8192 has at most 13 prime factors

// Plan of one fft_size (device copy inside the DSP state; tw points to device memory there).
struct GenFftPlan {
    int N, M, nst;
    int rad[kGenMaxStages];   // radix of stage 0, 1, ...
    const float2 *tw;         // [N] e^{-2 pi i k / N}
};

// Host: factorisation of M (fours first, then twos, threes, fives, sevens, then the remaining primes ascending) and the
// twiddle table.  Returns false when N is outside [2, kGenMaxN].
inline bool gen_fft_plan(int N, GenFftPlan &pl, std::vector<float2> &tw) {
    if (N < 2 || N > kGenMaxN) return false;
    pl.N = N;
    pl.M = (N % 2 == 0) ? N / 2 : N;
    pl.nst = 0;
    int m = pl.M;
    for (int p : {4, 2, 3, 5, 7})
        while (m % p == 0) { pl.rad[pl.nst++] = p; m /= p; }
    for (int p = 11; m > 1; p += 2)
        while (m % p == 0) { pl.rad[pl.nst++] = p; m /= p; }
    tw.resize(N);
    for (int k = 0; k < N; k++) {
        const double a = 2.0 * kPi * (double)k / (double)N;
        tw[k] = make_float2((float)cos(a), (float)-sin(a));
    }
    pl.tw = nullptr;
    return true;
}

// Length-7 DFT in registers: X[q] = v0 + sum_m cos(2 pi m q / 7) (v_m + v_{7-m}) -+ i sum_m sin(2 pi m q / 7) (v_m - v_{7-m})
template <bool INV>
struct Dft<7, INV> {
    static DFB_HD void run(float2 (&v)[7]) {
        constexpr float c1 = float(cx_cos2pi(1, 7)), c2 = float(cx_cos2pi(2, 7)), c3 = float(cx_cos2pi(3, 7));
        constexpr float s1 = float(cx_sin2pi(1, 7)), s2 = float(cx_sin2pi(2, 7)), s3 = float(cx_sin2pi(3, 7));
        const float2 a1 = cadd(v[1], v[6]), a2 = cadd(v[2], v[5]), a3 = cadd(v[3], v[4]);
        const float2 d1 = csub(v[1], v[6]), d2 = csub(v[2], v[5]), d3 = csub(v[3], v[4]);
        const float2 x0 = v[0];
        auto p = [&](float ca, float cb, float cc) {
            return make_float2(x0.x + ca * a1.x + cb * a2.x + cc * a3.x, x0.y + ca * a1.y + cb * a2.y + cc * a3.y);
        };
        auto q = [&](float sa, float sb, float sc) {
            return cmul_mi<INV>(make_float2(sa * d1.x + sb * d2.x + sc * d3.x, sa * d1.y + sb * d2.y + sc * d3.y));
        };
        // cos(2 pi m q / 7) and sin(2 pi m q / 7) for q = 1, 2, 3 (m q reduced mod 7, sin odd)
        const float2 p1 = p(c1, c2, c3), q1 = q(s1, s2, s3);
        const float2 p2 = p(c2, c3, c1), q2 = q(s2, -s3, -s1);
        const float2 p3 = p(c3, c1, c2), q3 = q(s3, -s1, s2);
        v[0] = cadd(x0, cadd(a1, cadd(a2, a3)));
        v[1] = cadd(p1, q1); v[6] = csub(p1, q1);
        v[2] = cadd(p2, q2); v[5] = csub(p2, q2);
        v[3] = cadd(p3, q3); v[4] = csub(p3, q3);
    }
};

DFB_HD float2 gen_tw(const float2 *tw, int idx, bool inv) {
#ifdef __CUDA_ARCH__
    const float2 w = __ldg(tw + idx);
#else
    const float2 w = tw[idx];
#endif
    return inv ? cconj(w) : w;
}

// One radix-R butterfly (R in {2, 3, 4, 5, 7}) of a Stockham stage: j in [0, M / R), Ns = product of the earlier radices,
// ts = N / M (twiddle table stride).
template <int R, bool INV>
DFB_HD void gen_bfly(const float2 *src, float2 *dst, int M, int Ns, int j, const float2 *tw, int ts) {
    const int k = j % Ns, stride = M / R;
    float2 v[R];
#pragma unroll
    for (int r = 0; r < R; r++) v[r] = src[j + r * stride];
    if (k != 0) {
        const int step = k * (M / (Ns * R)) * ts;   // w_{Ns R}^{r k} = tw[r step]
#pragma unroll
        for (int r = 1; r < R; r++) v[r] = cmul(v[r], gen_tw(tw, r * step, INV));
    }
    Dft<R, INV>::run(v);
    const int base = (j - k) * R + k;
#pragma unroll
    for (int r = 0; r < R; r++) dst[base + r * Ns] = v[r];
}

// The same for any radix R as a direct DFT: dst[base + q Ns] = sum_r src[j + r M / R] w_{Ns R}^{r (k + q Ns)}.
template <bool INV>
DFB_HD void gen_bfly_any(const float2 *src, float2 *dst, int M, int Ns, int R, int j, const float2 *tw, int ts) {
    const int k = j % Ns, stride = M / R, L = Ns * R, unit = (M / L) * ts;
    const int base = (j - k) * R + k;
    for (int q = 0; q < R; q++) {
        const int e = k + q * Ns;
        float2 acc = src[j];
        int idx = e;   // (r e) mod L
        for (int r = 1; r < R; r++) {
            acc = cadd(acc, cmul(src[j + r * stride], gen_tw(tw, idx * unit, INV)));
            idx += e;
            if (idx >= L) idx -= L;
        }
        dst[base + q * Ns] = acc;
    }
}

// Radix dispatch of butterfly j of a stage.
template <bool INV>
DFB_HD void gen_stage_bfly(const float2 *src, float2 *dst, int M, int Ns, int R, int j, const float2 *tw, int ts) {
    switch (R) {
        case 2: gen_bfly<2, INV>(src, dst, M, Ns, j, tw, ts); break;
        case 3: gen_bfly<3, INV>(src, dst, M, Ns, j, tw, ts); break;
        case 4: gen_bfly<4, INV>(src, dst, M, Ns, j, tw, ts); break;
        case 5: gen_bfly<5, INV>(src, dst, M, Ns, j, tw, ts); break;
        case 7: gen_bfly<7, INV>(src, dst, M, Ns, j, tw, ts); break;
        default: gen_bfly_any<INV>(src, dst, M, Ns, R, j, tw, ts); break;
    }
}

#ifdef __CUDACC__
// Block-wide transforms of several frames at once (the generic STFT / ISTFT kernels of dfb_dsp.cu, the STOI STFT of
// dfb_metrics.cu).
// The stage radices go to shared memory (a dynamically indexed kernel-parameter array would be copied to local memory).
__device__ __forceinline__ void gen_load_radices(const GenFftPlan &pl, int *s_rad) {
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < kGenMaxStages; i++) s_rad[i] = pl.rad[i];
    }
}

// M-point complex FFT of the first nf frames (frame f at a + f M), with b as the second buffer; returns the buffer that
// holds the result.  Every thread of the CTA takes part; ends with a barrier.
template <bool INV>
__device__ __forceinline__ float2 *gen_block_fft(float2 *a, float2 *b, const GenFftPlan &pl, const int *s_rad, int nf) {
    const int M = pl.M, ts = pl.N / pl.M;
    int Ns = 1;
    for (int s = 0; s < pl.nst; s++) {
        const int R = s_rad[s], nb = M / R, total = nf * nb;
#define DFB_GEN_STAGE(CALL)                                                   \
    for (int i = threadIdx.x; i < total; i += blockDim.x) {                   \
        const int f = i / nb, j = i - f * nb;                                 \
        CALL;                                                                 \
    }
        switch (R) {
            case 2: DFB_GEN_STAGE((gen_bfly<2, INV>(a + f * M, b + f * M, M, Ns, j, pl.tw, ts))) break;
            case 3: DFB_GEN_STAGE((gen_bfly<3, INV>(a + f * M, b + f * M, M, Ns, j, pl.tw, ts))) break;
            case 4: DFB_GEN_STAGE((gen_bfly<4, INV>(a + f * M, b + f * M, M, Ns, j, pl.tw, ts))) break;
            case 5: DFB_GEN_STAGE((gen_bfly<5, INV>(a + f * M, b + f * M, M, Ns, j, pl.tw, ts))) break;
            case 7: DFB_GEN_STAGE((gen_bfly<7, INV>(a + f * M, b + f * M, M, Ns, j, pl.tw, ts))) break;
            default: DFB_GEN_STAGE((gen_bfly_any<INV>(a + f * M, b + f * M, M, Ns, R, j, pl.tw, ts))) break;
        }
#undef DFB_GEN_STAGE
        __syncthreads();
        float2 *t = a; a = b; b = t;
        Ns *= R;
    }
    return a;
}
#endif

}  // namespace dfb
