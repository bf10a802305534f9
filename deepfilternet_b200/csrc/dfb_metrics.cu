// dfb_metrics.cu -- batched speech-quality metrics of a ragged batch (dfb_metrics* in include/dfb200.h; DESIGN.md section 5j):
// SI-SDR (DeepFilterNet/df/evaluation_utils.py si_sdr_speechmetrics), STOI (df/stoi.py stoi, after io.resample to 10 kHz)
// segmental SNR (df/sepm.py SNRseg, after io.resample to 16 kHz), and the two spectral distances of df/sepm.py's composite
// measure on the same 16 kHz rows: LLR (sepm.llr) and WSS (sepm.wss); and pystoi's STOI and extended STOI on the 10 kHz rows
// (pystoi.stoi(x, y, 10000, extended), which df/evaluation_utils.py stoi reports; section 5n).
//
// One call is a fixed sequence of launches, with no host round trip between them:
//   k_resample_rows (dfb_dsp.cu)  clean and degraded rows -> 10 kHz / 16 kHz, one launch per signal
//   k_stoi_energy                 one warp per 256-sample frame: the frame's energy in dB
//   k_stoi_mask                   one CTA per entry: the entry's loudest frame, the 40 dB mask, the prefix count of kept
//                                 frames (their index list), the compacted and STFT lengths
//   k_stoi_stft                   four STFT frames of both signals per CTA, their samples computed from the kept-frame list
//                                 (never materialised): the 15 third-octave band magnitudes
//   k_stoi_seg                    one warp per 30-frame segment: the sum over bands of the clipped, normalised correlations
//   k_ssnr                        one warp per 480-sample frame at 16 kHz: the clipped segmental SNR (fp64)
//   k_llr                         one warp per 480-sample frame at 16 kHz: the log-likelihood ratio of the order-16 LPC
//                                 models of both signals (fp64)
//   k_wss                         one CTA per 480-sample frame at 16 kHz: a 1024-point fp64 FFT of both signals, the 25
//                                 critical-band energies and Klatt's weighted spectral slope distance (fp64)
//   k_pystoi_energy               one warp per pystoi frame (256 samples at hop 128, unpadded): its energy in dB (fp64)
//   k_stoi_mask<true>             one CTA per entry: the same mask and prefix count on those energies, pystoi's counts
//   k_pystoi_stft                 one CTA per STFT frame: its samples from at most two kept frames, one fp64 512-point FFT
//                                 of both signals, the 15 band magnitudes of each (fp64)
//   k_pystoi_seg                  one warp per 30-frame segment: its STOI sum and its ESTOI sum (fp64)
//   k_sisdr                       one CTA per 4096-sample chunk: fp64 sums r.r, r.e, e.e
//   k_metrics_final               one CTA per entry: the per-entry means / SI-SDR from the frame, segment and chunk values,
//                                 LLR / WSS as the mean of the round(0.95 T) smallest frame values (a radix select), and
//                                 pystoi's STOI / ESTOI as segment means
// Every per-entry sum runs in an order fixed relative to the entry's start (per-thread strided sums, then a fixed shuffle
// and shared-memory tree), with no atomics, so an entry's results are the same bits wherever and with whatever it is batched.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <type_traits>
#include <vector>

#include "dfb_common.cuh"

namespace dfb {
namespace {

constexpr int kStoiFs = 10000, kSsnrFs = 16000;
constexpr int kStoiFrame = 256, kStoiHop = 128, kStoiFft = 512, kStoiBands = 15, kStoiSeg = 30;
constexpr int kSsnrWin = 480, kSsnrHop = 120;            // round(0.03 fs), floor(0.25 * 0.03 fs) at 16 kHz
constexpr int kSisdrChunk = 4096;
constexpr int kLpcOrder = 16;                            // sepm.llr's P at fs >= 10 kHz
constexpr int kWssFft = 1024, kWssBins = 512, kWssBands = 25;   // 2^ceil(log2(2 * 480)); bins 0 .. 511 (the last is dropped)
constexpr int kMaxCritTaps = 1024;                       // nonzero critical-band filter weights (about 600 are used)
constexpr int kStftFrames = 4;                           // STFT frames per CTA of k_stoi_stft (two signals each)
constexpr float kEps64f = 2.220446049250313e-16f;        // np.finfo(float).eps, as df/stoi.py adds it to float32 tensors
constexpr double kEps64 = 2.220446049250313e-16;         // np.finfo(np.float64).eps (sepm.SNRseg)
constexpr double kEps32 = 1.1920928955078125e-07;        // np.finfo(np.float32).eps (si_sdr_speechmetrics on float32)

__constant__ float c_w256[kStoiFrame];   // torch.hann_window(258, periodic=False)[1:-1]
__constant__ double c_w256d[kStoiFrame]; // np.hanning(258)[1:-1] (pystoi), fp64
__constant__ double c_wss[kSsnrWin];     // SNRseg's hannWin: 0.5 (1 - cos(2 pi n / 481)), n = 1 .. 480
__constant__ double c_crit[kMaxCritTaps]; // critical-band filter weights of band i at bins [crit_lo[i], crit_lo[i] + crit_n[i])
__constant__ int c_crit_lo[kWssBands], c_crit_n[kWssBands], c_crit_off[kWssBands];

// One entry of a call, planned on the host.
struct MetEntry {
    int64_t in_off, len;    // clean / degraded samples at the call's rate
    int64_t o10, t10;       // its 10 kHz rows at x10 / y10 + o10
    int64_t o16, t16;       // its 16 kHz rows at x16 / y16 + o16
    int64_t fo;             // first STOI frame: energies en[fo ..], kept list kidx[fo ..], segments seg[fo ..], bands at 15 fo
    int64_t so;             // first SSNR frame value
    int64_t co;             // first SI-SDR chunk
    int64_t cf;             // first LLR / WSS frame value
    int nfr, pad_front, pad_end, nfs, nch;
    int nct, kct;           // LLR / WSS frames T = (t16 - 480) / 120 (0 when t16 < 480) and k = round(0.95 T)
    int pnf;                // pystoi frames F = ceil((t10 - 256) / 128) (0 when t10 <= 256)
    int64_t po;             // first pystoi frame: energies pen[po ..], kept list pkidx[po ..], segments at po, bands at 15 po
};
// What the device finds out about an entry's STOI (dfb_debug_metrics_counts reads it back) or, for pystoi, its kept
// frames K, silence-free length lc and STFT frames nf = K - 1 (dfb_debug_metrics_pystoi).
struct MetState { int nk, s0, lc, nf; };
struct StoiBands { int lo[kStoiBands], hi[kStoiBands]; float inv_wsum; };

struct MetBufs {
    const float *x10, *y10, *x16, *y16, *clean, *degraded;
    float *en, *bx, *by, *seg;
    int *kidx;
    double *ss;
    double *ch;   // [3][chunks]
    double *llr, *wss;   // per-frame distortions at cf
    const double2 *fft_tw;   // e^(-2 pi i m / 1024), m = 0 .. 1023
    MetState *st;
    int64_t n_fr, n_ch;
    double *pen, *pbx, *pby, *pseg;   // pystoi: frame energies, band magnitudes [15][F], segment sums [2][n_pf] at po
    int *pkidx;
    MetState *pst;
    int64_t n_pf;
};

// ---- deterministic reductions ----
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// Sum over the CTA (blockDim.x a multiple of 32, <= 1024); every thread gets the result.  A fixed tree.
template <typename T>
__device__ T block_sum(T v, T *sm) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) sm[w] = v;
    __syncthreads();
    T r = lane < nw ? sm[lane] : T(0);
    r = warp_sum(r);
    return r;
}

__device__ __forceinline__ float xat(const float *x, int64_t n, int64_t p) { return p >= 0 && p < n ? __ldg(x + p) : 0.f; }

// grid (ceil(max nfr / 8), B), 256 threads: warp w of CTA x is frame 8 x + w of entry blockIdx.y.  Frame i is samples
// [128 i, 128 i + 256) of the clean 10 kHz row padded by pad_front zeros in front, times the window:
// en = 20 log10(|frame| / sqrt(256) + eps).
__global__ void __launch_bounds__(256) k_stoi_energy(const MetEntry *__restrict__ ents, MetBufs b) {
    const MetEntry e = ents[blockIdx.y];
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= e.nfr) return;
    const float *x = b.x10 + e.o10;
    const int64_t p0 = (int64_t)i * kStoiHop - e.pad_front;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < kStoiFrame / 32; k++) {
        const int n = lane + 32 * k;
        const float v = xat(x, e.t10, p0 + n) * c_w256[n];
        s = fmaf(v, v, s);
    }
    s = warp_sum(s);
    if (lane == 0) b.en[e.fo + i] = 20.f * log10f(sqrtf(s) / 16.f + kEps64f);
}

// grid B, 1024 threads: frame i is kept when (max_j en_j - 40) - en_i < 0 (df/stoi.py remove_silent_frames, in float32);
// kidx[fo + j] is the j-th kept frame.  The overlap-added kept frames have (nk - 1) 128 + 256 samples; the first pad_front
// are dropped when frame 0 is kept, the last pad_end when the last frame is kept.  STOI needs at least 512 samples.
// PY: pystoi's remove_silent_frames on the fp64 energies pen of its F unpadded frames, into pkidx / pst: nothing is
// trimmed, and the nk - 1 STFT frames of the (nk - 1) 128 + 256 samples are all used (an entry without a frame has none).
template <bool PY>
__global__ void __launch_bounds__(1024) k_stoi_mask(const MetEntry *__restrict__ ents, MetBufs b) {
    using T = typename std::conditional<PY, double, float>::type;
    __shared__ T s_red[32];
    __shared__ int s_cnt[33];
    const MetEntry e = ents[blockIdx.x];
    const int nfr = PY ? e.pnf : e.nfr;
    if (PY && nfr == 0) {
        if (threadIdx.x == 0) b.pst[blockIdx.x] = MetState{0, 0, 0, 0};
        return;
    }
    const T *en = PY ? (const T *)(b.pen + e.po) : (const T *)(b.en + e.fo);
    int *kidx = PY ? b.pkidx + e.po : b.kidx + e.fo;
    T mx = -INFINITY;
    for (int i = threadIdx.x; i < nfr; i += blockDim.x) mx = max(mx, en[i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (lane == 0) s_red[w] = mx;
    __syncthreads();
    mx = s_red[0];
    for (int k = 1; k < nw; k++) mx = max(mx, s_red[k]);
    const T thr = mx - T(40);
    int base = 0;
    for (int c0 = 0; c0 < nfr; c0 += blockDim.x) {
        const int i = c0 + threadIdx.x;
        const bool keep = i < nfr && (thr - en[i]) < T(0);
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        __syncthreads();   // s_cnt of the previous chunk is consumed
        if (lane == 0) s_cnt[w] = __popc(bal);
        __syncthreads();
        if (threadIdx.x == 0) {
            int a = 0;
            for (int k = 0; k < nw; k++) { const int c = s_cnt[k]; s_cnt[k] = a; a += c; }
            s_cnt[32] = a;
        }
        __syncthreads();
        if (keep) kidx[base + s_cnt[w] + __popc(bal & ((1u << lane) - 1u))] = i;
        base += s_cnt[32];
    }
    if (PY) {
        if (threadIdx.x == 0) b.pst[blockIdx.x] = MetState{base, 0, (base - 1) * kStoiHop + kStoiFrame, base - 1};
    } else if (threadIdx.x == 0) {
        const int nk = base;
        const bool first = (thr - en[0]) < 0.f, last = (thr - en[e.nfr - 1]) < 0.f;
        MetState s;
        s.nk = nk;
        s.s0 = first ? e.pad_front : 0;
        s.lc = (nk - 1) * kStoiHop + kStoiFrame - s.s0 - (last ? e.pad_end : 0);
        s.nf = s.lc >= kStoiFft ? 1 + (s.lc - kStoiFrame) / kStoiHop : 0;
        b.st[blockIdx.x] = s;
    }
}

// Sample s of the compacted signal (after the front trim s0): overlap-add of the kept frames that cover it, at most two at
// 50 % overlap, divided by the overlap-added window.
__device__ __forceinline__ void compact_at(const MetEntry &e, const MetState &st, const int *__restrict__ kidx, const float *x,
                                           const float *y, int64_t s, float &xv, float &yv) {
    const int64_t r = s + st.s0;
    const int64_t j1 = r >> 7;
    const int q = (int)(r & 127);
    float nx = 0.f, ny = 0.f, den = 0.f;
    if (j1 >= 1) {
        const int64_t p = (int64_t)__ldg(kidx + j1 - 1) * kStoiHop + q + kStoiHop - e.pad_front;
        const float w = c_w256[q + kStoiHop];
        nx = xat(x, e.t10, p) * w; ny = xat(y, e.t10, p) * w; den = w;
    }
    if (j1 < st.nk) {
        const int64_t p = (int64_t)__ldg(kidx + j1) * kStoiHop + q - e.pad_front;
        const float w = c_w256[q];
        nx += xat(x, e.t10, p) * w; ny += xat(y, e.t10, p) * w; den += w;
    }
    xv = nx / den;
    yv = ny / den;
}

// grid (ceil(max nfr / 4), B), 256 threads: STFT frames [4 x, 4 x + 4) of entry blockIdx.y (df/stoi.py _stft: the windowed
// 256 samples [128 f, 128 f + 256) of the compacted signal in a 512-point real FFT, / sum(window)), both signals: 8 real
// transforms as 256-point complex ones (dfb_fft_generic.cuh), then the band magnitudes sqrt(sum_band |X_k|^2) to
// bx / by [15 fo + band nfr + f].
__global__ void __launch_bounds__(256) k_stoi_stft(const MetEntry *__restrict__ ents, MetBufs b, GenFftPlan pl, StoiBands bands) {
    constexpr int M = kStoiFft / 2, NS = 2 * kStftFrames;
    __shared__ __align__(16) float2 A[NS * M], Bf[NS * M];
    __shared__ int s_rad[kGenMaxStages];
    const MetEntry e = ents[blockIdx.y];
    const MetState st = b.st[blockIdx.y];
    const int f0 = blockIdx.x * kStftFrames;
    if (f0 >= st.nf) return;
    const int nf = min(kStftFrames, st.nf - f0);
    gen_load_radices(pl, s_rad);
    const int *kidx = b.kidx + e.fo;
    const float *x = b.x10 + e.o10, *y = b.y10 + e.o10;
    for (int i = threadIdx.x; i < kStftFrames * kStoiFft; i += blockDim.x) {
        const int f = i / kStoiFft, n = i - f * kStoiFft;
        float xv = 0.f, yv = 0.f;
        if (f < nf && n < kStoiFrame) {
            compact_at(e, st, kidx, x, y, (int64_t)(f0 + f) * kStoiHop + n, xv, yv);
            xv *= c_w256[n];
            yv *= c_w256[n];
        }
        reinterpret_cast<float *>(A + (2 * f) * M)[n] = xv;
        reinterpret_cast<float *>(A + (2 * f + 1) * M)[n] = yv;
    }
    __syncthreads();
    float2 *Z = gen_block_fft<false>(A, Bf, pl, s_rad, NS);
    float *P = reinterpret_cast<float *>(Z == A ? Bf : A);   // |X_k|^2, bins [klo, khi) of each transform
    const int klo = bands.lo[0], khi = bands.hi[kStoiBands - 1], nk = khi - klo;
    for (int i = threadIdx.x; i < NS * nk; i += blockDim.x) {
        const int t = i / nk, k = klo + (i - t * nk);
        float2 xk, xnk;
        rfft_split(Z[t * M + k % M], Z[t * M + (M - k) % M], __ldg(pl.tw + k), xk, xnk);
        xk.x *= bands.inv_wsum; xk.y *= bands.inv_wsum;
        P[t * nk + (k - klo)] = xk.x * xk.x + xk.y * xk.y;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < NS * kStoiBands; i += blockDim.x) {
        const int t = i / kStoiBands, band = i - t * kStoiBands, f = t >> 1;
        if (f >= nf) continue;
        float acc = 0.f;
        for (int k = bands.lo[band]; k < bands.hi[band]; k++) acc += P[t * nk + (k - klo)];
        float *dst = (t & 1) ? b.by : b.bx;
        dst[kStoiBands * e.fo + (int64_t)band * e.nfr + f0 + f] = sqrtf(acc);
    }
}

// grid (ceil(max nfr / 8), B), 256 threads: warp w of CTA x is segment m = 8 x + w of entry blockIdx.y: frames [m, m + 30)
// (one segment of all L frames when L <= 30).  seg[fo + m] = sum over the bands of the correlation of the normalised,
// clipped, mean-free band envelopes (df/stoi.py stoi), lane l holding frame m + l.
__global__ void __launch_bounds__(256) k_stoi_seg(const MetEntry *__restrict__ ents, MetBufs b) {
    const MetEntry e = ents[blockIdx.y];
    const int L = b.st[blockIdx.y].nf;
    const int J = L > kStoiSeg ? L - kStoiSeg + 1 : 1, N = L > kStoiSeg ? kStoiSeg : L;
    const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (L == 0 || m >= J) return;
    const float c1 = 1.f + 5.62341325190349f;   // 1 + 10^(15 / 20), Beta = -15 dB
    const bool in = lane < N;
    float corr = 0.f;
    for (int band = 0; band < kStoiBands; band++) {
        const int64_t o = kStoiBands * e.fo + (int64_t)band * e.nfr + m + lane;
        const float xv = in ? b.bx[o] : 0.f, yv0 = in ? b.by[o] : 0.f;
        const float nrm = sqrtf(warp_sum(xv * xv)) / (sqrtf(warp_sum(yv0 * yv0)) + kEps64f);
        const float yv = in ? fminf(yv0 * nrm, xv * c1) : 0.f;
        const float xm = warp_sum(xv) / (float)N, ym = warp_sum(yv) / (float)N;
        const float xd = in ? xv - xm : 0.f, yd = in ? yv - ym : 0.f;
        const float xn = xd / (sqrtf(warp_sum(xd * xd)) + kEps64f), yn = yd / (sqrtf(warp_sum(yd * yd)) + kEps64f);
        corr += warp_sum(xn * yn);
    }
    if (lane == 0) b.seg[e.fo + m] = corr;
}

__device__ __forceinline__ double2 cmul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// ---- pystoi (0.4.1) on the 10 kHz rows, fp64 throughout as numpy computes it: frame i is samples [128 i, 128 i + 256)
// of the unpadded row times np.hanning(258)[1:-1], i < F = ceil((t10 - 256) / 128) ----

// grid (ceil(max F / 8), B), 256 threads: warp w of CTA x is frame i = 8 x + w of entry blockIdx.y:
// pen[po + i] = 20 log10(|frame| + eps).
__global__ void __launch_bounds__(256) k_pystoi_energy(const MetEntry *__restrict__ ents, MetBufs b) {
    const MetEntry e = ents[blockIdx.y];
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= e.pnf) return;
    const float *x = b.x10 + e.o10 + (int64_t)i * kStoiHop;
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < kStoiFrame / 32; k++) {
        const int n = lane + 32 * k;
        const double v = c_w256d[n] * (double)__ldg(x + n);
        s = fma(v, v, s);
    }
    s = warp_sum(s);
    if (lane == 0) b.pen[e.po + i] = 20.0 * log10(sqrt(s) + kEps64);
}

// In-place 512-point complex FFT of z (shared) by the CTA's 128 threads: four Stockham radix-4 stages, then one radix-2
// stage; tw[m] = e^(-2 pi i m / 1024) (the WSS table, every second entry).
__device__ __forceinline__ void fft512(double2 *z, const double2 *__restrict__ tw) {
    constexpr int N = kStoiFft, TS = kWssFft / kStoiFft;
    const int j = threadIdx.x;
#pragma unroll 1
    for (int ns = 1; ns * 4 <= N; ns *= 4) {
        const int jm = j & (ns - 1), step = N / (4 * ns);
        double2 v[4];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            v[r] = z[j + r * (N / 4)];
            if (r) v[r] = cmul(v[r], __ldg(tw + TS * r * jm * step));
        }
        const double2 a0 = make_double2(v[0].x + v[2].x, v[0].y + v[2].y), a1 = make_double2(v[0].x - v[2].x, v[0].y - v[2].y);
        const double2 a2 = make_double2(v[1].x + v[3].x, v[1].y + v[3].y), a3 = make_double2(v[1].x - v[3].x, v[1].y - v[3].y);
        const int d = (j - jm) * 4 + jm;
        __syncthreads();
        z[d] = make_double2(a0.x + a2.x, a0.y + a2.y);
        z[d + ns] = make_double2(a1.x + a3.y, a1.y - a3.x);          // a1 - i a3
        z[d + 2 * ns] = make_double2(a0.x - a2.x, a0.y - a2.y);
        z[d + 3 * ns] = make_double2(a1.x - a3.y, a1.y + a3.x);      // a1 + i a3
        __syncthreads();
    }
    // last stage, ns = 256: z[k] = v0 + w^k v1, z[k + 256] = v0 - w^k v1
    double2 v0[2], v1[2];
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const int k = j + r * (N / 4);
        v0[r] = z[k];
        v1[r] = cmul(z[k + N / 2], __ldg(tw + TS * k));
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 2; r++) {
        const int k = j + r * (N / 4);
        z[k] = make_double2(v0[r].x + v1[r].x, v0[r].y + v1[r].y);
        z[k + N / 2] = make_double2(v0[r].x - v1[r].x, v0[r].y - v1[r].y);
    }
    __syncthreads();
}

// grid (max F, B), 128 threads: STFT frame f = blockIdx.x < nf of entry blockIdx.y.  Sample s = 128 f + n of the
// silence-free signal is the overlap-add (no division) of the windowed kept frames j1 - 1 and j1 = s / 128 that cover
// it; the frame is that times the window again, both signals as one complex 512-point FFT (clean real, degraded
// imaginary), and pbx / pby [15 po + band F + f] = sqrt(sum over the band's bins of |X_k|^2).
__global__ void __launch_bounds__(128) k_pystoi_stft(const MetEntry *__restrict__ ents, MetBufs b, StoiBands bands) {
    __shared__ double2 z[kStoiFft];
    const MetEntry e = ents[blockIdx.y];
    const int f = blockIdx.x, nk = b.pst[blockIdx.y].nk;
    if (f >= nk - 1) return;
    const int *kidx = b.pkidx + e.po;
    const float *x = b.x10 + e.o10, *y = b.y10 + e.o10;
    for (int n = threadIdx.x; n < kStoiFft; n += blockDim.x) {
        double2 v = make_double2(0.0, 0.0);
        if (n < kStoiFrame) {
            const int j1 = f + (n >> 7), q = n & 127;
            const int64_t pa = (int64_t)__ldg(kidx + j1) * kStoiHop + q;   // j1 <= nk - 1: kept frame j1, first half
            double xs = c_w256d[q] * (double)__ldg(x + pa), ys = c_w256d[q] * (double)__ldg(y + pa);
            if (j1 >= 1) {   // kept frame j1 - 1, second half
                const int64_t pb = (int64_t)__ldg(kidx + j1 - 1) * kStoiHop + q + kStoiHop;
                xs += c_w256d[q + kStoiHop] * (double)__ldg(x + pb);
                ys += c_w256d[q + kStoiHop] * (double)__ldg(y + pb);
            }
            v.x = c_w256d[n] * xs;
            v.y = c_w256d[n] * ys;
        }
        z[n] = v;
    }
    __syncthreads();
    fft512(z, b.fft_tw);
    if (threadIdx.x >= 2 * kStoiBands) return;
    const int band = threadIdx.x % kStoiBands, sig = threadIdx.x / kStoiBands;
    double acc = 0.0;
    for (int k = bands.lo[band]; k < bands.hi[band]; k++) {
        const double2 zk = z[k], zn = z[(kStoiFft - k) & (kStoiFft - 1)];
        // X_k = (Z_k + conj Z_-k) / 2, Y_k = (Z_k - conj Z_-k) / 2i
        const double re = sig ? 0.5 * (zk.y + zn.y) : 0.5 * (zk.x + zn.x);
        const double im = sig ? 0.5 * (zn.x - zk.x) : 0.5 * (zk.y - zn.y);
        acc += re * re + im * im;
    }
    (sig ? b.pby : b.pbx)[kStoiBands * e.po + (int64_t)band * e.pnf + f] = sqrt(acc);
}

// grid (ceil(max F / 8), B), 256 threads: warp w of CTA x is segment m = 8 x + w < J = nf - 29 of entry blockIdx.y,
// frames [m, m + 30), lane l < 30 holding frame m + l of all 15 bands of both signals.
// pseg[po + m] = STOI's sum over the bands of the correlation of the scaled, clipped, centred and normalised rows;
// pseg[n_pf + po + m] = ESTOI's sum of x_n y_n / 30 over the segment, the rows then the columns of both 15 x 30 matrices
// centred and normalised (a centred row or column of norm 0 normalises to 0).
__global__ void __launch_bounds__(256) k_pystoi_seg(const MetEntry *__restrict__ ents, MetBufs b) {
    const MetEntry e = ents[blockIdx.y];
    const int J = b.pst[blockIdx.y].nf - kStoiSeg + 1;
    const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (m >= J) return;
    const double c1 = 1.0 + 5.623413251903491;   // 1 + 10^(15 / 20)
    const bool in = lane < kStoiSeg;
    const double inv_n = 1.0 / kStoiSeg;
    double xr[kStoiBands], yr[kStoiBands];
    double corr = 0.0;
#pragma unroll
    for (int band = 0; band < kStoiBands; band++) {
        const int64_t o = kStoiBands * e.po + (int64_t)band * e.pnf + m + lane;
        const double xv = in ? b.pbx[o] : 0.0, yv0 = in ? b.pby[o] : 0.0;
        // STOI
        const double nrm = sqrt(warp_sum(xv * xv)) / (sqrt(warp_sum(yv0 * yv0)) + kEps64);
        const double yv = in ? fmin(yv0 * nrm, xv * c1) : 0.0;
        const double xm = warp_sum(xv) / kStoiSeg, ym = warp_sum(yv) / kStoiSeg;
        const double xd = in ? xv - xm : 0.0, yd = in ? yv - ym : 0.0;
        const double xn = xd / (sqrt(warp_sum(xd * xd)) + kEps64), yn = yd / (sqrt(warp_sum(yd * yd)) + kEps64);
        corr += warp_sum(xn * yn);
        // ESTOI: the band's row centred and normalised
        const double ym0 = warp_sum(yv0) / kStoiSeg;   // every lane shuffles: outside the conditionals
        const double xc = in ? xv - xm : 0.0, yc = in ? yv0 - ym0 : 0.0;
        const double nx = sqrt(warp_sum(xc * xc)), ny = sqrt(warp_sum(yc * yc));
        xr[band] = nx > 0.0 ? xc / nx : 0.0;
        yr[band] = ny > 0.0 ? yc / ny : 0.0;
    }
    // ESTOI: this lane's column centred and normalised
    double sx = 0.0, sy = 0.0;
#pragma unroll
    for (int band = 0; band < kStoiBands; band++) { sx += xr[band]; sy += yr[band]; }
    sx /= kStoiBands;
    sy /= kStoiBands;
    double qx = 0.0, qy = 0.0;
#pragma unroll
    for (int band = 0; band < kStoiBands; band++) {
        xr[band] -= sx; yr[band] -= sy;
        qx = fma(xr[band], xr[band], qx);
        qy = fma(yr[band], yr[band], qy);
    }
    qx = sqrt(qx);
    qy = sqrt(qy);
    double es = 0.0;
#pragma unroll
    for (int band = 0; band < kStoiBands; band++) {
        const double xn = qx > 0.0 ? xr[band] / qx : 0.0, yn = qy > 0.0 ? yr[band] / qy : 0.0;
        es += xn * yn * inv_n;
    }
    es = warp_sum(in ? es : 0.0);
    if (lane == 0) {
        b.pseg[e.po + m] = corr;
        b.pseg[b.n_pf + e.po + m] = es;
    }
}

// grid (ceil(max nfs / 8), B), 256 threads: warp w of CTA x is SSNR frame i = 8 x + w (samples [120 i, 120 i + 480) at 16 kHz)
// of entry blockIdx.y; the last frame is not computed (SNRseg drops it).  fp64, as SNRseg computes.
__global__ void __launch_bounds__(256) k_ssnr(const MetEntry *__restrict__ ents, MetBufs b) {
    const MetEntry e = ents[blockIdx.y];
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= e.nfs - 1) return;
    const float *c = b.x16 + e.o16 + (int64_t)i * kSsnrHop, *d = b.y16 + e.o16 + (int64_t)i * kSsnrHop;
    double sig = 0.0, noi = 0.0;
    for (int n = lane; n < kSsnrWin; n += 32) {
        const double w = c_wss[n], cw = w * (double)__ldg(c + n), dw = w * (double)__ldg(d + n);
        sig = fma(cw, cw, sig);
        noi = fma(cw - dw, cw - dw, noi);
    }
    sig = warp_sum(sig);
    noi = warp_sum(noi);
    if (lane == 0) {
        double v = 10.0 * log10(sig / (noi + kEps64) + kEps64);
        b.ss[e.so + i] = v < -10.0 ? -10.0 : (v > 35.0 ? 35.0 : v);
    }
}

// ---- df/sepm.py's composite measure: LLR and WSS on the 16 kHz rows (frame i: samples [120 i, 120 i + 480)) ----

// sepm.lpcoeff's Levinson-Durbin on the fp64 lags r (the error floored at eps), returned as the reference returns it:
// A = [1, -a_1 .. -a_16] in float32.  Fully unrolled, so every array stays in registers.
__device__ __forceinline__ void levinson(const double (&r)[kLpcOrder + 1], float (&A)[kLpcOrder + 1]) {
    double a[kLpcOrder];
    double E = r[0];
#pragma unroll
    for (int i = 0; i < kLpcOrder; i++) {
        double sum = 0.0;
#pragma unroll
        for (int j = 0; j < i; j++) sum += a[j] * r[i - j];
        const double k = (r[i + 1] - sum) / fmax(E, kEps64);
        double na[kLpcOrder];
#pragma unroll
        for (int j = 0; j < i; j++) na[j] = a[j] - k * a[i - 1 - j];
#pragma unroll
        for (int j = 0; j < i; j++) a[j] = na[j];
        a[i] = k;
        E = (1.0 - k * k) * E;
    }
    A[0] = 1.f;
#pragma unroll
    for (int j = 0; j < kLpcOrder; j++) A[j + 1] = (float)(-a[j]);
}

// A' toeplitz(R) A in fp64 from float32 operands.
__device__ __forceinline__ double toeplitz_form(const float (&A)[kLpcOrder + 1], const float (&R)[kLpcOrder + 1]) {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i <= kLpcOrder; i++) {
        double v = 0.0;
#pragma unroll
        for (int j = 0; j <= kLpcOrder; j++) v = fma((double)R[i > j ? i - j : j - i], (double)A[j], v);
        s = fma((double)A[i], v, s);
    }
    return s;
}

// grid (ceil(max T / 4), B), 128 threads: warp w of CTA x is frame i = 4 x + w of entry blockIdx.y.  sepm.llr at 16 kHz:
// the autocorrelation lags 0 .. 16 of each windowed frame (w_n x_n in fp64), its LPC model, then
// llr[cf + i] = ln(A_d' toeplitz(R_c) A_d / (A_c' toeplitz(R_c) A_c + eps)), 1000 standing in for a ratio <= 0.
__global__ void __launch_bounds__(128) k_llr(const MetEntry *__restrict__ ents, MetBufs b) {
    constexpr int NP = kSsnrWin + kLpcOrder;   // the frame, then 16 zeros for the lags that run past it
    __shared__ double s_x[4][NP];
    const MetEntry e = ents[blockIdx.y];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * 4 + w;
    if (i >= e.nct) return;
    double *x = s_x[w];
    float A[2][kLpcOrder + 1], Rc[kLpcOrder + 1];
#pragma unroll
    for (int sig = 0; sig < 2; sig++) {
        const float *src = (sig ? b.y16 : b.x16) + e.o16 + (int64_t)i * kSsnrHop;
        __syncwarp();
        for (int n = lane; n < NP; n += 32) x[n] = n < kSsnrWin ? c_wss[n] * (double)__ldg(src + n) : 0.0;
        __syncwarp();
        double r[kLpcOrder + 1];
#pragma unroll
        for (int k = 0; k <= kLpcOrder; k++) r[k] = 0.0;
        for (int n = lane; n < kSsnrWin; n += 32) {
            const double xn = x[n];
#pragma unroll
            for (int k = 0; k <= kLpcOrder; k++) r[k] = fma(xn, x[n + k], r[k]);
        }
#pragma unroll
        for (int k = 0; k <= kLpcOrder; k++) r[k] = warp_sum(r[k]);
        levinson(r, A[sig]);
        if (sig == 0) {
#pragma unroll
            for (int k = 0; k <= kLpcOrder; k++) Rc[k] = (float)r[k];
        }
    }
    if (lane == 0) {
        double frac = toeplitz_form(A[1], Rc) / (toeplitz_form(A[0], Rc) + kEps64);
        if (frac <= 0.0) frac = 1000.0;
        b.llr[e.cf + i] = log(frac);
    }
}

// In-place 1024-point complex FFT of z (shared) by the CTA's 256 threads: five Stockham radix-4 stages, one butterfly per
// thread and stage; tw[m] = e^(-2 pi i m / 1024).
__device__ __forceinline__ void fft1024(double2 *z, const double2 *__restrict__ tw) {
    const int j = threadIdx.x;
#pragma unroll 1
    for (int ns = 1; ns < kWssFft; ns *= 4) {
        const int jm = j & (ns - 1), step = kWssFft / (4 * ns);
        double2 v[4];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            v[r] = z[j + r * (kWssFft / 4)];
            if (r) v[r] = cmul(v[r], __ldg(tw + r * jm * step));
        }
        const double2 a0 = make_double2(v[0].x + v[2].x, v[0].y + v[2].y), a1 = make_double2(v[0].x - v[2].x, v[0].y - v[2].y);
        const double2 a2 = make_double2(v[1].x + v[3].x, v[1].y + v[3].y), a3 = make_double2(v[1].x - v[3].x, v[1].y - v[3].y);
        const int d = (j - jm) * 4 + jm;
        __syncthreads();   // every thread has read its inputs
        z[d] = make_double2(a0.x + a2.x, a0.y + a2.y);
        z[d + ns] = make_double2(a1.x + a3.y, a1.y - a3.x);          // a1 - i a3
        z[d + 2 * ns] = make_double2(a0.x - a2.x, a0.y - a2.y);
        z[d + 3 * ns] = make_double2(a1.x - a3.y, a1.y + a3.x);      // a1 + i a3
        __syncthreads();
    }
}

// findLocPeaks for the band of this lane (slopes on lanes 0 .. 23, energies on lanes 0 .. 24), its exact rule: for a
// rising slope, walk up while the slope rises (to band 24 at most) and take energy[n - 1]; otherwise walk down while it
// does not rise and take energy[n + 1].  The walks are a ballot and a find-first-set.
__device__ __forceinline__ double loc_peak(double slope, double en, int lane) {
    const unsigned rise = __ballot_sync(0xffffffffu, lane < kWssBands - 1 && slope > 0.0);
    int src;
    if ((rise >> lane) & 1u) {
        const unsigned m = ~rise & ((1u << (kWssBands - 1)) - 1u) & (~0u << lane);
        src = (m ? __ffs(m) - 1 : kWssBands - 1) - 1;
    } else {
        const unsigned m = rise & (lane < 31 ? (2u << lane) - 1u : ~0u);
        src = (m ? 31 - __clz(m) : -1) + 1;
    }
    return __shfl_sync(0xffffffffu, en, src & 31);
}

// grid (max T, B), 256 threads: frame i = blockIdx.x of entry blockIdx.y.  sepm.wss at 16 kHz: both windowed frames
// w_n (x_n + eps) in fp64 as one complex 1024-point FFT (clean real, degraded imaginary), the power of bins 0 .. 511 of
// each, the 25 critical-band energies in dB (clamped at -100), their 24 slopes, Klatt's weights (Kmax 20, Klocmax 1)
// averaged over both signals, and wss[cf + i] = sum W (slope_c - slope_d)^2 / sum W.
__global__ void __launch_bounds__(256) k_wss(const MetEntry *__restrict__ ents, MetBufs b) {
    __shared__ double2 z[kWssFft];
    const MetEntry e = ents[blockIdx.y];
    const int i = blockIdx.x;
    if (i >= e.nct) return;
    const float *c = b.x16 + e.o16 + (int64_t)i * kSsnrHop, *d = b.y16 + e.o16 + (int64_t)i * kSsnrHop;
    for (int n = threadIdx.x; n < kWssFft; n += blockDim.x) {
        double2 v = make_double2(0.0, 0.0);
        if (n < kSsnrWin) {
            const double w = c_wss[n];
            v.x = w * ((double)__ldg(c + n) + kEps64);
            v.y = w * ((double)__ldg(d + n) + kEps64);
        }
        z[n] = v;
    }
    __syncthreads();
    fft1024(z, b.fft_tw);
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    double ec = 0.0, ed = 0.0;
    if (lane < kWssBands) {
        const int lo = c_crit_lo[lane], nb = c_crit_n[lane], off = c_crit_off[lane];
        for (int t = 0; t < nb; t++) {
            const int k = lo + t;
            const double2 zk = z[k], zn = z[(kWssFft - k) & (kWssFft - 1)];
            // X_k = (Z_k + conj Z_-k) / 2, Y_k = (Z_k - conj Z_-k) / 2i
            const double xr = 0.5 * (zk.x + zn.x), xi = 0.5 * (zk.y - zn.y);
            const double yr = 0.5 * (zk.y + zn.y), yi = 0.5 * (zn.x - zk.x);
            const double g = c_crit[off + t];
            ec = fma(g, xr * xr + xi * xi, ec);
            ed = fma(g, yr * yr + yi * yi, ed);
        }
    }
    double lc = 10.0 * log10(ec), ld = 10.0 * log10(ed);
    if (!(lc >= -100.0)) lc = -100.0;   // log10(0) = -inf
    if (!(ld >= -100.0)) ld = -100.0;
    const double sc = __shfl_down_sync(0xffffffffu, lc, 1) - lc, sd = __shfl_down_sync(0xffffffffu, ld, 1) - ld;
    double mc = lane < kWssBands ? lc : -INFINITY, md = lane < kWssBands ? ld : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mc = fmax(mc, __shfl_xor_sync(0xffffffffu, mc, o));
        md = fmax(md, __shfl_xor_sync(0xffffffffu, md, o));
    }
    const double pc = loc_peak(sc, lc, lane), pd = loc_peak(sd, ld, lane);
    double num = 0.0, den = 0.0;
    if (lane < kWssBands - 1) {
        const double wc = 20.0 / ((20.0 + mc) - lc) * (1.0 / ((1.0 + pc) - lc));
        const double wd = 20.0 / ((20.0 + md) - ld) * (1.0 / ((1.0 + pd) - ld));
        const double W = (wc + wd) / 2.0;
        num = W * ((sc - sd) * (sc - sd));
        den = W;
    }
    num = warp_sum(num);
    den = warp_sum(den);
    if (lane == 0) b.wss[e.cf + i] = num / den;
}

// Order-preserving key of a double: a larger value has a larger key.
__device__ __forceinline__ unsigned long long okey(double v) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// The mean of the k smallest of v[0 .. n) (1 <= k <= n) by the CTA, independent of their order: a bitwise radix select of
// the k-th smallest key t (64 counting passes), then (sum of the values below t in a fixed order + (k - their count) t) / k.
__device__ double trimmed_mean(const double *__restrict__ v, int n, int k, double *sm) {
    unsigned long long t = 0;
    for (int bit = 63; bit >= 0; bit--) {
        const unsigned long long hi = t | ((1ull << bit) - 1ull);   // the largest key with t's prefix and a 0 here
        int c = 0;
        for (int j = threadIdx.x; j < n; j += blockDim.x) c += okey(v[j]) <= hi;
        c = block_sum(c, reinterpret_cast<int *>(sm));
        if (c < k) t |= 1ull << bit;
    }
    double s = 0.0;
    int c = 0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const double x = v[j];
        if (okey(x) < t) { s += x; c++; }
    }
    s = block_sum(s, sm);
    c = block_sum(c, reinterpret_cast<int *>(sm));
    const double tv = __longlong_as_double((long long)((t >> 63) ? (t & 0x7fffffffffffffffull) : ~t));
    return (s + (double)(k - c) * tv) / (double)k;
}

// grid (ceil(max chunks), B), 256 threads: chunk k of entry blockIdx.y, samples [4096 k, 4096 k + 4096): fp64 sums of
// r r, r e and e e (each product of two floats is exact in fp64).
__global__ void __launch_bounds__(256) k_sisdr(const MetEntry *__restrict__ ents, MetBufs b) {
    __shared__ double sm[32];
    const MetEntry e = ents[blockIdx.y];
    if ((int)blockIdx.x >= e.nch) return;
    const int64_t p0 = e.in_off + (int64_t)blockIdx.x * kSisdrChunk;
    const int64_t n = min((int64_t)kSisdrChunk, e.len - (int64_t)blockIdx.x * kSisdrChunk);
    double rr = 0.0, re = 0.0, ee = 0.0;
    for (int64_t k = threadIdx.x; k < n; k += blockDim.x) {
        const double r = __ldg(b.clean + p0 + k), s = __ldg(b.degraded + p0 + k);
        rr = fma(r, r, rr); re = fma(r, s, re); ee = fma(s, s, ee);
    }
    rr = block_sum(rr, sm);
    re = block_sum(re, sm);
    ee = block_sum(ee, sm);
    if (threadIdx.x == 0) {
        const int64_t o = e.co + blockIdx.x;
        b.ch[o] = rr; b.ch[b.n_ch + o] = re; b.ch[2 * b.n_ch + o] = ee;
    }
}

// grid B, 256 threads: out[row][b] for the metrics of `bits`, rows in the order SI-SDR, STOI, SSNR, LLR, WSS, PYSTOI, ESTOI.
__global__ void __launch_bounds__(256) k_metrics_final(const MetEntry *__restrict__ ents, MetBufs b, int bits, float *out, int64_t B) {
    __shared__ double sm[32];
    const MetEntry e = ents[blockIdx.x];
    int row = 0;
    if (bits & DFB_METRIC_SISDR) {
        double rr = 0.0, re = 0.0, ee = 0.0;
        for (int k = threadIdx.x; k < e.nch; k += blockDim.x) {
            rr += b.ch[e.co + k]; re += b.ch[b.n_ch + e.co + k]; ee += b.ch[2 * b.n_ch + e.co + k];
        }
        rr = block_sum(rr, sm);
        re = block_sum(re, sm);
        ee = block_sum(ee, sm);
        if (threadIdx.x == 0) {
            const double a = (kEps32 + re) / (rr + kEps32);
            const double sss = a * a * rr;
            double snn = ee - 2.0 * a * re + a * a * rr;   // |e - a r|^2; the sums are exact to ~1e-16 of ee
            if (snn < 0.0) snn = 0.0;
            out[row * B + blockIdx.x] = (float)(10.0 * log10((kEps32 + sss) / (kEps32 + snn)));
        }
        row++;
    }
    if (bits & DFB_METRIC_STOI) {
        const int L = b.st[blockIdx.x].nf, J = L > kStoiSeg ? L - kStoiSeg + 1 : 1;
        float s = 0.f;
        for (int k = threadIdx.x; k < J && L > 0; k += blockDim.x) s += b.seg[e.fo + k];
        s = block_sum(s, reinterpret_cast<float *>(sm));
        if (threadIdx.x == 0) out[row * B + blockIdx.x] = L > 0 ? s / (float)(kStoiBands * J) : __int_as_float(0x7fc00000);
        row++;
    }
    if (bits & DFB_METRIC_SSNR) {
        const int n = e.nfs - 1;
        double s = 0.0;
        for (int k = threadIdx.x; k < n; k += blockDim.x) s += b.ss[e.so + k];
        s = block_sum(s, sm);
        if (threadIdx.x == 0) out[row * B + blockIdx.x] = n > 0 ? (float)(s / n) : __int_as_float(0x7fc00000);
        row++;
    }
    for (int m = 0; m < 2; m++) {
        if (!(bits & (m ? DFB_METRIC_WSS : DFB_METRIC_LLR))) continue;
        const double v = e.nct > 0 ? trimmed_mean((m ? b.wss : b.llr) + e.cf, e.nct, e.kct, sm) : 0.0;
        if (threadIdx.x == 0) out[row * B + blockIdx.x] = e.nct > 0 ? (float)v : __int_as_float(0x7fc00000);
        row++;
    }
    // pystoi: NaN without a frame (pystoi raises), 1e-5 with fewer than 30 STFT frames (pystoi warns and returns it)
    for (int m = 0; m < 2; m++) {
        if (!(bits & (m ? DFB_METRIC_ESTOI : DFB_METRIC_PYSTOI))) continue;
        const int nf = e.pnf > 0 ? b.pst[blockIdx.x].nf : 0, J = nf - kStoiSeg + 1;
        double s = 0.0;
        for (int k = threadIdx.x; k < J; k += blockDim.x) s += b.pseg[m * b.n_pf + e.po + k];
        s = block_sum(s, sm);
        if (threadIdx.x == 0)
            out[row * B + blockIdx.x] = e.pnf == 0 ? __int_as_float(0x7fc00000)
                                        : J <= 0   ? 1e-5f
                                                   : (float)(m ? s / J : s / ((double)J * kStoiBands));
        row++;
    }
}

// thirdoct (df/stoi.py): band i covers the FFT bins [lo, hi) nearest to 150 Hz 2^((2 i -+ 1) / 6) at 10 kHz, 512 points
StoiBands stoi_bands() {
    StoiBands b{};
    const int nb = kStoiFft / 2 + 1;
    auto nearest = [&](double fq) {
        int best = 0;
        double bd = INFINITY;
        for (int k = 0; k < nb; k++) {
            const double d = (k * ((double)kStoiFs / kStoiFft) - fq) * (k * ((double)kStoiFs / kStoiFft) - fq);
            if (d < bd) { bd = d; best = k; }
        }
        return best;
    };
    for (int i = 0; i < kStoiBands; i++) {
        b.lo[i] = nearest(150.0 * std::pow(2.0, (2.0 * i - 1) / 6));
        b.hi[i] = nearest(150.0 * std::pow(2.0, (2.0 * i + 1) / 6));
    }
    double ws = 0.0;
    for (int n = 0; n < kStoiFrame; n++) ws += (double)(float)(0.5 - 0.5 * std::cos(2.0 * M_PI * (n + 1) / (kStoiFrame + 1)));
    b.inv_wsum = (float)(1.0 / ws);
    return b;
}

// The 25 critical bands of D. H. Klatt, "Prediction of perceived phonetic distance from critical-band spectra: a first
// step", Proc. IEEE ICASSP 1982, pp. 1278-1281: centre frequencies and bandwidths in Hz, as the weighted spectral slope
// measure uses them (7 bands of 70 Hz, then each band starting where the previous one ends).
constexpr double kCritCentre[kWssBands] = {50.0,    120.0,   190.0,   260.0,   330.0,   400.0,   470.0,   540.0,   617.372,
                                           703.378, 798.717, 904.128, 1020.38, 1148.30, 1288.72, 1442.54, 1610.70, 1794.16,
                                           1993.93, 2211.08, 2446.71, 2701.97, 2978.04, 3276.17, 3597.63};
constexpr double kCritWidth[kWssBands] = {70.0,    70.0,    70.0,    70.0,    70.0,    70.0,    70.0,    77.3724, 86.0056,
                                          95.3398, 105.411, 116.256, 127.914, 140.423, 153.823, 168.154, 183.457, 199.776,
                                          217.153, 235.631, 255.255, 276.072, 298.126, 321.465, 346.136};

// The critical-band filters over the 512 kept bins at 16 kHz: band i weighs bin j by
// exp(-11 ((j - floor(f0)) / bw)^2 + ln(70 / width_i)), f0 and bw the centre and width in bins, where that exceeds the
// filter's -30 dB point exp(-30 / (2 * 2.303)); each band's nonzero weights are one contiguous run of bins.
struct CritFilters { double w[kMaxCritTaps]; int lo[kWssBands], n[kWssBands], off[kWssBands]; };
bool crit_filters(CritFilters &f) {
    const double min_factor = std::exp(-30.0 / (2.0 * 2.303));
    int used = 0;
    for (int i = 0; i < kWssBands; i++) {
        const double f0 = std::floor(kCritCentre[i] / (kSsnrFs / 2.0) * kWssBins);
        const double bw = kCritWidth[i] / (kSsnrFs / 2.0) * kWssBins;
        const double norm = std::log(kCritWidth[0]) - std::log(kCritWidth[i]);
        f.lo[i] = -1;
        f.n[i] = 0;
        f.off[i] = used;
        for (int j = 0; j < kWssBins; j++) {
            const double q = (j - f0) / bw;
            const double w = std::exp(-11.0 * (q * q) + norm);
            if (!(w > min_factor)) continue;
            if (f.lo[i] < 0) f.lo[i] = j;
            if (j != f.lo[i] + f.n[i] || used >= kMaxCritTaps) return false;
            f.w[used++] = w;
            f.n[i]++;
        }
        if (f.lo[i] < 0) f.lo[i] = 0;
    }
    return true;
}

}  // namespace
}  // namespace dfb

using namespace dfb;

struct dfb_metrics {
    int device, sr;
    cudaStream_t stream = nullptr;
    float *d_taps = nullptr;      // the sr -> 10 kHz and sr -> 16 kHz tap tables
    RateDir dirs[2]{};            // 0: -> 10 kHz, 1: -> 16 kHz (taps null: sr is that rate)
    RateDir *d_dirs = nullptr;
    float2 *d_tw = nullptr;       // twiddles of the 512-point real FFT
    GenFftPlan plan{};
    StoiBands bands{};
    Arena arena;                  // per-call workspace, grown when a call needs more
    int64_t last_b = 0;           // entries of the last call (dfb_debug_metrics_counts)
    MetState *last_st = nullptr;  // their STOI states, inside the arena
    double2 *d_fft_tw = nullptr;  // twiddles of WSS's 1024-point fp64 FFT
    std::vector<int64_t> last_nct;             // LLR / WSS frames of each entry of the last call (dfb_debug_metrics_frames)
    double *last_llr = nullptr, *last_wss = nullptr;   // their per-frame values, inside the arena
    std::vector<int64_t> last_pnf, last_po;    // pystoi frames F and first frame of each entry of the last call
    MetState *last_pst = nullptr;              // their pystoi states, inside the arena (dfb_debug_metrics_pystoi)
    double *last_pbx = nullptr, *last_pby = nullptr;   // their band magnitudes, inside the arena
};

namespace {

int64_t resampled_len(int64_t T, int og, int nw) { return (nw * T + og - 1) / og; }

int check_taps(int sr, int to, const float *taps, int og, int nw, int width, int64_t *floats) {
    *floats = 0;
    if (sr == to) return DFB_OK;
    int64_t g = std::gcd((int64_t)sr, (int64_t)to);
    if (!taps || og != sr / g || nw != to / g || width <= 0)
        return fail(DFB_ERR_INVALID, "the taps of %d Hz -> %d Hz are io.resample_kernel(%d, %d) (og %lld, nw %lld)", sr, to, sr, to,
                    (long long)(sr / g), (long long)(to / g));
    *floats = (int64_t)nw * (2 * width + og);
    return DFB_OK;
}

// The buffers of a call of B entries, planned on the host: (entries, workspace bytes).
struct MetPlan {
    std::vector<MetEntry> ents;
    std::vector<RateRow> rows;
    int64_t n10 = 0, n16 = 0, n_fr = 0, n_ss = 0, n_ch = 0, n_cf = 0, max_fr = 0, max_ss = 0, max_ch = 0, max_cf = 0, max_out = 0;
    int64_t n_pf = 0, max_pf = 0;   // pystoi frames
};

int plan_call(const dfb_metrics *h, int64_t in_numel, const int64_t *offsets, const int64_t *lengths, const int64_t *deg_lengths,
              int64_t B, int bits, MetPlan &p) {
    if (B <= 0 || B > 32767) return fail(DFB_ERR_INVALID, "batch of %lld entries: 1 .. 32767 per call", (long long)B);
    if (bits <= 0 || (bits & ~(DFB_METRIC_SISDR | DFB_METRIC_STOI | DFB_METRIC_SSNR | DFB_METRIC_LLR | DFB_METRIC_WSS |
                               DFB_METRIC_PYSTOI | DFB_METRIC_ESTOI)))
        return fail(DFB_ERR_INVALID, "unknown metric bits 0x%x (SI-SDR 1, STOI 2, SSNR 4, LLR 16, WSS 32, PYSTOI 128, ESTOI 256)",
                    bits);
    if (!offsets || !lengths || !deg_lengths) return fail(DFB_ERR_INVALID, "null layout");
    const bool stoi = bits & DFB_METRIC_STOI, ssnr = bits & DFB_METRIC_SSNR, comp = bits & (DFB_METRIC_LLR | DFB_METRIC_WSS);
    const bool py = bits & (DFB_METRIC_PYSTOI | DFB_METRIC_ESTOI);
    const bool rs10 = (stoi || py) && h->dirs[0].taps, rs16 = (ssnr || comp) && h->dirs[1].taps;
    p.ents.resize(B);
    for (int64_t b = 0; b < B; b++) {
        const int64_t T = lengths[b];
        if (T <= 0) return fail(DFB_ERR_INVALID, "entry %lld: length %lld, must be > 0", (long long)b, (long long)T);
        if (deg_lengths[b] != T)
            return fail(DFB_ERR_INVALID, "entry %lld: clean has %lld samples, degraded %lld", (long long)b, (long long)T,
                        (long long)deg_lengths[b]);
        if (offsets[b] < 0 || offsets[b] > in_numel - T)
            return fail(DFB_ERR_INVALID, "entry %lld reaches outside the %lld input samples", (long long)b, (long long)in_numel);
        MetEntry &e = p.ents[b];
        std::memset(&e, 0, sizeof e);
        e.in_off = offsets[b];
        e.len = T;
        if (stoi || py) {
            e.t10 = rs10 ? resampled_len(T, h->dirs[0].og, h->dirs[0].nw) : T;
            e.o10 = rs10 ? p.n10 : e.in_off;
            if (rs10) {
                p.rows.push_back(RateRow{e.in_off, T, e.o10, e.t10, 0, 0});
                p.n10 += e.t10;
                p.max_out = std::max(p.max_out, e.t10);
            }
        }
        if (py) {
            const int64_t pnf = e.t10 > kStoiFrame ? (e.t10 - kStoiFrame + kStoiHop - 1) / kStoiHop : 0;
            if (pnf > (1 << 30)) return fail(DFB_ERR_INVALID, "entry %lld is too long", (long long)b);
            e.pnf = (int)pnf;
            e.po = p.n_pf;
            p.n_pf += pnf;
            p.max_pf = std::max(p.max_pf, pnf);
        }
        if (stoi) {
            const int64_t pad = kStoiFrame - e.t10 % kStoiFrame;
            e.pad_front = (int)(pad / 2);
            e.pad_end = (int)(pad - pad / 2);
            const int64_t nfr = (e.t10 + pad) / kStoiHop - 1;
            if (nfr > (1 << 30)) return fail(DFB_ERR_INVALID, "entry %lld is too long", (long long)b);
            e.nfr = (int)nfr;
            e.fo = p.n_fr;
            p.n_fr += nfr;
            p.max_fr = std::max(p.max_fr, nfr);
        }
        if (ssnr || comp) {
            e.t16 = rs16 ? resampled_len(T, h->dirs[1].og, h->dirs[1].nw) : T;
            e.o16 = rs16 ? 0 : e.in_off;   // (16 kHz rows follow the 10 kHz ones: offset set below)
            if (rs16) {
                p.rows.push_back(RateRow{e.in_off, T, p.n16, e.t16, 0, 1});
                e.o16 = p.n16;
                p.n16 += e.t16;
                p.max_out = std::max(p.max_out, e.t16);
            }
        }
        if (comp) {
            const int64_t nct = e.t16 >= kSsnrWin ? (e.t16 - kSsnrWin) / kSsnrHop : 0;
            if (nct > (1 << 30)) return fail(DFB_ERR_INVALID, "entry %lld is too long", (long long)b);
            e.nct = (int)nct;
            e.kct = (int)std::nearbyint((double)nct * 0.95);   // Python's round(T * 0.95): half to even
            e.cf = p.n_cf;
            p.n_cf += nct;
            p.max_cf = std::max(p.max_cf, nct);
        }
        if (ssnr) {
            const int64_t nfs = e.t16 >= kSsnrWin - kSsnrHop ? (e.t16 - kSsnrWin + kSsnrHop) / kSsnrHop : 0;
            e.nfs = (int)nfs;
            e.so = p.n_ss;
            p.n_ss += std::max<int64_t>(nfs - 1, 0);
            p.max_ss = std::max(p.max_ss, nfs);
        }
        if (bits & DFB_METRIC_SISDR) {
            e.nch = (int)((T + kSisdrChunk - 1) / kSisdrChunk);
            e.co = p.n_ch;
            p.n_ch += e.nch;
            p.max_ch = std::max<int64_t>(p.max_ch, e.nch);
        }
    }
    // the 16 kHz rows live after the 10 kHz ones in the same resampled buffer
    for (auto &r : p.rows)
        if (r.dir == 1) r.out_off += p.n10;
    for (auto &e : p.ents)
        if (rs16) e.o16 += p.n10;
    return DFB_OK;
}

size_t a256(size_t n) { return (n + 255) & ~size_t(255); }

size_t call_bytes(const MetPlan &p, int64_t B, bool host, int64_t in_numel, int n_rows) {
    size_t s = a256(sizeof(MetEntry) * B) + a256(sizeof(RateRow) * (p.rows.size() + 1)) + a256(sizeof(MetState) * B);
    s += 2 * a256(sizeof(float) * (p.n10 + p.n16 + 1));                  // resampled clean / degraded
    s += a256(sizeof(float) * (p.n_fr + 1)) * 2 + a256(sizeof(int) * (p.n_fr + 1));   // energies, segments, kept list
    s += 2 * a256(sizeof(float) * (kStoiBands * p.n_fr + 1));            // band magnitudes
    s += a256(sizeof(double) * (p.n_ss + 1)) + a256(sizeof(double) * (3 * p.n_ch + 1));
    s += 2 * a256(sizeof(double) * (p.n_cf + 1));                        // LLR / WSS frame values
    // pystoi: energies, kept list, band magnitudes of both signals, STOI / ESTOI segment sums, states
    s += a256(sizeof(double) * (p.n_pf + 1)) + a256(sizeof(int) * (p.n_pf + 1)) + 2 * a256(sizeof(double) * (kStoiBands * p.n_pf + 1));
    s += a256(sizeof(double) * (2 * p.n_pf + 1)) + a256(sizeof(MetState) * B);
    if (host) s += 2 * a256(sizeof(float) * in_numel) + a256(sizeof(float) * n_rows * B);
    return s;
}

int run_call(dfb_metrics *h, const float *d_clean, const float *d_deg, const MetPlan &p, int64_t B, int bits, float *d_out,
             cudaStream_t s, const float *h_clean, const float *h_deg, int64_t in_numel, float *h_out) {
    const bool host = h_clean != nullptr;
    const int n_rows = __builtin_popcount(bits);
    int rc = h->arena.reserve(call_bytes(p, B, host, in_numel, n_rows));
    if (rc) return rc;
    Arena &a = h->arena;
    a.reset();
    MetEntry *d_ents = a.take<MetEntry>(B);
    RateRow *d_rows = a.take<RateRow>(p.rows.size() + 1);
    MetBufs mb{};
    mb.st = a.take<MetState>(B);
    float *rx = a.take<float>(p.n10 + p.n16 + 1), *ry = a.take<float>(p.n10 + p.n16 + 1);
    mb.en = a.take<float>(p.n_fr + 1);
    mb.seg = a.take<float>(p.n_fr + 1);
    mb.kidx = a.take<int>(p.n_fr + 1);
    mb.bx = a.take<float>(kStoiBands * p.n_fr + 1);
    mb.by = a.take<float>(kStoiBands * p.n_fr + 1);
    mb.ss = a.take<double>(p.n_ss + 1);
    mb.ch = a.take<double>(3 * p.n_ch + 1);
    mb.llr = a.take<double>(p.n_cf + 1);
    mb.wss = a.take<double>(p.n_cf + 1);
    mb.pen = a.take<double>(p.n_pf + 1);
    mb.pkidx = a.take<int>(p.n_pf + 1);
    mb.pbx = a.take<double>(kStoiBands * p.n_pf + 1);
    mb.pby = a.take<double>(kStoiBands * p.n_pf + 1);
    mb.pseg = a.take<double>(2 * p.n_pf + 1);
    mb.pst = a.take<MetState>(B);
    mb.n_pf = p.n_pf;
    mb.fft_tw = h->d_fft_tw;
    mb.n_fr = p.n_fr;
    mb.n_ch = p.n_ch;
    if (host) {
        float *c = a.take<float>(in_numel), *d = a.take<float>(in_numel);
        d_out = a.take<float>((size_t)n_rows * B);
        DFB_CUDA(cudaMemcpyAsync(c, h_clean, sizeof(float) * in_numel, cudaMemcpyHostToDevice, s));
        DFB_CUDA(cudaMemcpyAsync(d, h_deg, sizeof(float) * in_numel, cudaMemcpyHostToDevice, s));
        d_clean = c;
        d_deg = d;
    }
    mb.clean = d_clean;
    mb.degraded = d_deg;
    mb.x10 = h->dirs[0].taps ? rx : d_clean;
    mb.y10 = h->dirs[0].taps ? ry : d_deg;
    mb.x16 = h->dirs[1].taps ? rx : d_clean;
    mb.y16 = h->dirs[1].taps ? ry : d_deg;
    DFB_CUDA(cudaMemcpyAsync(d_ents, p.ents.data(), sizeof(MetEntry) * B, cudaMemcpyHostToDevice, s));
    if (!p.rows.empty()) {
        DFB_CUDA(cudaMemcpyAsync(d_rows, p.rows.data(), sizeof(RateRow) * p.rows.size(), cudaMemcpyHostToDevice, s));
        int smem = 0;
        for (const RateDir &d : h->dirs)
            if (d.taps && d.nw * d.K <= kRateSmemFloats) smem = std::max(smem, d.nw * d.K);
        for (int sig = 0; sig < 2; sig++) {
            const RateIO io{sig ? d_deg : d_clean, sig ? ry : rx, 0, p.max_out, 0, 0};
            rc = launch_resample_rows(s, true, h->d_dirs, d_rows, (int)p.rows.size(), io, p.max_out, smem);
            if (rc) return rc;
        }
    }
    const unsigned ub = (unsigned)B;
    if (bits & DFB_METRIC_STOI) {
        k_stoi_energy<<<dim3((unsigned)((p.max_fr + 7) / 8), ub), 256, 0, s>>>(d_ents, mb);
        DFB_LAUNCH_CHECK();
        k_stoi_mask<false><<<ub, 1024, 0, s>>>(d_ents, mb);
        DFB_LAUNCH_CHECK();
        k_stoi_stft<<<dim3((unsigned)((p.max_fr + kStftFrames - 1) / kStftFrames), ub), 256, 0, s>>>(d_ents, mb, h->plan, h->bands);
        DFB_LAUNCH_CHECK();
        k_stoi_seg<<<dim3((unsigned)((p.max_fr + 7) / 8), ub), 256, 0, s>>>(d_ents, mb);
        DFB_LAUNCH_CHECK();
    }
    if (bits & (DFB_METRIC_PYSTOI | DFB_METRIC_ESTOI)) {
        if (p.max_pf > 0) {
            k_pystoi_energy<<<dim3((unsigned)((p.max_pf + 7) / 8), ub), 256, 0, s>>>(d_ents, mb);
            DFB_LAUNCH_CHECK();
        }
        k_stoi_mask<true><<<ub, 1024, 0, s>>>(d_ents, mb);
        DFB_LAUNCH_CHECK();
        if (p.max_pf > 1) {
            k_pystoi_stft<<<dim3((unsigned)p.max_pf, ub), 128, 0, s>>>(d_ents, mb, h->bands);
            DFB_LAUNCH_CHECK();
        }
        if (p.max_pf > kStoiSeg) {
            k_pystoi_seg<<<dim3((unsigned)((p.max_pf + 7) / 8), ub), 256, 0, s>>>(d_ents, mb);
            DFB_LAUNCH_CHECK();
        }
    }
    if ((bits & DFB_METRIC_SSNR) && p.max_ss > 1) {
        k_ssnr<<<dim3((unsigned)((p.max_ss + 7) / 8), ub), 256, 0, s>>>(d_ents, mb);
        DFB_LAUNCH_CHECK();
    }
    if ((bits & DFB_METRIC_LLR) && p.max_cf > 0) {
        k_llr<<<dim3((unsigned)((p.max_cf + 3) / 4), ub), 128, 0, s>>>(d_ents, mb);
        DFB_LAUNCH_CHECK();
    }
    if ((bits & DFB_METRIC_WSS) && p.max_cf > 0) {
        k_wss<<<dim3((unsigned)p.max_cf, ub), 256, 0, s>>>(d_ents, mb);
        DFB_LAUNCH_CHECK();
    }
    if (bits & DFB_METRIC_SISDR) {
        k_sisdr<<<dim3((unsigned)p.max_ch, ub), 256, 0, s>>>(d_ents, mb);
        DFB_LAUNCH_CHECK();
    }
    k_metrics_final<<<ub, 256, 0, s>>>(d_ents, mb, bits, d_out, B);
    DFB_LAUNCH_CHECK();
    h->last_b = (bits & DFB_METRIC_STOI) ? B : 0;
    h->last_st = mb.st;
    h->last_nct.clear();
    if (bits & (DFB_METRIC_LLR | DFB_METRIC_WSS))
        for (const MetEntry &e : p.ents) h->last_nct.push_back(e.nct);
    h->last_llr = mb.llr;
    h->last_wss = mb.wss;
    h->last_pnf.clear();
    h->last_po.clear();
    if (bits & (DFB_METRIC_PYSTOI | DFB_METRIC_ESTOI))
        for (const MetEntry &e : p.ents) { h->last_pnf.push_back(e.pnf); h->last_po.push_back(e.po); }
    h->last_pst = mb.pst;
    h->last_pbx = mb.pbx;
    h->last_pby = mb.pby;
    if (host) {
        DFB_CUDA(cudaMemcpyAsync(h_out, d_out, sizeof(float) * n_rows * B, cudaMemcpyDeviceToHost, s));
        DFB_CUDA(cudaStreamSynchronize(s));
    }
    return DFB_OK;
}

}  // namespace

extern "C" int dfb_metrics_create(dfb_metrics **out, int device, int sr, const float *taps10, int og10, int nw10, int width10,
                                  const float *taps16, int og16, int nw16, int width16) {
    if (!out) return fail(DFB_ERR_INVALID, "null argument");
    *out = nullptr;
    if (sr <= 0) return fail(DFB_ERR_UNSUPPORTED, "sample rate %d Hz", sr);
    int64_t f10 = 0, f16 = 0;
    int rc = check_taps(sr, kStoiFs, taps10, og10, nw10, width10, &f10);
    if (!rc) rc = check_taps(sr, kSsnrFs, taps16, og16, nw16, width16, &f16);
    if (rc) return rc;
    if (f10 + f16 > (1 << 18))
        return fail(DFB_ERR_UNSUPPORTED, "sample rate %d Hz: its resampler taps hold %lld floats, more than 2^18", sr,
                    (long long)(f10 + f16));
    rc = use_device(device);
    if (rc) return rc;
    auto *h = new dfb_metrics();
    h->device = device;
    h->sr = sr;
    auto bail = [&](int code) { dfb_metrics_free(h); return code; };
    std::vector<float2> tw;
    gen_fft_plan(kStoiFft, h->plan, tw);
    h->bands = stoi_bands();
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaMalloc(&h->d_tw, sizeof(float2) * tw.size()) != cudaSuccess ||
        cudaMalloc(&h->d_dirs, sizeof(RateDir) * 2) != cudaSuccess || cudaMalloc(&h->d_fft_tw, sizeof(double2) * kWssFft) != cudaSuccess ||
        cudaMalloc(&h->d_taps, sizeof(float) * (size_t)(f10 + f16 + 1)) != cudaSuccess)
        return bail(fail(DFB_ERR_OOM, "metrics handle allocation failed"));
    if (f10) {
        if (cudaMemcpy(h->d_taps, taps10, sizeof(float) * f10, cudaMemcpyHostToDevice) != cudaSuccess)
            return bail(fail(DFB_ERR_CUDA, "tap upload failed"));
        h->dirs[0] = RateDir{h->d_taps, og10, nw10, 2 * width10 + og10, width10};
    }
    if (f16) {
        if (cudaMemcpy(h->d_taps + f10, taps16, sizeof(float) * f16, cudaMemcpyHostToDevice) != cudaSuccess)
            return bail(fail(DFB_ERR_CUDA, "tap upload failed"));
        h->dirs[1] = RateDir{h->d_taps + f10, og16, nw16, 2 * width16 + og16, width16};
    }
    float w256[kStoiFrame];
    for (int n = 0; n < kStoiFrame; n++) w256[n] = (float)(0.5 - 0.5 * std::cos(2.0 * M_PI * (n + 1) / (kStoiFrame + 1)));
    double w256d[kStoiFrame];
    for (int n = 0; n < kStoiFrame; n++) w256d[n] = 0.5 - 0.5 * std::cos(2.0 * M_PI * (n + 1) / (kStoiFrame + 1));
    double wss[kSsnrWin];
    for (int n = 0; n < kSsnrWin; n++) wss[n] = 0.5 * (1.0 - std::cos(2.0 * M_PI * (n + 1) / (kSsnrWin + 1)));
    std::vector<double2> tw64(kWssFft);
    for (int m = 0; m < kWssFft; m++) tw64[m] = make_double2(std::cos(2.0 * M_PI * m / kWssFft), -std::sin(2.0 * M_PI * m / kWssFft));
    static CritFilters crit;
    if (!crit_filters(crit)) return bail(fail(DFB_ERR_UNSUPPORTED, "critical-band filter table overflow"));
    if (cudaMemcpy(h->d_tw, tw.data(), sizeof(float2) * tw.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(h->d_fft_tw, tw64.data(), sizeof(double2) * kWssFft, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpyToSymbol(c_crit, crit.w, sizeof crit.w) != cudaSuccess || cudaMemcpyToSymbol(c_crit_lo, crit.lo, sizeof crit.lo) != cudaSuccess ||
        cudaMemcpyToSymbol(c_crit_n, crit.n, sizeof crit.n) != cudaSuccess || cudaMemcpyToSymbol(c_crit_off, crit.off, sizeof crit.off) != cudaSuccess ||
        cudaMemcpy(h->d_dirs, h->dirs, sizeof(RateDir) * 2, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpyToSymbol(c_w256, w256, sizeof w256) != cudaSuccess || cudaMemcpyToSymbol(c_wss, wss, sizeof wss) != cudaSuccess ||
        cudaMemcpyToSymbol(c_w256d, w256d, sizeof w256d) != cudaSuccess)
        return bail(fail(DFB_ERR_CUDA, "metrics table upload failed"));
    h->plan.tw = h->d_tw;
    *out = h;
    return DFB_OK;
}

extern "C" void dfb_metrics_free(dfb_metrics *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    h->arena.release();
    cudaFree(h->d_taps);
    cudaFree(h->d_dirs);
    cudaFree(h->d_tw);
    cudaFree(h->d_fft_tw);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

extern "C" int64_t dfb_metrics_workspace_bytes(const dfb_metrics *h) { return h ? (int64_t)h->arena.cap : -1; }

extern "C" int dfb_metrics_compute(dfb_metrics *h, const float *d_clean, const float *d_degraded, int64_t in_numel, const int64_t *offsets,
                           const int64_t *clean_lengths, const int64_t *degraded_lengths, int64_t B, int metrics, float *d_out,
                           void *stream) {
    if (!h || !d_clean || !d_degraded || !d_out) return fail(DFB_ERR_INVALID, "null argument");
    MetPlan p;
    int rc = plan_call(h, in_numel, offsets, clean_lengths, degraded_lengths, B, metrics, p);
    if (rc) return rc;
    DFB_CUDA(cudaSetDevice(h->device));
    return run_call(h, d_clean, d_degraded, p, B, metrics, d_out, (cudaStream_t)stream, nullptr, nullptr, in_numel, nullptr);
}

extern "C" int dfb_metrics_compute_host(dfb_metrics *h, const float *h_clean, const float *h_degraded, int64_t in_numel,
                                const int64_t *offsets, const int64_t *clean_lengths, const int64_t *degraded_lengths, int64_t B,
                                int metrics, float *h_out) {
    if (!h || !h_clean || !h_degraded || !h_out) return fail(DFB_ERR_INVALID, "null argument");
    MetPlan p;
    int rc = plan_call(h, in_numel, offsets, clean_lengths, degraded_lengths, B, metrics, p);
    if (rc) return rc;
    DFB_CUDA(cudaSetDevice(h->device));
    return run_call(h, nullptr, nullptr, p, B, metrics, nullptr, h->stream, h_clean, h_degraded, in_numel, h_out);
}

extern "C" int dfb_debug_metrics_counts(dfb_metrics *h, const float *h_clean, const float *h_degraded, int64_t in_numel,
                                        const int64_t *offsets, const int64_t *lengths, int64_t B, int64_t *h_counts) {
    if (!h || !h_counts) return fail(DFB_ERR_INVALID, "null argument");
    std::vector<float> stoi((size_t)(B > 0 ? B : 1));
    int rc = dfb_metrics_compute_host(h, h_clean, h_degraded, in_numel, offsets, lengths, lengths, B, DFB_METRIC_STOI, stoi.data());
    if (rc) return rc;
    std::vector<MetState> st(B);
    DFB_CUDA(cudaMemcpy(st.data(), h->last_st, sizeof(MetState) * B, cudaMemcpyDeviceToHost));
    for (int64_t b = 0; b < B; b++) {
        h_counts[3 * b] = st[b].nk;
        h_counts[3 * b + 1] = st[b].lc;
        h_counts[3 * b + 2] = st[b].nf;
    }
    return DFB_OK;
}

extern "C" int dfb_debug_metrics_frames(dfb_metrics *h, const float *h_clean, const float *h_degraded, int64_t in_numel,
                                        const int64_t *offsets, const int64_t *lengths, int64_t B, int64_t *h_frames,
                                        double *h_llr, double *h_wss, int64_t capacity) {
    if (!h || !h_frames || !h_llr || !h_wss) return fail(DFB_ERR_INVALID, "null argument");
    std::vector<float> rows((size_t)(2 * (B > 0 ? B : 1)));
    int rc = dfb_metrics_compute_host(h, h_clean, h_degraded, in_numel, offsets, lengths, lengths, B,
                                      DFB_METRIC_LLR | DFB_METRIC_WSS, rows.data());
    if (rc) return rc;
    int64_t n = 0;
    for (int64_t b = 0; b < B; b++) n += (h_frames[b] = h->last_nct[b]);
    if (n > capacity) return fail(DFB_ERR_INVALID, "%lld frames, room for %lld", (long long)n, (long long)capacity);
    DFB_CUDA(cudaMemcpy(h_llr, h->last_llr, sizeof(double) * n, cudaMemcpyDeviceToHost));
    DFB_CUDA(cudaMemcpy(h_wss, h->last_wss, sizeof(double) * n, cudaMemcpyDeviceToHost));
    return DFB_OK;
}

extern "C" int dfb_debug_metrics_pystoi(dfb_metrics *h, const float *h_clean, const float *h_degraded, int64_t in_numel,
                                        const int64_t *offsets, const int64_t *lengths, int64_t B, int64_t *h_counts,
                                        double *h_bands, int64_t capacity) {
    if (!h || !h_counts) return fail(DFB_ERR_INVALID, "null argument");
    std::vector<float> rows((size_t)(2 * (B > 0 ? B : 1)));
    int rc = dfb_metrics_compute_host(h, h_clean, h_degraded, in_numel, offsets, lengths, lengths, B,
                                      DFB_METRIC_PYSTOI | DFB_METRIC_ESTOI, rows.data());
    if (rc) return rc;
    std::vector<MetState> st(B);
    DFB_CUDA(cudaMemcpy(st.data(), h->last_pst, sizeof(MetState) * B, cudaMemcpyDeviceToHost));
    int64_t n = 0;
    for (int64_t b = 0; b < B; b++) {
        const int64_t F = h->last_pnf[b], nf = F > 0 ? st[b].nf : 0;
        int64_t *c = h_counts + 5 * b;
        c[0] = F;
        c[1] = F > 0 ? st[b].nk : 0;
        c[2] = F > 0 ? st[b].lc : 0;
        c[3] = nf;
        c[4] = nf >= kStoiSeg ? nf - kStoiSeg + 1 : 0;
        n += 2 * kStoiBands * nf;
    }
    if (!h_bands) return DFB_OK;
    if (n > capacity) return fail(DFB_ERR_INVALID, "%lld band magnitudes, room for %lld", (long long)n, (long long)capacity);
    int64_t o = 0;
    for (int64_t b = 0; b < B; b++) {
        const int64_t F = h->last_pnf[b], nf = h_counts[5 * b + 3];
        if (nf == 0) continue;
        for (int sig = 0; sig < 2; sig++) {
            const double *src = (sig ? h->last_pby : h->last_pbx) + kStoiBands * h->last_po[b];
            DFB_CUDA(cudaMemcpy2D(h_bands + o, sizeof(double) * nf, src, sizeof(double) * F, sizeof(double) * nf, kStoiBands,
                                  cudaMemcpyDeviceToHost));
            o += kStoiBands * nf;
        }
    }
    return DFB_OK;
}
