// dfb_dsp.cu -- analysis (windowed real FFT + ERB band energies), feature normalisation scans,
// and the fused apply (ERB gain x spectrum + deep filter) + synthesis (irFFT + window + OLA)
// kernels, plus the C-ABI entry points of the DSP state.
//
// Reference semantics (paths relative to /root/reference):
//   frame_analysis        libDF/src/lib.rs:356-394     (pyDF/src/lib.rs:41-72 batches it)
//   compute_band_corr     libDF/src/lib.rs:280-295, dB at :207-210
//   band_mean_norm_erb    libDF/src/lib.rs:244-251
//   band_unit_norm        libDF/src/lib.rs:253-259
//   apply_interp_band_gain libDF/src/lib.rs:314-326 == Mask.forward DeepFilterNet/df/modules.py:266-269
//   MF.DF                 DeepFilterNet/df/multiframe.py:72-74,126-136,169-180
//   frame_synthesis       libDF/src/lib.rs:396-427     (pyDF/src/lib.rs:74-107)
//
// HBM layout: audio f32[B,T]; spec c64[B,Tf,481] (frame-major, 3848 B rows); features
// f32[B,Tf,32] and c64[B,Tf,96]; every kernel reads/writes whole rows with consecutive lanes on
// consecutive addresses.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "dfb_common.cuh"
#include "dfb_fft.cuh"

namespace dfb {

thread_local std::string g_err;
std::atomic<int64_t> g_launches{0};

// ---- per-kernel event profiler -------------------------------------------------------------
namespace {
struct ProfRec { std::string name; cudaEvent_t a, b; };
std::vector<ProfRec> g_prof;
std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_pool;
bool g_prof_on = false;
std::string g_prof_only;
}  // namespace

ProfScope::ProfScope(const char *name, cudaStream_t stream) : s(stream) {
    if (!g_prof_on) return;
    if (!g_prof_only.empty() && g_prof_only != name) return;
    ProfRec r;
    r.name = name;
    if (!g_prof_pool.empty()) {
        r.a = g_prof_pool.back().first; r.b = g_prof_pool.back().second;
        g_prof_pool.pop_back();
    } else if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) {
        return;
    }
    cudaEventRecord(r.a, s);
    g_prof.push_back(r);
    slot = (int)g_prof.size() - 1;
}
ProfScope::~ProfScope() {
    if (slot >= 0) cudaEventRecord(g_prof[slot].b, s);
}

int use_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(DFB_ERR_CUDA, "no CUDA device available (%s); libdfb200 has no CPU fallback",
                    e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    if (device < 0 || device >= n) return fail(DFB_ERR_INVALID, "device %d out of range [0,%d)", device, n);
    DFB_CUDA(cudaSetDevice(device));
    cudaDeviceProp p;
    DFB_CUDA(cudaGetDeviceProperties(&p, device));
    if (p.major != 9 || p.minor != 0)
        return fail(DFB_ERR_CUDA, "device %d is sm_%d%d; libdfb200 is built for sm_90a only", device, p.major,
                    p.minor);
    return DFB_OK;
}

int Arena::reserve(size_t bytes) {
    if (bytes <= cap) return DFB_OK;
    if (base) {
        DFB_CUDA(cudaDeviceSynchronize());
        DFB_CUDA(cudaFree(base));
        base = nullptr;
        cap = 0;
    }
    size_t want = (bytes + (size_t(1) << 20)) & ~((size_t(1) << 20) - 1);
    cudaError_t e = cudaMalloc(&base, want);
    if (e != cudaSuccess) {
        base = nullptr;
        return fail(DFB_ERR_OOM, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
    }
    cap = want;
    return DFB_OK;
}
void Arena::release() {
    if (base) cudaFree(base);
    base = nullptr;
    cap = off = 0;
}

// ============================================================================ kernels =====

constexpr int kFft = 960, kHop = 480, kF = 481;
constexpr int kAnaWarps = 8;           // frames per CTA in the analysis kernel (one per warp)
constexpr int kSynWarps = 4;           // warps per CTA in the synthesis kernel
constexpr int kSynChunk = 16;          // consecutive frames per warp in the synthesis kernel
constexpr int kAnaSmem = sizeof(float) * ((kAnaWarps + 1) * 480 + 960) + sizeof(float2) * (242 + kN2 * kN1 + kAnaWarps * kTileFloat2);

// One warp: 480-point complex FFT of the values gathered by `load(n)` (n = 24 n1 + lane), result
// in natural order in buf[0..480).  `buf` is a per-warp shared buffer of kTileFloat2 float2 that
// serves as the pass-A/B transpose tile and then as the natural-order output; `load` may read it.
template <bool INV, typename LoadF>
__device__ __forceinline__ void warp_fft480(LoadF load, const float2 (&tw)[kN1], float2 *buf, int lane) {
    float2 a[kN1];
    if (lane < kN2) {
#pragma unroll
        for (int n1 = 0; n1 < kN1; n1++) a[n1] = load(kN2 * n1 + lane);
    }
    __syncwarp();
    if (lane < kN2) fft480_pass_a<INV>(a, tw, buf, lane);
    __syncwarp();
    float2 b[kN2];
    if (lane < kN1) fft480_pass_b<INV>(b, buf, lane);
    __syncwarp();
    if (lane < kN1) fft480_store_natural(b, buf, lane);
    __syncwarp();
}

// variant with the pass-A twiddles of this lane read from memory (tw_lane -> 20 float2)
template <bool INV, typename LoadF>
__device__ __forceinline__ void warp_fft480_twptr(LoadF load, const float2 *tw_lane, float2 *buf, int lane) {
    float2 a[kN1];
    if (lane < kN2) {
#pragma unroll
        for (int n1 = 0; n1 < kN1; n1++) a[n1] = load(kN2 * n1 + lane);
    }
    __syncwarp();
    if (lane < kN2) fft480_pass_a_ptr<INV>(a, tw_lane, buf, lane);
    __syncwarp();
    float2 b[kN2];
    if (lane < kN1) fft480_pass_b<INV>(b, buf, lane);
    __syncwarp();
    if (lane < kN1) fft480_store_natural(b, buf, lane);
    __syncwarp();
}

// ---------------------------------------------------------------------------- analysis ----
// grid (ceil(Tf / kAnaWarps), B), block 32 * kAnaWarps.  Warp w transforms frame t0 + w.
// Algorithmic HBM bytes per frame: 1920 R (audio hop) + 3848 W (spec) + 128 W (erb dB).
// Frame window: the grid covers frames [t_begin, t_begin + nf) of every stream (time-chunked execution); their rows
// go to out_t0 ... of spec / erb_db buffers that hold Tbuf frames per stream.  The whole-signal call is
// (t_begin, nf, out_t0, Tbuf) = (0, Tf, 0, Tf).
// Row table (RG: batch path and streaming handles): stream b starts at audio + rows[b].in_off and reads zeros from sample
// rows[b].len on, so the `pad` zeros of enhance() are implicit and no padded copy of the input is needed (its own
// instantiation, so that the table-free kernel of dfb_analysis* is compiled as without it).
template <bool RG>
__global__ void __launch_bounds__(32 * kAnaWarps, 4)
k_analysis(const float *__restrict__ audio, int64_t T, int Tf, float2 *__restrict__ spec,
           float *__restrict__ erb_db, DspTables tb, const float *__restrict__ init_mem, int t_begin, int nf, int out_t0,
           int Tbuf, const RaggedRow *__restrict__ rows) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *s_stage = reinterpret_cast<float *>(smem_raw);                    // (W + 1) * hop
    float *s_win = s_stage + (kAnaWarps + 1) * kHop;                         // fft
    float2 *s_tw960 = reinterpret_cast<float2 *>(s_win + kFft);              // 241 (+1 pad)
    float2 *s_twa = s_tw960 + 242;                                           // pass-A twiddles [24][20]
    float2 *s_buf = s_twa + kN2 * kN1;                                       // W * kTileFloat2
    const int b = blockIdx.y, tl0 = blockIdx.x * kAnaWarps, t0 = t_begin + tl0;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float *x = audio + (RG ? rows[b].in_off : (int64_t)b * T);
    const int64_t s_end = RG ? min((int64_t)Tf * kHop, rows[b].len) : (int64_t)Tf * kHop;
    // stage samples [(t0-1)*hop, (t0+W)*hop); zeros before the stream start (analysis_mem = 0).  All 17 loads of a thread
    // are issued into registers before the first store: as a load / store loop with the bounds checks inside, the compiler
    // kept them in program order -- 17 dependent round trips to L2 / HBM per CTA.
    {
        constexpr int kPre = ((kAnaWarps + 1) * kHop + 32 * kAnaWarps - 1) / (32 * kAnaWarps);
        float pre[kPre];
        const int64_t s0 = (int64_t)(t0 - 1) * kHop;
#pragma unroll
        for (int q = 0; q < kPre; q++) {
            const int i = tid + q * 32 * kAnaWarps;
            const int64_t sidx = s0 + i;
            float v = 0.f;
            if (i < (kAnaWarps + 1) * kHop) {
                if (sidx >= 0 && sidx < s_end) v = __ldg(x + sidx);
                else if (sidx < 0 && init_mem) v = init_mem[(int64_t)b * kHop + (kHop + sidx)];  // carried analysis_mem (reset = False)
            }
            pre[q] = v;
        }
        for (int i = tid; i < kFft; i += blockDim.x) s_win[i] = tb.window[i];
        for (int i = tid; i < 241; i += blockDim.x) s_tw960[i] = tb.tw960[i];
        for (int i = tid; i < kN2 * kN1; i += blockDim.x) s_twa[i] = tb.tw_a_fwd[i];
#pragma unroll
        for (int q = 0; q < kPre; q++) {
            const int i = tid + q * 32 * kAnaWarps;
            if (i < (kAnaWarps + 1) * kHop) s_stage[i] = pre[q];
        }
    }
    __syncthreads();
    const int t = t0 + warp;
    if (tl0 + warp >= nf || t >= Tf) return;
    const int64_t orow = (int64_t)b * Tbuf + out_t0 + tl0 + warp;   // row of this frame in the output buffers
    const float *fr = s_stage + warp * kHop;  // frame t = samples [(t-1) hop, (t+1) hop)
    float2 *nat = s_buf + warp * kTileFloat2;
    warp_fft480_twptr<false>(
        [&](int n) {
            float2 v = *reinterpret_cast<const float2 *>(fr + 2 * n);
            float2 w = *reinterpret_cast<const float2 *>(s_win + 2 * n);
            return make_float2(v.x * w.x, v.y * w.y);
        },
        s_twa + (lane < kN2 ? lane : 0) * kN1, nat, lane);
    // split step + wnorm, write spec row, keep |X|^2 for the band energies
    float2 *row = spec + orow * kF;
    float pk[8], pnk[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        int k = lane + 32 * j;
        pk[j] = pnk[j] = 0.f;
        if (k <= 240) {
            float2 zk = nat[k], znk = nat[(kC - k) % kC];
            float2 xk, xnk;
            rfft_split(zk, znk, s_tw960[k], xk, xnk);
            xk.x *= tb.wnorm; xk.y *= tb.wnorm;
            xnk.x *= tb.wnorm; xnk.y *= tb.wnorm;
            row[k] = xk;
            if (k != 240) row[kC - k] = xnk;
            pk[j] = __fadd_rn(__fmul_rn(xk.x, xk.x), __fmul_rn(xk.y, xk.y));
            pnk[j] = __fadd_rn(__fmul_rn(xnk.x, xnk.x), __fmul_rn(xnk.y, xnk.y));
        }
    }
    if (erb_db == nullptr) return;
    __syncwarp();
    float *P = reinterpret_cast<float *>(nat);  // 481 floats, reuses the natural-order buffer
#pragma unroll
    for (int j = 0; j < 8; j++) {
        int k = lane + 32 * j;
        if (k <= 240) {
            P[k] = pk[j];
            if (k != 240) P[kC - k] = pnk[j];
        }
    }
    __syncwarp();
    // band energies: sequential sum inside each band, factor 1/width inside the sum (lib.rs:288-292)
    for (int band = lane; band < tb.E; band += 32) {
        int o = tb.erb_off[band], n = tb.erb_off[band + 1] - o;
        float kinv = tb.erb_kinv[band];
        float acc = 0.f;
        for (int j = 0; j < n; j++) acc = __fadd_rn(acc, __fmul_rn(P[o + j], kinv));
        erb_db[orow * tb.E + band] = __fmul_rn(log10f(__fadd_rn(acc, 1e-10f)), 10.f);
    }
}

// ----------------------------------------------------------- generic ERB (libdf.erb) ----
// one warp per frame, arbitrary F / E (API parity path, not the hot path)
__global__ void k_erb(const float2 *__restrict__ spec, int64_t n_frames, int F, const int *__restrict__ off,
                      int E, int db, float *__restrict__ out) {
    int64_t fr = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (fr >= n_frames) return;
    const float2 *x = spec + fr * F;
    for (int band = lane; band < E; band += 32) {
        int o = off[band], n = off[band + 1] - o;
        float kinv = __fdiv_rn(1.f, (float)n);
        float acc = 0.f;
        for (int j = 0; j < n; j++) {
            float2 v = x[o + j];
            acc = __fadd_rn(acc, __fmul_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)), kinv));
        }
        out[fr * E + band] = db ? __fmul_rn(log10f(__fadd_rn(acc, 1e-10f)), 10.f) : acc;
    }
}

__global__ void k_erb_inv(const float *__restrict__ gains, int64_t n_frames, int F, int E,
                          const unsigned char *__restrict__ band_of_bin, float *__restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frames * F) return;
    int64_t fr = i / F;
    int k = (int)(i - fr * F);
    out[i] = gains[fr * E + band_of_bin[k]];
}

// ------------------------------------------------------------- polyphase resampler ----
// torchaudio.functional.resample as used by df/io.py:107-129 (the reference resamples files to / from the model rate,
// enhance.py:56,85): out[c][i * nw + j] = sum_k kern[j][k] * xpad[c][i * og + k], xpad = x zero padded by `width` in
// front (torchaudio _apply_sinc_resample_kernel: conv1d with stride og).  kern [nw][K = 2 width + og] is built on the
// host exactly like torchaudio's _get_sinc_resample_kernel (io.py resample_kernel).
__global__ void __launch_bounds__(256) k_resample(const float *__restrict__ x, int64_t T, const float *__restrict__ kern, int og, int nw,
                                                  int width, int K, float *__restrict__ out, int64_t Tout) {
    extern __shared__ float s_k[];   // the nw x K taps when they fit (else read through L1)
    const bool in_smem = (size_t)nw * K * sizeof(float) <= 96 * 1024;
    if (in_smem) {
        for (int i = threadIdx.x; i < nw * K; i += blockDim.x) s_k[i] = kern[i];
        __syncthreads();
    }
    const float *kk = in_smem ? s_k : kern;
    const int c = blockIdx.y;
    const float *xc = x + (int64_t)c * T;
    for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < Tout; n += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = n / nw;
        const int j = (int)(n - i * nw);
        const int64_t p0 = i * og - width;
        const float *kr = kk + (size_t)j * K;
        float acc = 0.f;
        for (int k = 0; k < K; k++) {
            const int64_t p = p0 + k;
            if (p >= 0 && p < T) acc = fmaf(kr[k], xc[p], acc);
        }
        out[(int64_t)c * Tout + n] = acc;
    }
}

// Streaming resampler of a handle at another rate (dfb_stream_set_sample_rate / dfb_stream_add_slot_rate; ResampleDir in
// dfb_common.cuh): one row's call.  x: the call's nin input samples, the first nin_valid of them the session's (the rest
// read as zero: the session's zero extension); s_in0 / s_out0: the session's sample index of x[0] / y[0].  The taps are
// summed as k_resample sums them (fmaf over k = 0 .. K-1, taps outside the session's input skipped), so a streamed session
// is bit for bit k_resample of the whole session, delayed by Z.  y[0, nout_valid) are outputs, y[nout_valid, yw) zeros.
// The history is updated after every thread has read it.
__device__ __forceinline__ void resample_row(const ResampleDir &d, const float *__restrict__ x, int64_t nin, int64_t nin_valid,
                                             float *__restrict__ hist, int64_t s_in0, int64_t s_out0, float *__restrict__ y,
                                             int64_t nout_valid, int64_t yw) {
    const int64_t lim = s_in0 + nin_valid;
    for (int64_t o = threadIdx.x; o < yw; o += blockDim.x) {
        const int64_t t = s_out0 + o;
        float acc = 0.f;
        if (o < nout_valid && t >= d.Z) {
            const int64_t i = t / d.nw;
            const int j = (int)(t - i * d.nw);
            const int64_t p0 = i * d.og - d.S;       // session index of tap 0: >= s_in0 - S, the history's first sample
            const float *kr = d.taps + (size_t)j * d.K;
            for (int k = 0; k < d.K; k++) {
                const int64_t p = p0 + k;
                if (p >= 0 && p < lim) {
                    const int64_t l = p - s_in0;
                    acc = fmaf(__ldg(kr + k), l < 0 ? hist[d.S + l] : x[l], acc);
                }
            }
        }
        y[o] = acc;
    }
    __syncthreads();
    for (int q = threadIdx.x; q < d.S; q += blockDim.x) {   // nin >= S: the new history lies in this call's input
        const int64_t l = nin - d.S + q;
        hist[q] = l < nin_valid ? x[l] : 0.f;
    }
}

// the samples of a row's output from its call's first one on that the call writes: its n hops, then zeros up to out_w
__device__ __forceinline__ int64_t fill_to(const ResampleIO &io, const ResampleDir &d) {
    const int64_t w = io.out_w - io.out_col * d.hop_out, own = io.n * d.hop_out;
    return w > own ? w : own;
}

// rate r -> 48 kHz, each row in its own direction: a session's input ends ext hops before its end hop (a resampled
// session's slot path reads that hop, the zero extension; a 48 kHz row's input ends at its end hop)
__global__ void __launch_bounds__(256) k_resample_up(ResampleDirs dirs, const ResampleRow *__restrict__ rows, ResampleIO io) {
    const ResampleRow r = rows[blockIdx.x];
    const ResampleDir d = dirs.d[r.dir];   // in registers: the tap loops read it every iteration
    const int64_t s = io.a0 - r.first, n = io.n;
    int64_t v = io.in ? r.end - d.ext - io.a0 : 0;
    v = v < 0 ? 0 : (v > n ? n : v);
    resample_row(d, io.in ? io.in + r.slot * io.in_pitch + io.in_col * d.hop_in : nullptr, n * d.hop_in, v * d.hop_in,
                 io.hist + (int64_t)blockIdx.x * io.hist_pitch, s * d.hop_in, s * d.hop_out,
                 io.out + r.slot * io.out_pitch + io.out_col * d.hop_out, n * d.hop_out, fill_to(io, d));
}

// 48 kHz -> rate r, each row in its own direction: the slot path's output rows (zeros past a session's tail); a session's
// output ends `tail` hops after its end hop, and the hops after that are zeros
__global__ void __launch_bounds__(256) k_resample_down(ResampleDirs dirs, const ResampleRow *__restrict__ rows, ResampleIO io) {
    const ResampleRow r = rows[blockIdx.x];
    const ResampleDir d = dirs.d[r.dir];   // in registers: the tap loops read it every iteration
    const int64_t s = io.a0 - r.first, n = io.n;
    int64_t v = r.end + io.tail - io.a0;
    v = v < 0 ? 0 : (v > n ? n : v);
    resample_row(d, io.in + r.slot * io.in_pitch + io.in_col * d.hop_in, n * d.hop_in, n * d.hop_in,
                 io.hist + (int64_t)blockIdx.x * io.hist_pitch, s * d.hop_in, s * d.hop_out,
                 io.out + r.slot * io.out_pitch + io.out_col * d.hop_out, v * d.hop_out, fill_to(io, d));
}

// Offline resampler of a rated batch (dfb_enhance_ragged with rates; RateDir / RateRow / RateIO in dfb_common.cuh; DESIGN.md
// section 5i).  The whole input of a stream is on the device, so no history is carried: an output reads its taps straight
// from the input, and an output is computed once, by the launch in whose range it falls.  Grid (tiles, rows): CTA (x, b)
// writes row b's outputs [o0 + x kRateTile, o0 + (x + 1) kRateTile) of its range [o0, o1), so a row's outputs spread over
// as many CTAs as they fill, and a CTA holds its row's taps in shared memory when they fit.  The sum runs over the taps
// inside the input in k order from +0, which is k_resample's sum with the taps outside skipped.
constexpr int kRateTile = 1024;
template <bool kSmemTaps>
__device__ __forceinline__ void resample_tile(const float *__restrict__ taps, const RateDir &d, const float *__restrict__ x,
                                              int64_t n_in, float *__restrict__ y, int64_t t0, int64_t t1) {
    for (int64_t t = t0 + threadIdx.x; t < t1; t += blockDim.x) {
        const int64_t i = t / d.nw;
        const int j = (int)(t - i * d.nw);
        const int64_t p0 = i * d.og - d.width;
        const int k0 = p0 < 0 ? (int)-p0 : 0;
        const int64_t e = n_in - p0;
        const int k1 = e < d.K ? (int)e : d.K;
        const float *kr = taps + (size_t)j * d.K;
        float acc = 0.f;
        for (int k = k0; k < k1; k++) acc = fmaf(kSmemTaps ? kr[k] : __ldg(kr + k), __ldg(x + p0 + k), acc);
        y[t] = acc;
    }
}

__global__ void __launch_bounds__(256) k_resample_rows(const RateDir *__restrict__ dirs, const RateRow *__restrict__ rows, RateIO io,
                                                       bool up, int smem_floats) {
    const RateRow r = rows[blockIdx.y];
    if (r.dir < 0) return;
    const RateDir d = dirs[r.dir];
    int64_t o0, o1;
    rate_range(up, d, r, io, &o0, &o1);
    const int64_t t0 = o0 + (int64_t)blockIdx.x * kRateTile;
    if (t0 >= o1) return;   // (uniform over the CTA)
    const int64_t t1 = o1 - t0 < kRateTile ? o1 : t0 + kRateTile;
    const float *x = io.in + r.in_off;
    float *y = io.out + r.out_off;
    const int nk = d.nw * d.K;
    if (nk <= smem_floats) {
        extern __shared__ float s_taps[];
        for (int i = threadIdx.x; i < nk; i += blockDim.x) s_taps[i] = __ldg(d.taps + i);
        __syncthreads();
        resample_tile<true>(s_taps, d, x, r.in_len, y, t0, t1);
    } else {
        resample_tile<false>(d.taps, d, x, r.in_len, y, t0, t1);
    }
}

// ------------------------------------------------------------- feature norm scans ----
// Exponential mean norm of the ERB dB features and exponential unit norm of the first Fd bins,
// sequential in t per (stream, band | bin) exactly like the reference loops.
// grid B, block E + Fd threads (thread j < E: band j; else bin j - E).  Loads are batched kPf
// frames ahead so the dependent chain is arithmetic only.
// kPf = frames of loads in flight per thread: 24 for the enhancement path's shape (E + Fd = 128 threads per stream; with 8
// the kernel was latency bound at 0.10 of HBM), 4 for the generic libdf.erb_norm / unit_norm shapes (up to 1024 threads)
// Ts = frames per stream in the four buffers (the pointers are pre-offset to the first frame to process, Tf = number of
// frames processed); *_state_out (may alias the inputs) receive the EMA states after the last frame.
// REF_BITS (the libdf.unit_norm API): |x| as the reference computes it (Complex32::norm -> hypotf of glibc, which rounds
// sqrt(re^2 + im^2) evaluated in double), so that the results are its bits; CUDA's hypotf is within an ulp of it but not
// always the same float.  Separate instantiations: the enhancement path's kernels compile as without it.
__device__ __forceinline__ float norm_ref_bits(float2 v) {
    return __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn((double)v.x, (double)v.x), __dmul_rn((double)v.y, (double)v.y))));
}
// WIDE (E + Fd > 1024: spectra of fft_size > 2046): grid (B, blocks of the E + Fd values), value j = threadIdx.x +
// blockIdx.y * blockDim.x; every value is its own scan, so the results are those of one block.  Separate instantiations.
template <int kPf, bool REF_BITS = false, bool WIDE = false>
__global__ void __launch_bounds__(kPf > 8 ? 128 : 1024) k_feat_norm(const float *erb_in, int E, int64_t erb_stride_t,
                            const float2 *__restrict__ spec_in, int Fd, int64_t spec_stride_t, int Tf,
                            float alpha, const float *erb_state, const float *unit_state,
                            float *feat_erb, float2 *__restrict__ feat_spec, int Ts, float *erb_state_out,
                            float *unit_state_out) {
    const int b = blockIdx.x, j = threadIdx.x + (WIDE ? blockIdx.y * blockDim.x : 0);
    const float one_m_alpha = __fsub_rn(1.f, alpha);
    if (j < E) {
        const float *src = erb_in + (int64_t)b * Ts * erb_stride_t + j;
        float *dst = feat_erb + (int64_t)b * Ts * E + j;
        float s;
        if (erb_state) s = erb_state[(int64_t)b * E + j];
        else s = erb_norm_init(j, E);
        // software pipelined: the loads of batch n + 1 are in flight while batch n runs its (sequential) EMA
        float vn[kPf];
#pragma unroll
        for (int u = 0; u < kPf; u++) vn[u] = (u < Tf) ? src[(int64_t)u * erb_stride_t] : 0.f;
        for (int t = 0; t < Tf; t += kPf) {
            float v[kPf];
#pragma unroll
            for (int u = 0; u < kPf; u++) {
                v[u] = vn[u];
                vn[u] = (t + kPf + u < Tf) ? src[(int64_t)(t + kPf + u) * erb_stride_t] : 0.f;
            }
#pragma unroll
            for (int u = 0; u < kPf; u++) {
                if (t + u < Tf) {
                    s = __fadd_rn(__fmul_rn(v[u], one_m_alpha), __fmul_rn(s, alpha));
                    dst[(int64_t)(t + u) * E] = __fdiv_rn(__fsub_rn(v[u], s), 40.f);
                }
            }
        }
        if (erb_state_out) erb_state_out[(int64_t)b * E + j] = s;
    } else if (j < E + Fd) {
        const int k = j - E;
        const float2 *src = spec_in + (int64_t)b * Ts * spec_stride_t + k;
        float2 *dst = feat_spec + (int64_t)b * Ts * Fd + k;
        float s;
        if (unit_state) s = unit_state[(int64_t)b * Fd + k];
        else s = unit_norm_init(k, Fd);
        float2 vn[kPf];
#pragma unroll
        for (int u = 0; u < kPf; u++) vn[u] = (u < Tf) ? src[(int64_t)u * spec_stride_t] : make_float2(0.f, 0.f);
        for (int t = 0; t < Tf; t += kPf) {
            float2 v[kPf];
            float nrm[kPf], sv[kPf];
#pragma unroll
            for (int u = 0; u < kPf; u++) {
                v[u] = vn[u];
                vn[u] = (t + kPf + u < Tf) ? src[(int64_t)(t + kPf + u) * spec_stride_t] : make_float2(0.f, 0.f);
            }
            // the magnitudes and the normalisation are independent across frames; only the two-op EMA chain is serial
#pragma unroll
            for (int u = 0; u < kPf; u++) {
                if constexpr (REF_BITS) nrm[u] = norm_ref_bits(v[u]);
                else nrm[u] = hypotf(v[u].x, v[u].y);
            }
#pragma unroll
            for (int u = 0; u < kPf; u++) {
                if (t + u < Tf) s = __fadd_rn(__fmul_rn(nrm[u], one_m_alpha), __fmul_rn(s, alpha));
                sv[u] = s;
            }
#pragma unroll
            for (int u = 0; u < kPf; u++) {
                if (t + u < Tf) {
                    float d = __fsqrt_rn(sv[u]);
                    dst[(int64_t)(t + u) * Fd] = make_float2(__fdiv_rn(v[u].x, d), __fdiv_rn(v[u].y, d));
                }
            }
        }
        if (unit_state_out) unit_state_out[(int64_t)b * Fd + k] = s;
    }
}

// Time-segmented version for the enhancement path's shape (E + Fd <= 128 values per stream, long windows): the EMA is a
// linear recurrence, so a stream's frames are cut into kSeg segments scanned concurrently by kSeg x 128 threads --
//   pass 1: every (segment, value) thread runs the recurrence over its segment from state 0 (no stores) -> local end state
//   fold:   state at the start of segment g = alpha^(frames before) * s_in + sum of the earlier local end states, each
//           decayed by alpha^(frames after it) (evaluated in double: at most kSeg terms per thread)
//   pass 2: the same loop as k_feat_norm from the segment's true start state, with the reference's operation order, storing
//           the features (the inputs are re-read from L2)
// The serial chain per thread drops from Tf to 2 Tf / kSeg steps; the results differ from
// the one-thread scan only through the rounding of the folded start states (~1e-7 relative).
constexpr int kNormSeg = 8, kNormPf = 8;
template <bool WRITE>
__device__ __forceinline__ float norm_scan_erb(const float *src, int64_t stride, float *dst, int E, int ta, int tb, float s, float alpha,
                                               float one_m_alpha) {
    float vn[kNormPf];
#pragma unroll
    for (int u = 0; u < kNormPf; u++) vn[u] = (ta + u < tb) ? src[(int64_t)(ta + u) * stride] : 0.f;
    for (int t = ta; t < tb; t += kNormPf) {
        float v[kNormPf];
#pragma unroll
        for (int u = 0; u < kNormPf; u++) {
            v[u] = vn[u];
            vn[u] = (t + kNormPf + u < tb) ? src[(int64_t)(t + kNormPf + u) * stride] : 0.f;
        }
#pragma unroll
        for (int u = 0; u < kNormPf; u++) {
            if (t + u < tb) {
                s = __fadd_rn(__fmul_rn(v[u], one_m_alpha), __fmul_rn(s, alpha));
                if (WRITE) dst[(int64_t)(t + u) * E] = __fdiv_rn(__fsub_rn(v[u], s), 40.f);
            }
        }
    }
    return s;
}
template <bool WRITE>
__device__ __forceinline__ float norm_scan_unit(const float2 *src, int64_t stride, float2 *dst, int Fd, int ta, int tb, float s, float alpha,
                                                float one_m_alpha) {
    float2 vn[kNormPf];
#pragma unroll
    for (int u = 0; u < kNormPf; u++) vn[u] = (ta + u < tb) ? src[(int64_t)(ta + u) * stride] : make_float2(0.f, 0.f);
    for (int t = ta; t < tb; t += kNormPf) {
        float2 v[kNormPf];
        float nrm[kNormPf], sv[kNormPf];
#pragma unroll
        for (int u = 0; u < kNormPf; u++) {
            v[u] = vn[u];
            vn[u] = (t + kNormPf + u < tb) ? src[(int64_t)(t + kNormPf + u) * stride] : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < kNormPf; u++) nrm[u] = hypotf(v[u].x, v[u].y);
#pragma unroll
        for (int u = 0; u < kNormPf; u++) {
            if (t + u < tb) s = __fadd_rn(__fmul_rn(nrm[u], one_m_alpha), __fmul_rn(s, alpha));
            sv[u] = s;
        }
        if (WRITE) {
#pragma unroll
            for (int u = 0; u < kNormPf; u++) {
                if (t + u < tb) {
                    const float d = __fsqrt_rn(sv[u]);
                    dst[(int64_t)(t + u) * Fd] = make_float2(__fdiv_rn(v[u].x, d), __fdiv_rn(v[u].y, d));
                }
            }
        }
    }
    return s;
}
__global__ void __launch_bounds__(128 * kNormSeg) k_feat_norm_seg(const float *erb_in, int E, int64_t erb_stride_t,
                            const float2 *__restrict__ spec_in, int Fd, int64_t spec_stride_t, int Tf,
                            float alpha, const float *erb_state, const float *unit_state,
                            float *feat_erb, float2 *__restrict__ feat_spec, int Ts, float *erb_state_out,
                            float *unit_state_out) {
    __shared__ float s_loc[kNormSeg][128];
    const int b = blockIdx.x, j = threadIdx.x & 127, seg = threadIdx.x >> 7;
    const float one_m_alpha = __fsub_rn(1.f, alpha);
    const int L = (Tf + kNormSeg - 1) / kNormSeg;
    const int ta = min(seg * L, Tf), tb = min(ta + L, Tf);
    const bool is_erb = j < E, is_unit = !is_erb && j < E + Fd;
    const float *esrc = erb_in + (int64_t)b * Ts * erb_stride_t + j;
    float *edst = feat_erb + (int64_t)b * Ts * E + j;
    const int k = j - E;
    const float2 *usrc = spec_in + (int64_t)b * Ts * spec_stride_t + k;
    float2 *udst = feat_spec + (int64_t)b * Ts * Fd + k;
    float loc = 0.f;
    if (seg + 1 < kNormSeg) {   // the last segment's local end state is never folded
        if (is_erb) loc = norm_scan_erb<false>(esrc, erb_stride_t, nullptr, E, ta, tb, 0.f, alpha, one_m_alpha);
        else if (is_unit) loc = norm_scan_unit<false>(usrc, spec_stride_t, nullptr, Fd, ta, tb, 0.f, alpha, one_m_alpha);
    }
    s_loc[seg][j] = loc;
    __syncthreads();
    if (!is_erb && !is_unit) return;
    float s0;
    if (is_erb) {
        if (erb_state) s0 = erb_state[(int64_t)b * E + j];
        else s0 = erb_norm_init(j, E);
    } else {
        if (unit_state) s0 = unit_state[(int64_t)b * Fd + k];
        else s0 = unit_norm_init(k, Fd);
    }
    if (seg > 0) {
        double sd = (double)s0;
        const double pL = pow((double)alpha, (double)L);
        for (int g = 0; g < seg; g++) {   // segment g covers min(L, Tf - g L) frames
            const int lg = min(L, max(Tf - g * L, 0));
            sd = sd * (lg == L ? pL : pow((double)alpha, (double)lg)) + (double)s_loc[g][j];
        }
        s0 = (float)sd;
    }
    float s;
    if (is_erb) s = norm_scan_erb<true>(esrc, erb_stride_t, edst, E, ta, tb, s0, alpha, one_m_alpha);
    else s = norm_scan_unit<true>(usrc, spec_stride_t, udst, Fd, ta, tb, s0, alpha, one_m_alpha);
    if (seg == kNormSeg - 1 || tb == Tf) {   // the thread whose segment ends the window owns the carried state
        if (ta < tb || seg == 0) {
            if (is_erb && erb_state_out) erb_state_out[(int64_t)b * E + j] = s;
            if (is_unit && unit_state_out) unit_state_out[(int64_t)b * Fd + k] = s;
        }
    }
}

// ------------------------------------------------------ fused apply + synthesis ----
// mode 0: plain ISTFT of `spec` (pyDF DF.synthesis)
// mode 1: DeepFilterNet3: bins < nb_df <- deep filter of the NOISY spectrum, bins >= nb_df <- spec * gain
// mode 2: DeepFilterNet2: spectrum masked first (all bins), deep filter applied to the masked spectrum
// Optional attenuation limit: X <- noisy * lim + X * (1 - lim)   (enhance.py:238-240)
// One warp owns kSynChunk consecutive frames of one stream and keeps the overlap tail in registers;
// it re-synthesises frame t0-1 to obtain the tail of its first frame.
// Algorithmic HBM bytes per frame (mode 1/2): 3848 R spec + 128 R m + 3840 R coefs + 1920 W audio.

// Valin's post filter on an ERB gain (Mask.pf, modules.py:234-245).  __sinf on [0, pi/2] is within 2^-21 absolute; the
// accurate sinf / hypotf (argument-reduction slow paths, 16 inlined copies in the unrolled bin loop) bloated the apply kernel
// past the instruction cache and cost 30 % even with the filter off.
__device__ __forceinline__ float pf_gain_mask(float m, float beta) {
    const float ms = fmaxf(m * __sinf(3.14159265358979f * m / 2.f), 1e-12f);
    const float q = m / ms;
    return (1.f + beta) * m / (1.f + beta * q * q);
}
// ... and on an enhanced bin y of the noisy bin x (deepfilternet3.py:448-454): returns the factor for y
__device__ __forceinline__ float pf_gain_spec(float2 y, float2 x, float beta) {
    const float eps = 1e-12f;
    const float mask = fminf(fmaxf(sqrtf(y.x * y.x + y.y * y.y) / (sqrtf(x.x * x.x + x.y * x.y) + eps), eps), 1.f);
    const float ms = mask * fmaxf(__sinf(3.14159265358979f * mask / 2.f), eps);
    const float q = mask / ms;
    return (1.f + beta) / (1.f + beta * q * q);
}

__device__ __forceinline__ float2 apply_bin(const ApplyParams &p, const DspTables &tb, const float2 *srow0,
                                            const float *mrow0, const float *crow, int t, int k, int Tv) {
    // srow0 / mrow0: row pointers of frame 0 of this stream; spectrum rows >= Tv do not exist
    float2 x = srow0[(int64_t)t * kF + k];
    float2 y;
    if (p.mode == 0) return x;
    const int band = tb.band_of_bin[k];
    const bool pf2 = p.pf && p.mode == 2;
    if (k >= p.nb_df || p.mask_only) {
        float g = mrow0[(int64_t)t * tb.E + band];
        if (pf2) g = pf_gain_mask(g, 0.02f);
        y = make_float2(x.x * g, x.y * g);
    } else {
        // Y[t,k] = sum_o S[t + o - (O-1-L), k] * W[o,t,k]   (multiframe.py:72-74,126-136)
        const float *c = crow + (int64_t)k * (2 * p.order);
        float yr = 0.f, yi = 0.f;
        for (int o = 0; o < p.order; o++) {
            int tt = t + o - (p.order - 1 - p.lookahead);
            if (tt < 0 || tt >= Tv) continue;
            float2 s = srow0[(int64_t)tt * kF + k];
            if (p.mode == 2 && tt < (p.mc_T ? p.mc_T : p.Tf)) {
                float g = mrow0[(int64_t)tt * tb.E + band];
                if (pf2) g = pf_gain_mask(g, 0.02f);
                s.x *= g; s.y *= g;
            }
            float wr = c[2 * o], wi = c[2 * o + 1];
            yr += s.x * wr - s.y * wi;
            yi += s.x * wi + s.y * wr;
        }
        y = make_float2(yr, yi);
        if (p.alpha && p.mode == 2) {
            const float a = p.alpha[(mrow0 - p.m) / tb.E + t];   // same [b][mc_T] indexing as the mask rows
            float g = mrow0[(int64_t)t * tb.E + band];
            if (pf2) g = pf_gain_mask(g, 0.02f);
            y.x = y.x * a + x.x * g * (1.f - a);
            y.y = y.y * a + x.y * g * (1.f - a);
        }
    }
    if (p.pf && p.mode == 1) { const float g = pf_gain_spec(y, x, p.pf_beta); y.x *= g; y.y *= g; }
    if (p.atten_lim > 0.f) {
        y.x = x.x * p.atten_lim + y.x * (1.f - p.atten_lim);
        y.y = x.y * p.atten_lim + y.y * (1.f - p.atten_lim);
    }
    return y;
}

__global__ void __launch_bounds__(32 * kSynWarps) k_apply_synthesis_generic(ApplyParams p, DspTables tb) {
    __shared__ __align__(16) float s_win[kFft];
    __shared__ __align__(16) float2 s_tw960[241];
    __shared__ __align__(16) float2 s_buf[kSynWarps][kTileFloat2];
    const int b = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < kFft; i += blockDim.x) s_win[i] = tb.window[i];
    for (int i = tid; i < 241; i += blockDim.x) s_tw960[i] = tb.tw960[i];
    float2 tw[kN1];
#pragma unroll
    for (int k1 = 0; k1 < kN1; k1++) tw[k1] = lane < kN2 ? tb.tw_a_inv[lane * kN1 + k1] : make_float2(0.f, 0.f);
    __syncthreads();
    const int syn_chunk = p.frames_per_warp ? p.frames_per_warp : kSynChunk;
    const int t0 = (blockIdx.x * kSynWarps + warp) * syn_chunk;
    int Te = p.Tf, Tv = p.Tv ? p.Tv : p.Tf;     // frames this stream synthesises / spectrum rows that exist
    float *orow = p.audio ? p.audio + (int64_t)b * p.out_stride : nullptr;
    int64_t out_len = p.out_len;
    int t_zero = INT_MIN;   // frames before it synthesise to zero (streaming slots; t may be -1 for the carried tail)
    if (p.rows) {
        const RaggedRow r = p.rows[b];
        const int tfb = (int)(r.Tf - p.w0);
        if (p.first) t_zero = stream_first(p.first, b, p.w0);
        Te = tfb <= p.Tf ? tfb : p.t_emit;
        Tv = min(Tv, tfb);
        if (orow) orow = p.audio + r.out_off;
        out_len = r.out_len;
    }
    if (t0 >= Te) return;
    const int t1 = min(t0 + syn_chunk, Te);
    const float2 *srow0 = p.spec + (int64_t)b * (p.spec_T ? p.spec_T : p.Tf) * kF;
    const int mcT = p.mc_T ? p.mc_T : p.Tf;
    const float *mrow0 = p.m ? p.m + (int64_t)b * mcT * tb.E : nullptr;
    float2 *nat = s_buf[warp];
    float *yb = reinterpret_cast<float *>(nat);  // 960 windowed samples of the current frame
    float tail[15];
#pragma unroll
    for (int j = 0; j < 15; j++) tail[j] = (p.carry && t0 == 0 && b == 0 && p.init_tail) ? p.init_tail[lane + 32 * j] : 0.f;
    // carried state: channel b > 0 continues from the tail of channel b - 1's last frame, which is row -1
    // relative to this channel in the contiguous [C,Tf,F] spectrum (mode 0 only)
    const int tstart = t0 > 0 ? t0 - 1 : ((p.carry && b > 0) ? -1 : 0);
    for (int t = tstart; t < t1; t++) {
        const float *crow = p.coefs ? p.coefs + ((int64_t)b * mcT + t) * p.nb_df * (2 * p.order) : nullptr;
        // gather X[k], X[480-k], merge into Z (natural order in `nat`)
#pragma unroll
        for (int j = 0; j < 8; j++) {
            int k = lane + 32 * j;
            if (k <= 240) {
                float2 xk = apply_bin(p, tb, srow0, mrow0, crow, t, k, Tv);
                float2 xnk = apply_bin(p, tb, srow0, mrow0, crow, t, kC - k, Tv);
                if (t < t_zero) xk = xnk = make_float2(0.f, 0.f);
                if (p.spec_out && t >= t0) {
                    float2 *orow = p.spec_out + ((int64_t)b * p.Tf + t) * kF;
                    orow[k] = xk;
                    orow[kC - k] = xnk;
                }
                if (k == 0) { xk.y = 0.f; xnk.y = 0.f; }  // imag of DC / Nyquist ignored (lib.rs:402)
                float2 w = s_tw960[k];
                float2 zk, znk;
                irfft_merge(xk, xnk, make_float2(w.x, -w.y), zk, znk);
                nat[k] = zk;
                if (k > 0 && k < 240) nat[kC - k] = znk;
            }
        }
        __syncwarp();
        if (p.audio) {
            // reads of nat complete inside pass A before pass B overwrites it (warp syncs inside)
            warp_fft480<true>([&](int n) { return nat[n]; }, tw, nat, lane);
            // nat[n] = (x[2n], x[2n+1]); window in place
#pragma unroll
            for (int j = 0; j < 15; j++) {
                int n = lane + 32 * j;
                float2 v = nat[n];
                float2 w = *reinterpret_cast<const float2 *>(s_win + 2 * n);
                nat[n] = make_float2(v.x * w.x, v.y * w.y);
            }
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 15; j++) {
                int i = lane + 32 * j;
                float o = yb[i] + tail[j];      // lib.rs:407-411
                tail[j] = yb[kHop + i];         // lib.rs:423-426 (hop == fft/2)
                int64_t g = (int64_t)t * kHop + i - p.out_offset;
                if (t >= t0 && t >= p.t_first && g >= 0 && g < out_len) orow[g] = o;
            }
        }
        __syncwarp();
    }
    if (p.final_tail && b == (int)gridDim.y - 1 && t1 == p.Tf) {
#pragma unroll
        for (int j = 0; j < 15; j++) p.final_tail[lane + 32 * j] = tail[j];
    }
}

// Specialised version for the shipped models (df_order 5, nb_df 96, 32 ERB bands): a lane owns the bins
// k = lane + 32 j (and 480 - k) for every frame of its chunk, so the deep-filter input history of its DF
// bins lives in registers as a 5-deep shift register (one new look-ahead value per bin and frame instead of
// five reloads), the band gains come from one register per lane via warp shuffles, and all global loads of
// a frame are issued up front, coalesced (256-byte rows), before any use.
// RG: row table (p.rows: batch path and streaming handles), a separate instantiation so that the table-free kernel of
// dfb_apply and dfb_model_forward_full compiles exactly as without it.
// LINK: linked channels (p.links, with RG), likewise separate.  The mask of a frame is reduced over the link group where it is
// loaded: lane e reads row e of each member's mask and reduces in registers, so the shared mask never reaches HBM and
// the unlinked instantiations are untouched.
// CTL: per-stream attenuation limit, post-filter beta and LSNR gating thresholds (ctl_tab: streaming slots, and batches
// with a settings table), likewise separate.  Each frame picks the row's new or previous limit and beta by its absolute
// frame against the row's switch frame; with the LSNR head on (p.lsnr), a row gates when its entry says so.
template <int ORDER, int NDFJ, int MINB, bool RG, bool LINK = false, bool CTL = false>
__global__ void __launch_bounds__(32 * kSynWarps, MINB) k_apply_synthesis(ApplyParams p, DspTables tb, const SlotCtl *ctl_tab) {
    __shared__ __align__(16) float s_win[kFft];
    __shared__ __align__(16) float2 s_tw960[241];
    __shared__ __align__(16) float2 s_buf[kSynWarps][kTileFloat2];
    __shared__ __align__(16) float2 s_twa[kN2 * kN1];  // pass-A twiddles, reloaded into registers per frame
    const int b = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < kFft; i += blockDim.x) s_win[i] = tb.window[i];
    for (int i = tid; i < 241; i += blockDim.x) s_tw960[i] = tb.tw960[i];
    for (int i = tid; i < kN2 * kN1; i += blockDim.x) s_twa[i] = tb.tw_a_inv[i];
    __syncthreads();
    const int syn_chunk = p.frames_per_warp ? p.frames_per_warp : kSynChunk;
    const int t0 = (blockIdx.x * kSynWarps + warp) * syn_chunk;
    const int Tf = p.Tf, L = p.lookahead, back = ORDER - 1 - L;
    int Te = Tf, Tv = p.Tv ? p.Tv : Tf;                    // frames synthesised; spectrum rows >= Tv do not exist (end of the stream)
    int64_t orow0 = (int64_t)b * p.out_stride, out_len = p.out_len;
    int t_zero = 0;                                        // streaming slots: frames before it synthesise to zero
    if constexpr (RG) {                                    // ragged batch: this stream's own end and output row
        t_zero = stream_first(p.first, b, p.w0);
        const RaggedRow r = p.rows[b];
        const int tfb = (int)(r.Tf - p.w0);
        Te = tfb <= Tf ? tfb : p.t_emit;
        Tv = min(Tv, tfb);
        orow0 = r.out_off;
        out_len = r.out_len;
    }
    if (t0 >= Te) return;
    const int t1 = min(t0 + syn_chunk, Te);
    const float2 *srow0 = p.spec + (int64_t)b * (p.spec_T ? p.spec_T : Tf) * kF;
    const int mcT = p.mc_T ? p.mc_T : Tf;                  // m / coefs rows per stream
    const float *mrow0 = p.m + (int64_t)b * mcT * 32;
    int lb = b;                                            // stream whose LSNR gates this one: the link group's first
    if constexpr (LINK) lb = p.links[b].first;
    // ERB gain of band `lane` in frame tt: this stream's own, or (LINK) the link group's max / mean in channel order,
    // the mean as the fp32 sum times fl32(1 / n) (tract.rs:881-898)
    auto mask_at = [&](int tt) -> float {
        if constexpr (!LINK) {
            return mrow0[(int64_t)tt * 32 + lane];
        } else {
            const int n = p.links[b].n;
            const int64_t stride = (int64_t)mcT * 32;
            const float *q = p.m + (int64_t)lb * stride + (int64_t)tt * 32 + lane;
            float v = q[0];
            if (p.reduce == kReduceMax) {
                for (int c = 1; c < n; c++) v = fmaxf(v, q[c * stride]);
                return v;
            }
            for (int c = 1; c < n; c++) v += q[c * stride];
            return v * __frcp_rn((float)n);
        }
    };
    const bool masked_df = p.mode == 2 && !p.mask_only;
    // CTL: this row's settings (either of its two) in place of the handle's limit and DeepFilterNet3 post filter
    const SlotCtl ctl = CTL ? ctl_tab[b] : SlotCtl{};
    const bool pf1 = CTL ? p.mode == 1 && (ctl.beta > 0.f || ctl.beta0 > 0.f) : p.pf && p.mode == 1, pf2 = p.pf && p.mode == 2;
    const bool blend = p.alpha != nullptr && masked_df;   // DeepFilterNet v1: alpha blend with the masked bin
    const bool need_xk = (CTL ? ctl.lim > 0.f || ctl.lim0 > 0.f : p.atten_lim > 0.f) || pf1 || p.mask_only || p.lsnr || blend;   // noisy DF bins are only loaded when something reads them
    // bands of this lane's bins: bk[j] for k = lane + 32 j, bn[j] for 480 - k
    unsigned long long bkp = 0, bnp = 0;  // 8 band indices each, one byte per j
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int k = lane + 32 * j;
        bkp |= (unsigned long long)(k <= 240 ? tb.band_of_bin[k] : 0) << (8 * j);
        bnp |= (unsigned long long)(k <= 240 ? tb.band_of_bin[kC - k] : 0) << (8 * j);
    }
#define BK(j) ((int)((bkp >> (8 * (j))) & 0xff))
#define BN(j) ((int)((bnp >> (8 * (j))) & 0xff))
    float2 *nat = s_buf[warp];
    float *yb = reinterpret_cast<float *>(nat);
    float tail[15];
#pragma unroll
    for (int j = 0; j < 15; j++) tail[j] = 0.f;
    // S'[tt][k] for the DF bins; tt = t + o - back.  Rows outside [0, Tf) are zero (multiframe.py:72-74).
    auto load_df_row = [&](int tt, float2 (&dst)[NDFJ]) {
        float g = 1.f;
        const bool ok = tt >= 0 && tt < Tv;
        // (DFN2) the mask of a look-ahead frame beyond the window's DNN frames does not exist yet: such rows are only
        // read for frames that are re-synthesised in the next window
        float mrow = (ok && masked_df && tt < mcT) ? mask_at(tt) : 1.f;
        if (pf2 && ok && masked_df && tt < mcT) mrow = pf_gain_mask(mrow, 0.02f);
#pragma unroll
        for (int j = 0; j < NDFJ; j++) {
            float2 v = ok ? srow0[(int64_t)tt * kF + lane + 32 * j] : make_float2(0.f, 0.f);
            if (masked_df) { g = __shfl_sync(0xffffffffu, mrow, BK(j)); v.x *= g; v.y *= g; }
            dst[j] = v;
        }
    };
    const int tstart = t0 > 0 ? t0 - 1 : 0;
    float2 hist[ORDER][NDFJ];
#pragma unroll
    for (int o = 1; o < ORDER; o++) load_df_row(tstart + o - 1 - back, hist[o]);  // becomes taps 0..O-2 after the first shift
    for (int t = tstart; t < t1; t++) {
        // ---- loads of this frame, all issued before use
        float mcur = mask_at(t);
        if (pf2) mcur = pf_gain_mask(mcur, 0.02f);
        const float al = blend ? p.alpha[(int64_t)b * mcT + t] : 1.f;
        int stage = 3;   // 0 zero gains, 1 unprocessed, 2 gains only, 3 gains + deep filter (tract.rs apply_stages)
        if (p.lsnr && (!CTL || ctl.gate)) {   // CTL: the row's own thresholds
            const float l = p.lsnr[(int64_t)lb * mcT + t];
            const float th_min = CTL ? ctl.th_min : p.th_min, th_erb = CTL ? ctl.th_erb : p.th_erb, th_df = CTL ? ctl.th_df : p.th_df;
            stage = l < th_min ? 0 : (l > th_erb ? 1 : (l > th_df ? 2 : 3));
        }
        if (RG && t < t_zero) stage = 0;   // zero gains, no deep filter: the stream has not started
        // CTL: the setting frame t was output with; the frame before the switch is only re-synthesised for its tail
        const bool now = CTL && p.w0 + t >= ctl.sw;
        const float lim = now ? ctl.lim : ctl.lim0, beta = now ? ctl.beta : ctl.beta0;
#pragma unroll
        for (int o = 0; o < ORDER - 1; o++)
#pragma unroll
            for (int j = 0; j < NDFJ; j++) hist[o][j] = hist[o + 1][j];
        load_df_row(t + L, hist[ORDER - 1]);
        float2 cf[NDFJ][ORDER];
        const float2 *crow = reinterpret_cast<const float2 *>(p.coefs + ((int64_t)b * mcT + t) * (NDFJ * 32) * (2 * ORDER));
#pragma unroll
        for (int j = 0; j < NDFJ; j++)
#pragma unroll
            for (int o = 0; o < ORDER; o++) cf[j][o] = crow[(lane + 32 * j) * ORDER + o];
        float2 xk[8], xn[8];
        const float2 *srow = srow0 + (int64_t)t * kF;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int k = lane + 32 * j;
            xk[j] = (k <= 240 && (j >= NDFJ || need_xk)) ? srow[k] : make_float2(0.f, 0.f);
            xn[j] = k <= 240 ? srow[kC - k] : make_float2(0.f, 0.f);
        }
        // ---- deep filter (bins < 96), gain (others), optional attenuation limit
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int k = lane + 32 * j;
            float2 y;
            if (j < NDFJ && !p.mask_only && stage == 3) {
                float yr = 0.f, yi = 0.f;
#pragma unroll
                for (int o = 0; o < ORDER; o++) {
                    const float2 s = hist[o][j], w = cf[j][o];
                    yr += s.x * w.x - s.y * w.y;
                    yi += s.x * w.y + s.y * w.x;
                }
                y = make_float2(yr, yi);
                if (blend) {
                    const float g = __shfl_sync(0xffffffffu, mcur, BK(j)) * (1.f - al);
                    y.x = y.x * al + xk[j].x * g; y.y = y.y * al + xk[j].y * g;
                }
            } else {
                const float g = __shfl_sync(0xffffffffu, mcur, BK(j));
                y = make_float2(xk[j].x * g, xk[j].y * g);
            }
            const float gn = __shfl_sync(0xffffffffu, mcur, BN(j));
            float2 yn = make_float2(xn[j].x * gn, xn[j].y * gn);
            if (stage == 0) { y = make_float2(0.f, 0.f); yn = y; }
            else if (stage == 1) { y = xk[j]; yn = xn[j]; }
            if ((CTL ? p.mode == 1 && beta > 0.f : pf1) && stage >= 2) {
                const float g1 = pf_gain_spec(y, xk[j], CTL ? beta : p.pf_beta), g2 = pf_gain_spec(yn, xn[j], CTL ? beta : p.pf_beta);
                y.x *= g1; y.y *= g1; yn.x *= g2; yn.y *= g2;
            }
            if (CTL ? lim > 0.f : p.atten_lim > 0.f) {
                const float a = CTL ? lim : p.atten_lim, c = 1.f - a;
                y.x = xk[j].x * a + y.x * c; y.y = xk[j].y * a + y.y * c;
                yn.x = xn[j].x * a + yn.x * c; yn.y = xn[j].y * a + yn.y * c;
            }
            if (k <= 240) {
                if (p.spec_out && t >= t0) {
                    float2 *orow = p.spec_out + ((int64_t)b * Tf + t) * kF;
                    orow[k] = y;
                    orow[kC - k] = yn;
                }
                if (k == 0) { y.y = 0.f; yn.y = 0.f; }  // imag of DC / Nyquist ignored (lib.rs:402)
                const float2 w = s_tw960[k];
                float2 zk, znk;
                irfft_merge(y, yn, make_float2(w.x, -w.y), zk, znk);
                nat[k] = zk;
                if (k > 0 && k < 240) nat[kC - k] = znk;
            }
        }
        __syncwarp();
        if (p.audio) {
            warp_fft480_twptr<true>([&](int n) { return nat[n]; }, s_twa + (lane < kN2 ? lane : 0) * kN1, nat, lane);
#pragma unroll
            for (int j = 0; j < 15; j++) {
                int n = lane + 32 * j;
                float2 v = nat[n];
                float2 w = *reinterpret_cast<const float2 *>(s_win + 2 * n);
                nat[n] = make_float2(v.x * w.x, v.y * w.y);
            }
            __syncwarp();
            float *orow = p.audio + orow0;
#pragma unroll
            for (int j = 0; j < 15; j++) {
                int i = lane + 32 * j;
                float o = yb[i] + tail[j];      // lib.rs:407-411
                tail[j] = yb[kHop + i];         // lib.rs:423-426 (hop == fft/2)
                int64_t g = (int64_t)t * kHop + i - p.out_offset;
                if (t >= t0 && t >= p.t_first && g >= 0 && g < out_len) orow[g] = o;
            }
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------- generic STFT / ISTFT ----
// Every (fft_size N, hop H) other than 960 / 480: the real FFT of dfb_fft_generic.cuh, one CTA per group of G frames of
// one stream, all G frames transformed together (every Stockham stage is one pass of the CTA's threads over the G M / R
// butterflies, then a barrier).  Shared memory: two ping-pong buffers of G x M complex values (G = gen_frames(M): about
// kGenCplx values, 32 KB), plus for the synthesis two overlap-add tails of N - H samples.
constexpr int kGenThreads = 256;
constexpr int kGenCplx = 2048;
constexpr int kGenSmemMax = 200 * 1024;   // odd N = 8191: 2 x 8191 x 8 B of buffers + 2 x 8190 x 4 B of tails
inline int gen_frames(int M) { return std::max(1, std::min(32, kGenCplx / M)); }

// grid (ceil(Tf / G), B), kGenThreads threads.  Frame t = window x samples [t H - (N - H), t H + H) of stream b, zeros
// (or init_mem [B][N - H], the carried analysis memory) before sample 0; spec [B][Tf][F] = wnorm * rfft; erb_db (or null)
// [B][Tf][E] = the ERB dB of the spectrum (lib.rs:280-295, 207-210), from the band energies kept in shared memory.
__global__ void __launch_bounds__(kGenThreads) k_analysis_gen(const float *__restrict__ audio, int64_t T, int Tf,
                                                              float2 *__restrict__ spec, float *__restrict__ erb_db, DspTables tb,
                                                              GenFftPlan pl, int G, const float *__restrict__ init_mem) {
    extern __shared__ __align__(16) float2 gsm[];
    __shared__ int s_rad[kGenMaxStages];
    const int N = pl.N, M = pl.M, H = tb.hop, F = tb.F, mem = N - H;
    const int b = blockIdx.y, t0 = blockIdx.x * G, nf = min(G, Tf - t0);
    float2 *A = gsm, *Bf = gsm + G * M;
    gen_load_radices(pl, s_rad);
    const float *x = audio + (int64_t)b * T;
    for (int i = threadIdx.x; i < nf * N; i += blockDim.x) {
        const int f = i / N, n = i - f * N;
        const int64_t s = (int64_t)(t0 + f) * H - mem + n;
        float v = 0.f;
        if (s >= 0) v = __ldg(x + s);
        else if (init_mem) v = init_mem[(int64_t)b * mem + mem + s];
        v = __fmul_rn(v, __ldg(tb.window + n));
        if (N % 2 == 0) reinterpret_cast<float *>(A + f * M)[n] = v;   // z[n / 2] = (x[2 (n / 2)], x[2 (n / 2) + 1])
        else A[f * M + n] = make_float2(v, 0.f);
    }
    __syncthreads();
    float2 *Z = gen_block_fft<false>(A, Bf, pl, s_rad, nf);
    float *P = reinterpret_cast<float *>(Z == A ? Bf : A);   // |X|^2 of every bin, F floats per frame
    const float wn = tb.wnorm;
    auto emit = [&](int f, int k, float2 v) {
        v.x *= wn; v.y *= wn;
        spec[((int64_t)b * Tf + t0 + f) * F + k] = v;
        P[f * F + k] = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
    };
    if (N % 2 == 0) {
        const int nk = M / 2 + 1;   // k in [0, M / 2] gives X[k] and X[M - k]
        for (int i = threadIdx.x; i < nf * nk; i += blockDim.x) {
            const int f = i / nk, k = i - f * nk;
            float2 xk, xnk;
            rfft_split(Z[f * M + k], Z[f * M + (M - k) % M], __ldg(pl.tw + k), xk, xnk);
            emit(f, k, xk);
            if (M - k != k) emit(f, M - k, xnk);
        }
    } else {
        for (int i = threadIdx.x; i < nf * F; i += blockDim.x) {
            const int f = i / F, k = i - f * F;
            emit(f, k, Z[f * M + k]);
        }
    }
    if (erb_db == nullptr) return;
    __syncthreads();
    for (int i = threadIdx.x; i < nf * tb.E; i += blockDim.x) {
        const int f = i / tb.E, band = i - f * tb.E;
        const int o = tb.erb_off[band], n = tb.erb_off[band + 1] - o;
        const float kinv = tb.erb_kinv[band];
        float acc = 0.f;
        for (int j = 0; j < n; j++) acc = __fadd_rn(acc, __fmul_rn(P[f * F + o + j], kinv));
        erb_db[((int64_t)b * Tf + t0 + f) * tb.E + band] = __fmul_rn(log10f(__fadd_rn(acc, 1e-10f)), 10.f);
    }
}

// grid (ceil(Tf / chunk), B), kGenThreads threads: frame_synthesis (lib.rs:396-427) of frames [c0, c0 + chunk) of stream b.
// Output sample p of frame t is the sum of the windowed inverse transforms of every frame that covers it, oldest first
// (the reference's order: the carried partial sum, then the new frame).  The CTA starts K = ceil((N - H) / H) frames
// before c0 so that its overlap-add tail is complete when c0 begins (their own outputs are not written), and
// transforms G frames at a time: the tail (N - H partial sums) plus G frames give G H output samples and the next tail.
// Stream b starts from init_tail [N - H] when given (the carried synthesis memory) and the tail after its last frame goes
// to final_tail when given (last stream only).
__global__ void __launch_bounds__(kGenThreads) k_synthesis_gen(const float2 *__restrict__ spec, int Tf, float *__restrict__ audio,
                                                               DspTables tb, GenFftPlan pl, int G, int chunk,
                                                               const float *__restrict__ init_tail, float *__restrict__ final_tail) {
    extern __shared__ __align__(16) float2 gsm[];
    __shared__ int s_rad[kGenMaxStages];
    const int N = pl.N, M = pl.M, H = tb.hop, F = tb.F, mem = N - H;
    const int b = blockIdx.y, c0 = blockIdx.x * chunk, c1 = min(c0 + chunk, Tf);
    float2 *A = gsm, *Bf = gsm + G * M;
    float *tails = reinterpret_cast<float *>(gsm + 2 * G * M);   // [2][N - H]: current and next tail
    int cur = 0;
    gen_load_radices(pl, s_rad);
    int tg = max(0, c0 - (mem + H - 1) / H);
    for (int i = threadIdx.x; i < mem; i += blockDim.x) tails[i] = (tg == 0 && init_tail) ? init_tail[i] : 0.f;
    const float2 *srow = spec + (int64_t)b * Tf * F;
    float *orow = audio + (int64_t)b * Tf * H;
    while (tg < c1) {
        const int gn = min(G, c1 - tg);
        // Hermitian half spectrum -> input of the M-point inverse transform (imaginary parts of DC and, for even N,
        // Nyquist are ignored: lib.rs:402, realfft)
        if (N % 2 == 0) {
            const int nk = M / 2 + 1;
            for (int i = threadIdx.x; i < gn * nk; i += blockDim.x) {
                const int f = i / nk, k = i - f * nk;
                const float2 *row = srow + (int64_t)(tg + f) * F;
                float2 xk = row[k], xnk = row[M - k];
                if (k == 0) { xk.y = 0.f; xnk.y = 0.f; }
                const float2 w = __ldg(pl.tw + k);
                float2 zk, znk;
                irfft_merge(xk, xnk, make_float2(w.x, -w.y), zk, znk);
                A[f * M + k] = zk;
                if (k > 0 && k < M - k) A[f * M + M - k] = znk;
            }
        } else {
            for (int i = threadIdx.x; i < gn * N; i += blockDim.x) {
                const int f = i / N, n = i - f * N;
                const float2 *row = srow + (int64_t)(tg + f) * F;
                float2 v = n < F ? row[n] : cconj(row[N - n]);
                if (n == 0) v.y = 0.f;
                A[f * M + n] = v;
            }
        }
        __syncthreads();
        const float2 *Y = gen_block_fft<true>(A, Bf, pl, s_rad, gn);
        // overlap-add: positions p in [0, gn H + N - H) relative to sample tg H
        for (int p = threadIdx.x; p < gn * H + mem; p += blockDim.x) {
            float v = p < mem ? tails[cur * mem + p] : 0.f;
            const int f_lo = p >= N ? (p - N) / H + 1 : 0, f_hi = min(gn - 1, p / H);
            for (int f = f_lo; f <= f_hi; f++) {
                const int q = p - f * H;
                const float y = (N % 2 == 0) ? reinterpret_cast<const float *>(Y + f * M)[q] : Y[f * M + q].x;
                v = __fadd_rn(v, __fmul_rn(y, __ldg(tb.window + q)));
            }
            if (p < gn * H) {
                if (tg + p / H >= c0) orow[(int64_t)tg * H + p] = v;
            } else {
                tails[(cur ^ 1) * mem + p - gn * H] = v;
            }
        }
        __syncthreads();
        cur ^= 1;
        tg += gn;
    }
    if (final_tail && c1 == Tf && b == (int)gridDim.y - 1)
        for (int i = threadIdx.x; i < mem; i += blockDim.x) final_tail[i] = tails[cur * mem + i];
}

}  // namespace dfb

// ====================================================================== host side / C ABI ==
using namespace dfb;

extern "C" const char *dfb_last_error(void) { return g_err.c_str(); }
extern "C" const char *dfb_version(void) { return "dfb200 0.2.0 sm_90a"; }
extern "C" int64_t dfb_kernel_launches(void) { return g_launches.load(); }

extern "C" int dfb_profile_enable(int on, const char *only_kernel) {
    g_prof_on = on != 0;
    g_prof_only = only_kernel ? only_kernel : "";
    return DFB_OK;
}

// Writes "name count total_ms\n" lines for everything recorded since the last report and clears.
extern "C" int64_t dfb_profile_report(char *buf, int64_t buflen) {
    if (!buf || buflen <= 0) return fail(DFB_ERR_INVALID, "bad buffer");
    cudaDeviceSynchronize();
    std::vector<std::string> names;
    std::vector<double> ms;
    std::vector<int64_t> cnt;
    // DFB_PROF_TIMELINE=1: start / end of every launch relative to the first one, to stderr (critical-path analysis)
    static const bool timeline = getenv("DFB_PROF_TIMELINE") && atoi(getenv("DFB_PROF_TIMELINE"));
    for (auto &r : g_prof) {
        float t = 0.f;
        if (cudaEventElapsedTime(&t, r.a, r.b) != cudaSuccess) t = 0.f;
        if (timeline) {
            float t0 = 0.f;
            cudaEventElapsedTime(&t0, g_prof.front().a, r.a);
            fprintf(stderr, "[timeline] %-34s %9.3f %9.3f\n", r.name.c_str(), t0, t0 + t);
        }
        size_t i = 0;
        for (; i < names.size(); i++) if (names[i] == r.name) break;
        if (i == names.size()) { names.push_back(r.name); ms.push_back(0); cnt.push_back(0); }
        ms[i] += t; cnt[i] += 1;
        g_prof_pool.push_back({r.a, r.b});
    }
    g_prof.clear();
    std::string out;
    char line[256];
    for (size_t i = 0; i < names.size(); i++) {
        snprintf(line, sizeof line, "%s %lld %.6f\n", names[i].c_str(), (long long)cnt[i], ms[i]);
        out += line;
    }
    if ((int64_t)out.size() + 1 > buflen) return fail(DFB_ERR_INVALID, "profile buffer too small");
    memcpy(buf, out.c_str(), out.size() + 1);
    return (int64_t)out.size();
}

// libDF/src/lib.rs:42-47,68-100 (f32 arithmetic, integer result)
extern "C" int dfb_erb_widths(int sr, int fft_size, int nb_erb, int min_nb_freqs, int64_t *out) {
    if (!out || nb_erb <= 0 || nb_erb > kMaxErb || fft_size <= 0) return fail(DFB_ERR_INVALID, "bad erb parameters");
    auto freq2erb = [](float f) { return 9.265f * log1pf(f / (24.7f * 9.265f)); };
    auto erb2freq = [](float e) { return 24.7f * 9.265f * (expf(e / 9.265f) - 1.f); };
    int nyq = sr / 2;
    float freq_width = (float)sr / (float)fft_size;
    float erb_low = freq2erb(0.f), erb_high = freq2erb((float)nyq);
    float step = (erb_high - erb_low) / (float)nb_erb;
    int prev_freq = 0, freq_over = 0;
    for (int i = 1; i <= nb_erb; i++) {
        float f = erb2freq(erb_low + (float)i * step);
        int fb = (int)roundf(f / freq_width);
        int nb = fb - prev_freq - freq_over;
        if (nb < min_nb_freqs) {
            freq_over = min_nb_freqs - nb;
            nb = min_nb_freqs;
        } else {
            freq_over = 0;
        }
        out[i - 1] = nb;
        prev_freq = fb;
    }
    out[nb_erb - 1] += 1;
    int64_t sum = 0;
    for (int i = 0; i < nb_erb; i++) sum += out[i];
    int64_t too_large = sum - (fft_size / 2 + 1);
    if (too_large > 0) out[nb_erb - 1] -= too_large;
    return DFB_OK;
}

extern "C" int dfb_state_create(dfb_state **out, int device, int sr, int fft_size, int hop_size, int nb_erb,
                                int min_nb_erb_freqs) {
    if (!out) return fail(DFB_ERR_INVALID, "null out");
    *out = nullptr;
    if (hop_size * 2 > fft_size) return fail(DFB_ERR_INVALID, "assertion failed: hop_size * 2 <= fft_size");
    if (hop_size < 1) return fail(DFB_ERR_INVALID, "hop_size must be positive (got %d)", hop_size);
    if (fft_size > kGenMaxN)
        return fail(DFB_ERR_UNSUPPORTED, "fft_size %d is above the largest built transform, %d", fft_size, kGenMaxN);
    GenFftPlan plan{};
    std::vector<float2> gtw;
    if (!gen_fft_plan(fft_size, plan, gtw)) return fail(DFB_ERR_INVALID, "fft_size %d outside [2, %d]", fft_size, kGenMaxN);
    if (nb_erb <= 0 || nb_erb > kMaxErb) return fail(DFB_ERR_INVALID, "nb_erb out of range");
    int rc = use_device(device);
    if (rc) return rc;
    dfb_state *st = new dfb_state();
    st->device = device; st->sr = sr; st->fft = fft_size; st->hop = hop_size; st->nb_erb = nb_erb;
    st->min_nb_erb_freqs = min_nb_erb_freqs;
    st->analysis_mem.assign(fft_size - hop_size, 0.f);
    st->synthesis_mem.assign(fft_size - hop_size, 0.f);
    st->erb.resize(nb_erb);
    dfb_erb_widths(sr, fft_size, nb_erb, min_nb_erb_freqs, st->erb.data());
    const int F = fft_size / 2 + 1;
    // vorbis window, f64 -> f32 (lib.rs:126-132)
    st->window.resize(fft_size);
    const double pi = 3.14159265358979323846;
    for (int i = 0; i < fft_size; i++) {
        double s = sin(0.5 * pi * ((double)i + 0.5) / (double)(fft_size / 2));
        st->window[i] = (float)sin(0.5 * pi * s * s);
    }
    // one slab: window | tw_a_fwd | tw_a_inv | tw960 | erb_off | erb_kinv | band_of_bin | generic FFT twiddles
    std::vector<float2> twf(kN2 * kN1), twi(kN2 * kN1), tw960(241);
    for (int l = 0; l < kN2; l++)
        for (int k1 = 0; k1 < kN1; k1++) {
            double a = 2.0 * pi * (double)((l * k1) % kC) / (double)kC;
            twf[l * kN1 + k1] = make_float2((float)cos(a), (float)-sin(a));
            twi[l * kN1 + k1] = make_float2((float)cos(a), (float)sin(a));
        }
    for (int k = 0; k <= 240; k++) {
        double a = 2.0 * pi * (double)k / (double)kFft;
        tw960[k] = make_float2((float)cos(a), (float)-sin(a));
    }
    std::vector<int> off(nb_erb + 1, 0);
    std::vector<float> kinv(nb_erb);
    std::vector<unsigned char> bob(F);
    for (int b = 0; b < nb_erb; b++) {
        off[b + 1] = off[b] + (int)st->erb[b];
        kinv[b] = 1.f / (float)st->erb[b];
        for (int k = off[b]; k < off[b + 1] && k < F; k++) bob[k] = (unsigned char)b;
    }
    if (off[nb_erb] != F) {
        delete st;
        return fail(DFB_ERR_INVALID, "erb widths sum to %d, expected %d", off[nb_erb], F);
    }
    // (the float2 tables start 256-byte aligned whatever fft_size is, odd included)
    size_t o_win = 0, o_twf = o_win + ((sizeof(float) * fft_size + 255) & ~size_t(255)), o_twi = o_twf + sizeof(float2) * twf.size(),
           o_960 = o_twi + sizeof(float2) * twi.size(), o_off = o_960 + sizeof(float2) * 256,
           o_kinv = o_off + sizeof(int) * (kMaxErb + 1 + 3), o_bob = o_kinv + sizeof(float) * kMaxErb,
           o_gtw = o_bob + ((F + 255) & ~255), total = o_gtw + sizeof(float2) * gtw.size();
    std::vector<char> slab(total, 0);
    memcpy(slab.data() + o_gtw, gtw.data(), sizeof(float2) * gtw.size());
    memcpy(slab.data() + o_win, st->window.data(), sizeof(float) * fft_size);
    memcpy(slab.data() + o_twf, twf.data(), sizeof(float2) * twf.size());
    memcpy(slab.data() + o_twi, twi.data(), sizeof(float2) * twi.size());
    memcpy(slab.data() + o_960, tw960.data(), sizeof(float2) * tw960.size());
    memcpy(slab.data() + o_off, off.data(), sizeof(int) * off.size());
    memcpy(slab.data() + o_kinv, kinv.data(), sizeof(float) * kinv.size());
    memcpy(slab.data() + o_bob, bob.data(), bob.size());
    char *d = nullptr;
    if (cudaMalloc(&d, total) != cudaSuccess || cudaMemcpy(d, slab.data(), total, cudaMemcpyHostToDevice) != cudaSuccess) {
        delete st;
        return fail(DFB_ERR_CUDA, "table upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    st->d_tables = d;
    st->tb.window = (const float *)(d + o_win);
    st->tb.tw_a_fwd = (const float2 *)(d + o_twf);
    st->tb.tw_a_inv = (const float2 *)(d + o_twi);
    st->tb.tw960 = (const float2 *)(d + o_960);
    st->tb.erb_off = (const int *)(d + o_off);
    st->tb.erb_kinv = (const float *)(d + o_kinv);
    st->tb.band_of_bin = (const unsigned char *)(d + o_bob);
    st->tb.wnorm = 1.f / ((float)((int64_t)fft_size * fft_size) / (float)(2 * hop_size));  // lib.rs:133
    st->tb.fft = fft_size; st->tb.hop = hop_size; st->tb.F = F; st->tb.E = nb_erb;
    st->plan = plan;
    st->plan.tw = (const float2 *)(d + o_gtw);
    cudaFuncSetAttribute(k_analysis<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAnaSmem);
    cudaFuncSetAttribute(k_analysis<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAnaSmem);
    cudaFuncSetAttribute(k_analysis_gen, cudaFuncAttributeMaxDynamicSharedMemorySize, kGenSmemMax);
    cudaFuncSetAttribute(k_synthesis_gen, cudaFuncAttributeMaxDynamicSharedMemorySize, kGenSmemMax);
    if (cudaStreamCreateWithFlags(&st->stream, cudaStreamNonBlocking) != cudaSuccess) {
        cudaFree(d);
        delete st;
        return fail(DFB_ERR_CUDA, "stream creation failed");
    }
    *out = st;
    return DFB_OK;
}

extern "C" void dfb_state_free(dfb_state *st) {
    if (!st) return;
    cudaSetDevice(st->device);
    st->arena.release();
    if (st->d_tables) cudaFree(st->d_tables);
    if (st->stream) cudaStreamDestroy(st->stream);
    delete st;
}

extern "C" int dfb_state_erb_widths(const dfb_state *st, int64_t *w) {
    if (!st || !w) return fail(DFB_ERR_INVALID, "null argument");
    memcpy(w, st->erb.data(), sizeof(int64_t) * st->nb_erb);
    return DFB_OK;
}
extern "C" int dfb_state_fft_window(const dfb_state *st, float *w) {
    if (!st || !w) return fail(DFB_ERR_INVALID, "null argument");
    memcpy(w, st->window.data(), sizeof(float) * st->fft);
    return DFB_OK;
}
extern "C" int dfb_state_params(const dfb_state *st, int *sr, int *fft, int *hop, int *nb_erb) {
    if (!st) return fail(DFB_ERR_INVALID, "null state");
    if (sr) *sr = st->sr;
    if (fft) *fft = st->fft;
    if (hop) *hop = st->hop;
    if (nb_erb) *nb_erb = st->nb_erb;
    return DFB_OK;
}

namespace dfb {

// fft 960 / hop 480: the specialised warp kernels; every other size runs the generic ones (outside the enhancement
// path, so not among the kernels DFB_PROF reports)
static bool is_960(const dfb_state *st) { return st->fft == kFft && st->hop == kHop; }

int launch_analysis(dfb_state *st, const float *d_audio, int64_t C, int64_t T, float *d_spec, float *d_erb_db,
                    cudaStream_t s, const float *d_init_mem, const AnaWindow *w) {
    int64_t Tf = T / st->hop;
    if (C <= 0 || Tf <= 0) return DFB_OK;
    if (C > 65535) return fail(DFB_ERR_INVALID, "more than 65535 channels per call");
    if (!is_960(st)) {
        if (w) return fail(DFB_ERR_UNSUPPORTED, "time-chunked analysis is built for fft_size 960 / hop_size 480 only");
        if (Tf > INT_MAX) return fail(DFB_ERR_INVALID, "more than 2^31 frames per channel");
        const int G = gen_frames(st->plan.M);
        dim3 grid((unsigned)((Tf + G - 1) / G), (unsigned)C);
        k_analysis_gen<<<grid, kGenThreads, sizeof(float2) * 2 * G * st->plan.M, s>>>(d_audio, T, (int)Tf, (float2 *)d_spec,
                                                                                     d_erb_db, st->tb, st->plan, G, d_init_mem);
        DFB_LAUNCH_CHECK();
        return DFB_OK;
    }
    const int t_begin = w ? w->t_begin : 0, nf = w ? w->nf : (int)Tf, out_t0 = w ? w->out_t0 : 0, Tbuf = w ? w->Tbuf : (int)Tf;
    if (nf <= 0) return DFB_OK;
    dim3 grid((unsigned)((nf + kAnaWarps - 1) / kAnaWarps), (unsigned)C);
    DFB_PROF("k_analysis", s);
    if (w)
        k_analysis<true><<<grid, 32 * kAnaWarps, kAnaSmem, s>>>(d_audio, T, (int)Tf, (float2 *)d_spec, d_erb_db, st->tb, d_init_mem,
                                                              t_begin, nf, out_t0, Tbuf, w->rows);
    else
        k_analysis<false><<<grid, 32 * kAnaWarps, kAnaSmem, s>>>(d_audio, T, (int)Tf, (float2 *)d_spec, d_erb_db, st->tb, d_init_mem,
                                                               t_begin, nf, out_t0, Tbuf, nullptr);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

int launch_feat_norm(const float *d_erb, int E, int64_t erb_stride, const float *d_spec, int Fd, int64_t spec_stride,
                     int64_t C, int64_t Tf, float alpha, const float *d_erb_state, const float *d_unit_state,
                     float *d_feat_erb, float *d_feat_spec, cudaStream_t s, int64_t Ts, float *d_erb_state_out,
                     float *d_unit_state_out, bool ref_bits) {
    if (C <= 0 || Tf <= 0 || E + Fd == 0) return DFB_OK;
    int threads = ((E + Fd + 31) / 32) * 32;
    DFB_PROF("k_feat_norm", s);
    if (E + Fd > 1024) {
        dim3 grid((unsigned)C, (unsigned)((E + Fd + 255) / 256));
        const int ts = (int)(Ts > 0 ? Ts : Tf);
        if (ref_bits)
            k_feat_norm<4, true, true><<<grid, 256, 0, s>>>(d_erb, E, erb_stride, (const float2 *)d_spec, Fd, spec_stride, (int)Tf, alpha,
                                                            d_erb_state, d_unit_state, d_feat_erb, (float2 *)d_feat_spec, ts,
                                                            d_erb_state_out, d_unit_state_out);
        else
            k_feat_norm<4, false, true><<<grid, 256, 0, s>>>(d_erb, E, erb_stride, (const float2 *)d_spec, Fd, spec_stride, (int)Tf, alpha,
                                                             d_erb_state, d_unit_state, d_feat_erb, (float2 *)d_feat_spec, ts,
                                                             d_erb_state_out, d_unit_state_out);
        DFB_LAUNCH_CHECK();
        return DFB_OK;
    }
    static const bool no_seg = getenv("DFB_NORM_SEG") && !atoi(getenv("DFB_NORM_SEG"));
    if (ref_bits && threads <= 128)
        k_feat_norm<24, true><<<(unsigned)C, threads, 0, s>>>(d_erb, E, erb_stride, (const float2 *)d_spec, Fd, spec_stride, (int)Tf,
                                                             alpha, d_erb_state, d_unit_state, d_feat_erb, (float2 *)d_feat_spec,
                                                             (int)(Ts > 0 ? Ts : Tf), d_erb_state_out, d_unit_state_out);
    else if (ref_bits)
        k_feat_norm<4, true><<<(unsigned)C, threads, 0, s>>>(d_erb, E, erb_stride, (const float2 *)d_spec, Fd, spec_stride, (int)Tf,
                                                            alpha, d_erb_state, d_unit_state, d_feat_erb, (float2 *)d_feat_spec,
                                                            (int)(Ts > 0 ? Ts : Tf), d_erb_state_out, d_unit_state_out);
    else if (threads <= 128 && Tf >= 16 * kNormSeg && !no_seg)
        k_feat_norm_seg<<<(unsigned)C, 128 * kNormSeg, 0, s>>>(d_erb, E, erb_stride, (const float2 *)d_spec, Fd, spec_stride, (int)Tf,
                                                            alpha, d_erb_state, d_unit_state, d_feat_erb, (float2 *)d_feat_spec,
                                                            (int)(Ts > 0 ? Ts : Tf), d_erb_state_out, d_unit_state_out);
    else if (threads <= 128)
        k_feat_norm<24><<<(unsigned)C, threads, 0, s>>>(d_erb, E, erb_stride, (const float2 *)d_spec, Fd, spec_stride, (int)Tf,
                                                       alpha, d_erb_state, d_unit_state, d_feat_erb, (float2 *)d_feat_spec,
                                                       (int)(Ts > 0 ? Ts : Tf), d_erb_state_out, d_unit_state_out);
    else
        k_feat_norm<4><<<(unsigned)C, threads, 0, s>>>(d_erb, E, erb_stride, (const float2 *)d_spec, Fd, spec_stride, (int)Tf,
                                                      alpha, d_erb_state, d_unit_state, d_feat_erb, (float2 *)d_feat_spec,
                                                      (int)(Ts > 0 ? Ts : Tf), d_erb_state_out, d_unit_state_out);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

// Plain ISTFT (mode 0) of a state other than 960 / 480.  With p.carry and several channels, channel c continues from the
// tail channel c - 1 leaves, which may still hold samples of the channels before it (a channel shorter than N - H):
// one launch per channel, the tails chained on the device through two ping-pong buffers after final_tail.
static int launch_synthesis_gen(dfb_state *st, const ApplyParams &p, int64_t B, cudaStream_t s) {
    if (p.mode != 0 || p.spec_out || p.rows || p.out_offset || p.t_first || p.spec_T || p.Tv || p.out_stride != (int64_t)p.Tf * st->hop)
        return fail(DFB_ERR_UNSUPPORTED, "the enhancement path is built for fft_size 960 / hop_size 480 only");
    const int M = st->plan.M, G = gen_frames(M), mem = st->fft - st->hop, K = (mem + st->hop - 1) / st->hop;
    const int chunk = G * std::max(2, (8 * K + G - 1) / G);
    const size_t smem = sizeof(float2) * 2 * G * M + sizeof(float) * 2 * mem;
    const int64_t F = st->tb.F, Tf = p.Tf;
    if (!p.carry || B == 1) {
        dim3 grid((unsigned)((Tf + chunk - 1) / chunk), (unsigned)B);
        k_synthesis_gen<<<grid, kGenThreads, smem, s>>>(p.spec, p.Tf, p.audio, st->tb, st->plan, G, chunk,
                                                        p.carry ? p.init_tail : nullptr, p.final_tail);
        DFB_LAUNCH_CHECK();
        return DFB_OK;
    }
    if (!p.final_tail) return fail(DFB_ERR_INVALID, "carried synthesis needs a final tail buffer of 3 (N - H) floats");
    dim3 grid((unsigned)((Tf + chunk - 1) / chunk), 1);
    const float *in = p.init_tail;
    for (int64_t c = 0; c < B; c++) {
        float *out = c == B - 1 ? p.final_tail : p.final_tail + mem * (1 + (c & 1));
        k_synthesis_gen<<<grid, kGenThreads, smem, s>>>(p.spec + c * Tf * F, p.Tf, p.audio + c * Tf * st->hop, st->tb, st->plan,
                                                        G, chunk, in, out);
        DFB_LAUNCH_CHECK();
        in = out;
    }
    return DFB_OK;
}

int launch_apply_synthesis(dfb_state *st, const ApplyParams &p, int64_t B, cudaStream_t s, const SlotCtl *ctl) {
    if (B <= 0 || p.Tf <= 0) return DFB_OK;
    if (B > 65535) return fail(DFB_ERR_INVALID, "more than 65535 channels per call");
    if (!is_960(st)) {
        if (ctl) return fail(DFB_ERR_UNSUPPORTED, "the enhancement path is built for fft_size 960 / hop_size 480 only");
        return launch_synthesis_gen(st, p, B, s);
    }
    if (p.mode != 0 && (p.nb_df > 240 || p.order > 8)) return fail(DFB_ERR_UNSUPPORTED, "nb_df > 240 or df_order > 8");
    // frames per warp: 16 amortises the re-synthesis of the frame before a warp's first one; short windows (time chunks)
    // take 8 so that the grid still fills the device with a few waves
    ApplyParams q = p;
    q.frames_per_warp = (B * (int64_t)p.Tf / kSynChunk >= 6000) ? kSynChunk : kSynChunk / 2;
    int per_cta = kSynWarps * q.frames_per_warp;
    dim3 grid((unsigned)((p.Tf + per_cta - 1) / per_cta), (unsigned)B);
    if (p.lsnr && !(p.mode == 1 && p.order == 5 && p.nb_df == 96 && st->tb.E == 32 && p.m && p.coefs))
        return fail(DFB_ERR_UNSUPPORTED, "LSNR stage gating is built for the DeepFilterNet3 apply kernel only");
    const bool special = p.mode != 0 && p.order == 5 && p.nb_df == 96 && st->tb.E == 32 && p.m && p.coefs;
    if (p.links && !(special && p.rows))
        return fail(DFB_ERR_UNSUPPORTED, "linked channels are built for the specialised row-table apply kernel only");
    if (p.links && p.reduce != kReduceMax && p.reduce != kReduceMean) return fail(DFB_ERR_INVALID, "bad mask reduction %d", p.reduce);
    if (ctl && !(special && p.rows))
        return fail(DFB_ERR_UNSUPPORTED, "per-stream settings are built for the specialised slot apply kernel only");
    DFB_PROF("k_apply_synthesis", s);
    // MINB 2: 2 CTAs/SM without spills measured fastest
    if (ctl && p.links)   // slot groups of linked channels (dfb_stream_open_linked) with per-group settings
        k_apply_synthesis<5, 3, 2, true, true, true><<<grid, 32 * kSynWarps, 0, s>>>(q, st->tb, ctl);
    else if (ctl)
        k_apply_synthesis<5, 3, 2, true, false, true><<<grid, 32 * kSynWarps, 0, s>>>(q, st->tb, ctl);
    else if (p.links)
        k_apply_synthesis<5, 3, 2, true, true><<<grid, 32 * kSynWarps, 0, s>>>(q, st->tb, nullptr);
    else if (special && p.rows)
        k_apply_synthesis<5, 3, 2, true><<<grid, 32 * kSynWarps, 0, s>>>(q, st->tb, nullptr);
    else if (special)
        k_apply_synthesis<5, 3, 2, false><<<grid, 32 * kSynWarps, 0, s>>>(q, st->tb, nullptr);
    else
        k_apply_synthesis_generic<<<grid, 32 * kSynWarps, 0, s>>>(q, st->tb);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

int launch_resample_stream(cudaStream_t s, bool up, const ResampleDirs &dirs, int n_dirs, const ResampleRow *rows, int nb,
                           const ResampleIO &io) {
    if (nb <= 0 || io.n <= 0) return DFB_OK;
    if (nb > 65535 || n_dirs <= 0 || n_dirs > kMaxRateDirs) return fail(DFB_ERR_INVALID, "bad resampler geometry");
    for (int i = 0; i < n_dirs; i++) {
        const ResampleDir &d = dirs.d[i];
        if (d.S > d.hop_in || d.S > io.hist_pitch)
            return fail(DFB_ERR_INVALID, "bad resampler geometry");
    }
    // (not in the DFB_PROF timing, which covers the 48 kHz enhancement path; torch.profiler names them)
    if (up)
        k_resample_up<<<nb, 256, 0, s>>>(dirs, rows, io);
    else
        k_resample_down<<<nb, 256, 0, s>>>(dirs, rows, io);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

int launch_resample_rows(cudaStream_t s, bool up, const RateDir *d_dirs, const RateRow *d_rows, int nb, const RateIO &io,
                         int64_t max_out, int smem_floats) {
    if (nb <= 0 || max_out <= 0) return DFB_OK;
    if (nb > 65535 || smem_floats < 0 || smem_floats > kRateSmemFloats) return fail(DFB_ERR_INVALID, "bad resampler geometry");
    const int64_t tiles = (max_out + kRateTile - 1) / kRateTile;
    // (not in the DFB_PROF timing, which covers the 48 kHz enhancement path; torch.profiler names it)
    k_resample_rows<<<dim3((unsigned)tiles, (unsigned)nb), 256, sizeof(float) * (size_t)smem_floats, s>>>(d_dirs, d_rows, io, up,
                                                                                                          smem_floats);
    DFB_LAUNCH_CHECK();
    return DFB_OK;
}

}  // namespace dfb

extern "C" int dfb_analysis(dfb_state *st, const float *d_audio, int64_t C, int64_t T, float *d_spec, void *stream) {
    if (!st || !d_audio || !d_spec) return fail(DFB_ERR_INVALID, "null argument");
    DFB_CUDA(cudaSetDevice(st->device));
    return launch_analysis(st, d_audio, C, T, d_spec, nullptr, (cudaStream_t)stream);
}

extern "C" int dfb_state_reset(dfb_state *st);

// pyDF DF.analysis(input, reset): reset != 0 starts every channel from zero memory (pyDF/src/lib.rs:56-58);
// reset == 0 carries the STFT memory from the previous call into channel 0 and from channel c into c + 1
// (one DFState is shared by all channels).  The memory holds the last N - H samples a channel's frames read: the memory
// entering channel c is the tail of (memory entering c - 1, then c - 1's first Tf hop samples), so a channel shorter than
// N - H keeps part of the older memory.  Either way the memory left behind is the one after the last channel.
extern "C" int dfb_analysis_host_ex(dfb_state *st, const float *h_audio, int64_t C, int64_t T, int reset, float *h_spec) {
    if (!st || !h_audio || !h_spec) return fail(DFB_ERR_INVALID, "null argument");
    if (C <= 0 || T <= 0) return fail(DFB_ERR_INVALID, "[df] Input array empty or not contiguous.");
    DFB_CUDA(cudaSetDevice(st->device));
    const int64_t Tf = T / st->hop, hop = st->hop, nm = st->fft - st->hop;
    if (reset) dfb_state_reset(st);  // DFState::reset clears BOTH memories (libDF/src/lib.rs:156-159)
    size_t nb_in = sizeof(float) * C * T, nb_out = sizeof(float) * 2 * C * Tf * st->tb.F;
    int rc = st->arena.reserve(nb_in + nb_out + sizeof(float) * C * nm + 2048);
    if (rc) return rc;
    st->arena.reset();
    float *d_in = st->arena.take<float>(C * T), *d_out = st->arena.take<float>(2 * C * Tf * st->tb.F + 2);
    float *d_mem = nullptr;
    DFB_CUDA(cudaMemcpyAsync(d_in, h_audio, nb_in, cudaMemcpyHostToDevice, st->stream));
    // the memory after a channel that entered with `m`: the last nm samples of m followed by its first Tf hop samples
    auto advance = [&](std::vector<float> &m, const float *xc) {
        const int64_t n = Tf * hop;
        if (n >= nm) {
            memcpy(m.data(), xc + n - nm, sizeof(float) * nm);
        } else {
            memmove(m.data(), m.data() + n, sizeof(float) * (nm - n));
            memcpy(m.data() + nm - n, xc, sizeof(float) * n);
        }
    };
    std::vector<float> mem, cur(st->analysis_mem);
    if (!reset && Tf > 0) {
        mem.resize((size_t)C * nm);
        for (int64_t c = 0; c < C; c++) {
            memcpy(mem.data() + c * nm, cur.data(), sizeof(float) * nm);
            if (c + 1 < C) advance(cur, h_audio + c * T);
        }
        d_mem = st->arena.take<float>(C * nm);
        DFB_CUDA(cudaMemcpyAsync(d_mem, mem.data(), sizeof(float) * C * nm, cudaMemcpyHostToDevice, st->stream));
    }
    rc = launch_analysis(st, d_in, C, T, d_out, nullptr, st->stream, d_mem);
    if (rc) return rc;
    if (nb_out) DFB_CUDA(cudaMemcpyAsync(h_spec, d_out, nb_out, cudaMemcpyDeviceToHost, st->stream));
    DFB_CUDA(cudaStreamSynchronize(st->stream));
    if (Tf > 0) {
        advance(cur, h_audio + (C - 1) * T);
        st->analysis_mem = cur;
    }
    return DFB_OK;
}
extern "C" int dfb_analysis_host(dfb_state *st, const float *h_audio, int64_t C, int64_t T, float *h_spec) {
    return dfb_analysis_host_ex(st, h_audio, C, T, 1, h_spec);
}
extern "C" int dfb_state_reset(dfb_state *st) {
    if (!st) return fail(DFB_ERR_INVALID, "null state");
    std::fill(st->analysis_mem.begin(), st->analysis_mem.end(), 0.f);
    std::fill(st->synthesis_mem.begin(), st->synthesis_mem.end(), 0.f);
    return DFB_OK;
}

extern "C" int dfb_synthesis(dfb_state *st, const float *d_spec, int64_t C, int64_t Tf, float *d_audio, void *stream) {
    if (!st || !d_spec || !d_audio) return fail(DFB_ERR_INVALID, "null argument");
    DFB_CUDA(cudaSetDevice(st->device));
    ApplyParams p{};
    p.spec = (const float2 *)d_spec; p.audio = d_audio; p.out_stride = Tf * st->hop; p.out_offset = 0;
    p.out_len = Tf * st->hop; p.Tf = (int)Tf; p.mode = 0;
    return launch_apply_synthesis(st, p, C, (cudaStream_t)stream);
}

// pyDF DF.synthesis(input, reset): see dfb_analysis_host_ex for the reset semantics (pyDF/src/lib.rs:91-93).
extern "C" int dfb_synthesis_host_ex(dfb_state *st, const float *h_spec, int64_t C, int64_t Tf, int reset, float *h_audio) {
    if (!st || !h_spec || !h_audio) return fail(DFB_ERR_INVALID, "null argument");
    if (C <= 0 || Tf <= 0) return fail(DFB_ERR_INVALID, "[df] Input array empty or not contiguous.");
    DFB_CUDA(cudaSetDevice(st->device));
    const int64_t hop = st->hop, nm = st->fft - st->hop;   // the tail: N - H partial overlap-add sums
    if (reset) dfb_state_reset(st);  // clears the analysis memory as well (libDF/src/lib.rs:156-159)
    size_t nb_in = sizeof(float) * 2 * C * Tf * st->tb.F, nb_out = sizeof(float) * C * Tf * hop;
    int rc = st->arena.reserve(nb_in + nb_out + sizeof(float) * 4 * nm + 2048);
    if (rc) return rc;
    st->arena.reset();
    float *d_in = st->arena.take<float>(2 * C * Tf * st->tb.F), *d_out = st->arena.take<float>(C * Tf * hop);
    // final tail + two ping-pong tails of the channel chain of the generic kernel
    float *d_init = st->arena.take<float>(nm), *d_final = st->arena.take<float>(3 * nm);
    DFB_CUDA(cudaMemcpyAsync(d_in, h_spec, nb_in, cudaMemcpyHostToDevice, st->stream));
    DFB_CUDA(cudaMemcpyAsync(d_init, st->synthesis_mem.data(), sizeof(float) * nm, cudaMemcpyHostToDevice, st->stream));
    ApplyParams p{};
    p.spec = (const float2 *)d_in; p.audio = d_out; p.out_stride = Tf * hop; p.out_offset = 0;
    p.out_len = Tf * hop; p.Tf = (int)Tf; p.mode = 0;
    p.carry = reset ? 0 : 1; p.init_tail = d_init; p.final_tail = d_final;
    rc = launch_apply_synthesis(st, p, C, st->stream);
    if (rc) return rc;
    DFB_CUDA(cudaMemcpyAsync(h_audio, d_out, nb_out, cudaMemcpyDeviceToHost, st->stream));
    DFB_CUDA(cudaMemcpyAsync(st->synthesis_mem.data(), d_final, sizeof(float) * nm, cudaMemcpyDeviceToHost, st->stream));
    DFB_CUDA(cudaStreamSynchronize(st->stream));
    return DFB_OK;
}
extern "C" int dfb_synthesis_host(dfb_state *st, const float *h_spec, int64_t C, int64_t Tf, float *h_audio) {
    return dfb_synthesis_host_ex(st, h_spec, C, Tf, 1, h_audio);
}

namespace {
// tiny RAII scratch for the stateless *_host helpers
struct Scratch {
    std::vector<void *> ptrs;
    ~Scratch() { for (void *p : ptrs) cudaFree(p); }
    template <typename T>
    T *alloc(size_t n) {
        void *p = nullptr;
        if (cudaMalloc(&p, (n ? n : 1) * sizeof(T)) != cudaSuccess) return nullptr;
        ptrs.push_back(p);
        return (T *)p;
    }
};
}  // namespace

extern "C" int dfb_erb_host(int device, const float *h_spec, int64_t n_frames, int64_t F, const int64_t *widths, int E,
                            int db, float *h_out) {
    if (!h_spec || !widths || !h_out || n_frames <= 0 || F <= 0 || E <= 0) return fail(DFB_ERR_INVALID, "bad argument");
    std::vector<int> off(E + 1, 0);
    for (int b = 0; b < E; b++) off[b + 1] = off[b] + (int)widths[b];
    if (off[E] != F) return fail(DFB_ERR_INVALID, "DF shape error: erb widths sum to %d but input has %lld bins", off[E], (long long)F);
    int rc = use_device(device);
    if (rc) return rc;
    Scratch s;
    float2 *d_in = s.alloc<float2>(n_frames * F);
    float *d_out = s.alloc<float>(n_frames * E);
    int *d_off = s.alloc<int>(E + 1);
    if (!d_in || !d_out || !d_off) return fail(DFB_ERR_OOM, "cudaMalloc failed");
    DFB_CUDA(cudaMemcpy(d_in, h_spec, sizeof(float2) * n_frames * F, cudaMemcpyHostToDevice));
    DFB_CUDA(cudaMemcpy(d_off, off.data(), sizeof(int) * (E + 1), cudaMemcpyHostToDevice));
    k_erb<<<(unsigned)((n_frames + 7) / 8), 256>>>(d_in, n_frames, (int)F, d_off, E, db, d_out);
    DFB_LAUNCH_CHECK();
    DFB_CUDA(cudaMemcpy(h_out, d_out, sizeof(float) * n_frames * E, cudaMemcpyDeviceToHost));
    return DFB_OK;
}

extern "C" int dfb_erb_inv_host(int device, const float *h_gains, int64_t n_frames, const int64_t *widths, int E,
                                float *h_out) {
    if (!h_gains || !widths || !h_out || n_frames <= 0 || E <= 0 || E > 255) return fail(DFB_ERR_INVALID, "bad argument");
    int64_t F = 0;
    for (int b = 0; b < E; b++) F += widths[b];
    std::vector<unsigned char> bob(F);
    int64_t o = 0;
    for (int b = 0; b < E; b++) { for (int64_t j = 0; j < widths[b]; j++) bob[o + j] = (unsigned char)b; o += widths[b]; }
    int rc = use_device(device);
    if (rc) return rc;
    Scratch s;
    float *d_in = s.alloc<float>(n_frames * E), *d_out = s.alloc<float>(n_frames * F);
    unsigned char *d_bob = s.alloc<unsigned char>(F);
    if (!d_in || !d_out || !d_bob) return fail(DFB_ERR_OOM, "cudaMalloc failed");
    DFB_CUDA(cudaMemcpy(d_in, h_gains, sizeof(float) * n_frames * E, cudaMemcpyHostToDevice));
    DFB_CUDA(cudaMemcpy(d_bob, bob.data(), F, cudaMemcpyHostToDevice));
    int64_t n = n_frames * F;
    k_erb_inv<<<(unsigned)((n + 255) / 256), 256>>>(d_in, n_frames, (int)F, E, d_bob, d_out);
    DFB_LAUNCH_CHECK();
    DFB_CUDA(cudaMemcpy(h_out, d_out, sizeof(float) * n, cudaMemcpyDeviceToHost));
    return DFB_OK;
}

extern "C" int dfb_erb_norm_host(int device, const float *h_erb, int64_t C, int64_t T, int64_t E, float alpha,
                                 const float *h_state, float *h_out) {
    if (!h_erb || !h_out || C <= 0 || T <= 0 || E <= 0) return fail(DFB_ERR_INVALID, "bad argument");
    int rc = use_device(device);
    if (rc) return rc;
    Scratch s;
    float *d_in = s.alloc<float>(C * T * E), *d_out = s.alloc<float>(C * T * E), *d_st = nullptr;
    if (!d_in || !d_out) return fail(DFB_ERR_OOM, "cudaMalloc failed");
    DFB_CUDA(cudaMemcpy(d_in, h_erb, sizeof(float) * C * T * E, cudaMemcpyHostToDevice));
    if (h_state) {
        d_st = s.alloc<float>(C * E);
        DFB_CUDA(cudaMemcpy(d_st, h_state, sizeof(float) * C * E, cudaMemcpyHostToDevice));
    }
    // pyDF's bits at every length (ref_bits)
    rc = launch_feat_norm(d_in, (int)E, E, nullptr, 0, 0, C, T, alpha, d_st, nullptr, d_out, nullptr, 0, 0, nullptr, nullptr, true);
    if (rc) return rc;
    DFB_CUDA(cudaMemcpy(h_out, d_out, sizeof(float) * C * T * E, cudaMemcpyDeviceToHost));
    return DFB_OK;
}

extern "C" int dfb_unit_norm_host(int device, const float *h_spec, int64_t C, int64_t T, int64_t F, float alpha,
                                  const float *h_state, float *h_out) {
    if (!h_spec || !h_out || C <= 0 || T <= 0 || F <= 0) return fail(DFB_ERR_INVALID, "bad argument");
    int rc = use_device(device);
    if (rc) return rc;
    Scratch s;
    float *d_in = s.alloc<float>(2 * C * T * F), *d_out = s.alloc<float>(2 * C * T * F), *d_st = nullptr;
    if (!d_in || !d_out) return fail(DFB_ERR_OOM, "cudaMalloc failed");
    DFB_CUDA(cudaMemcpy(d_in, h_spec, sizeof(float) * 2 * C * T * F, cudaMemcpyHostToDevice));
    if (h_state) {
        d_st = s.alloc<float>(C * F);
        DFB_CUDA(cudaMemcpy(d_st, h_state, sizeof(float) * C * F, cudaMemcpyHostToDevice));
    }
    rc = launch_feat_norm(nullptr, 0, 0, d_in, (int)F, F, C, T, alpha, nullptr, d_st, nullptr, d_out, 0, 0, nullptr, nullptr, true);
    if (rc) return rc;
    DFB_CUDA(cudaMemcpy(h_out, d_out, sizeof(float) * 2 * C * T * F, cudaMemcpyDeviceToHost));
    return DFB_OK;
}

extern "C" int dfb_unit_norm_init(int64_t n, float *h_out) {
    if (!h_out || n <= 0) return fail(DFB_ERR_INVALID, "bad argument");
    if (n == 1) { h_out[0] = 0.001f; return DFB_OK; }
    float step = (0.0001f - 0.001f) / (float)(n - 1);
    for (int64_t i = 0; i < n; i++) h_out[i] = 0.001f + (float)i * step;
    return DFB_OK;
}

extern "C" int dfb_features(dfb_state *st, const float *d_audio, int64_t C, int64_t T, int nb_df, float alpha,
                            float *d_spec, float *d_feat_erb, float *d_feat_spec, void *stream) {
    if (!st || !d_audio || !d_spec || !d_feat_erb || !d_feat_spec) return fail(DFB_ERR_INVALID, "null argument");
    if (nb_df <= 0 || nb_df > st->tb.F) return fail(DFB_ERR_INVALID, "nb_df out of range");
    DFB_CUDA(cudaSetDevice(st->device));
    cudaStream_t s = (cudaStream_t)stream;
    int64_t Tf = T / st->hop;
    // raw ERB dB goes to feat_erb and is normalised in place by the scan kernel
    int rc = launch_analysis(st, d_audio, C, T, d_spec, d_feat_erb, s);
    if (rc) return rc;
    return launch_feat_norm(d_feat_erb, st->tb.E, st->tb.E, d_spec, nb_df, st->tb.F, C, Tf, alpha, nullptr, nullptr,
                            d_feat_erb, d_feat_spec, s);
}

extern "C" int dfb_features_host(dfb_state *st, const float *h_audio, int64_t C, int64_t T, int nb_df, float alpha,
                                 float *h_spec, float *h_feat_erb, float *h_feat_spec) {
    if (!st || !h_audio || !h_spec || !h_feat_erb || !h_feat_spec) return fail(DFB_ERR_INVALID, "null argument");
    if (C <= 0 || T <= 0) return fail(DFB_ERR_INVALID, "[df] Input array empty or not contiguous.");
    DFB_CUDA(cudaSetDevice(st->device));
    int64_t Tf = T / st->hop, F = st->tb.F, E = st->tb.E;
    size_t n_spec = 2 * C * Tf * F, n_fe = C * Tf * E, n_fs = 2 * C * Tf * nb_df;
    int rc = st->arena.reserve(sizeof(float) * (C * T + n_spec + n_fe + n_fs) + 4096);
    if (rc) return rc;
    st->arena.reset();
    float *d_in = st->arena.take<float>(C * T), *d_spec = st->arena.take<float>(n_spec + 2),
          *d_fe = st->arena.take<float>(n_fe + 1), *d_fs = st->arena.take<float>(n_fs + 2);
    DFB_CUDA(cudaMemcpyAsync(d_in, h_audio, sizeof(float) * C * T, cudaMemcpyHostToDevice, st->stream));
    rc = dfb_features(st, d_in, C, T, nb_df, alpha, d_spec, d_fe, d_fs, st->stream);
    if (rc) return rc;
    if (Tf > 0) {
        DFB_CUDA(cudaMemcpyAsync(h_spec, d_spec, sizeof(float) * n_spec, cudaMemcpyDeviceToHost, st->stream));
        DFB_CUDA(cudaMemcpyAsync(h_feat_erb, d_fe, sizeof(float) * n_fe, cudaMemcpyDeviceToHost, st->stream));
        DFB_CUDA(cudaMemcpyAsync(h_feat_spec, d_fs, sizeof(float) * n_fs, cudaMemcpyDeviceToHost, st->stream));
    }
    DFB_CUDA(cudaStreamSynchronize(st->stream));
    return DFB_OK;
}

// df/io.py resample (torchaudio.functional.resample): h_audio [C][T] -> h_out [C][T_out]; h_kernel [nw][2 width + og]
extern "C" int dfb_resample_host(int device, const float *h_audio, int64_t C, int64_t T, const float *h_kernel, int og, int nw,
                                 int width, float *h_out, int64_t T_out) {
    if (!h_audio || !h_kernel || !h_out || C <= 0 || T <= 0 || T_out <= 0 || og <= 0 || nw <= 0 || width < 0)
        return fail(DFB_ERR_INVALID, "bad resample argument");
    if (C > 65535) return fail(DFB_ERR_INVALID, "more than 65535 channels per call");
    int rc = use_device(device);
    if (rc) return rc;
    const int K = 2 * width + og;
    Scratch s;
    float *d_in = s.alloc<float>(C * T), *d_out = s.alloc<float>(C * T_out), *d_k = s.alloc<float>((size_t)nw * K);
    if (!d_in || !d_out || !d_k) return fail(DFB_ERR_OOM, "cudaMalloc failed");
    DFB_CUDA(cudaMemcpy(d_in, h_audio, sizeof(float) * C * T, cudaMemcpyHostToDevice));
    DFB_CUDA(cudaMemcpy(d_k, h_kernel, sizeof(float) * (size_t)nw * K, cudaMemcpyHostToDevice));
    const size_t smem = (size_t)nw * K * sizeof(float) <= 96 * 1024 ? (size_t)nw * K * sizeof(float) : 0;
    static PerDeviceOnce attr_once;
    if (auto once_guard = attr_once.first()) DFB_CUDA(cudaFuncSetAttribute(k_resample, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    int64_t blocks = (T_out + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    k_resample<<<dim3((unsigned)blocks, (unsigned)C), 256, smem>>>(d_in, T, d_k, og, nw, width, K, d_out, T_out);
    DFB_LAUNCH_CHECK();
    DFB_CUDA(cudaMemcpy(h_out, d_out, sizeof(float) * C * T_out, cudaMemcpyDeviceToHost));
    return DFB_OK;
}
