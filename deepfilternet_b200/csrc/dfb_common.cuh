// dfb_common.cuh -- shared host-side plumbing of libdfb200.so (error reporting, launch counter,
// grow-only device arena) and the device tables of the DSP state.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/dfb200.h"
#include "dfb_fft_generic.cuh"

namespace dfb {

extern thread_local std::string g_err;
extern std::atomic<int64_t> g_launches;

inline int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define DFB_CUDA(expr)                                                                          \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess)                                                                 \
            return dfb::fail(DFB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                             __FILE__, __LINE__);                                               \
    } while (0)

#define DFB_LAUNCH_CHECK()                                                                      \
    do {                                                                                        \
        dfb::g_launches.fetch_add(1, std::memory_order_relaxed);                                \
        cudaError_t e__ = cudaGetLastError();                                                   \
        if (e__ != cudaSuccess)                                                                 \
            return dfb::fail(DFB_ERR_CUDA, "kernel launch failed: %s (%s:%d)",                  \
                             cudaGetErrorString(e__), __FILE__, __LINE__);                      \
    } while (0)

// Optional per-kernel timing with CUDA events on the launching stream (dfb_profile_* in the C ABI).
// Off by default; when on, every launch site brackets its kernel with two events.
struct ProfScope {
    int slot = -1;
    cudaStream_t s;
    ProfScope(const char *name, cudaStream_t stream);
    ~ProfScope();
};
#define DFB_PROF(name, stream) dfb::ProfScope prof_scope__(name, stream)

// Function attributes (dynamic shared memory limit, cluster size) are per device: launch sites set them the first
// time they run on each device of the process.  `first()` hands the caller a guard that holds the mutex while the
// one-time setup runs, so a second host thread cannot launch before the attribute is in place:
//     if (auto g = once.first()) { cudaFuncSetAttribute(...); }
struct PerDeviceOnce {
    std::mutex mu;
    std::atomic<unsigned long long> done{0};
    struct Guard {
        std::unique_lock<std::mutex> lk;
        PerDeviceOnce *o = nullptr;
        unsigned long long bit = 0;
        Guard() = default;
        Guard(Guard &&g) noexcept : lk(std::move(g.lk)), o(g.o), bit(g.bit) {}
        explicit operator bool() const { return lk.owns_lock(); }
        ~Guard() { if (lk.owns_lock()) o->done.fetch_or(bit, std::memory_order_release); }
    };
    Guard first() {
        int d = 0;
        cudaGetDevice(&d);
        const unsigned long long bit = 1ull << (d & 63);
        Guard g;
        if (done.load(std::memory_order_acquire) & bit) return g;
        g.lk = std::unique_lock<std::mutex>(mu);
        if (done.load(std::memory_order_acquire) & bit) { g.lk.unlock(); g.lk.release(); return g; }
        g.o = this; g.bit = bit;
        return g;
    }
};

// Selects `device` and verifies it is a Hopper (sm_90) part; no CPU fallback exists.
int use_device(int device);

// Grow-only device arena: one cudaMalloc'd slab, bump allocated per call, reset between calls.
struct Arena {
    char *base = nullptr;
    size_t cap = 0, off = 0;
    int reserve(size_t bytes);  // ensure capacity (may reallocate; invalidates old pointers)
    void reset() { off = 0; }
    template <typename T>
    T *take(size_t n) {
        size_t b = (n * sizeof(T) + 255) & ~size_t(255);
        if (off + b > cap) return nullptr;
        T *p = reinterpret_cast<T *>(base + off);
        off += b;
        return p;
    }
    void release();
};

constexpr int kMaxErb = 64;

// Device-resident tables of one DSP state (fft 960 / hop 480 kernels).
struct DspTables {
    const float *window;     // [fft]
    const float2 *tw_a_fwd;  // [24][20]  w480^{-lane k1}
    const float2 *tw_a_inv;  // [24][20]  conj
    const float2 *tw960;     // [241]     e^{-2 pi i k / 960}
    const int *erb_off;      // [E + 1]
    const float *erb_kinv;   // [E]  1 / width
    const unsigned char *band_of_bin;  // [F]
    float wnorm;
    int fft, hop, F, E;
};

// One stream of a batch (dfb_enhance*), in the executor's order (longest first): its samples are
// audio[in_off, in_off + len), its result out[out_off, out_off + out_len), and it has Tf STFT frames.  Kernels that take a
// table index their rows with it; a null table (streaming API, dfb_analysis, dfb_apply) means every row has the call's
// common length.
struct RaggedRow { int64_t in_off, len, out_off, out_len, Tf; };

// Link group of one stream (linked channels, dfb_enhance_ragged's link groups / dfb_stream_set_mask_reduce): the n streams
// first .. first + n - 1 of the kernel's batch, which include this one, are the channels of one recording and share one
// ERB mask.  A separate table rather than more RaggedRow fields: the analysis and input-conv kernels read RaggedRow.
struct LinkRow { int first, n; };
enum { kReduceNone = 0, kReduceMax = 1, kReduceMean = 2 };   // dfb_reduce_mask
// One direction of the resampler of a streaming handle at another rate than the model's (dfb_stream_set_sample_rate):
// torchaudio's sinc taps [nw][K = 2 width + og] for the gcd-reduced rates og -> nw.  Output sample t of a session is 0 for
// t < Z and otherwise sum_k taps[t % nw][k] * x[(t / nw) og - S + k] over the session's input x, taps outside the input
// received so far skipped: the resampled session delayed by Z = m nw output samples, m = ceil(width / og), so that every
// tap a hop's outputs need has arrived with that hop.  A row carries the last S = m og + width input samples between
// calls (S <= hop_in).  hop_in / hop_out: samples per 10 ms hop on either side.  ext: the hops of zero extension a
// session's input ends before its end hop (1; 0 for the identity direction of a 48 kHz slot on a mixed-rate handle:
// og = nw = K = 1, one tap of 1.0, S = Z = 0, which copies its row exactly: fmaf(1, x, +0) is x, but for -0, which
// comes out as +0).
struct ResampleDir { const float *taps; int og, nw, K, S, Z, hop_in, hop_out, ext; };
// The directions of one resampler of a handle, indexed by ResampleRow::dir: one on a handle at one rate, the identity and
// one per registered rate on a mixed-rate handle (dfb_stream_add_slot_rate).
constexpr int kMaxRateDirs = 7;
struct ResampleDirs { ResampleDir d[kMaxRateDirs]; };
// A live row of a resampled call: its slot (row of the caller's buffers), the handle's hop its session started at, the
// end hop of a closed session (as the slot path's rows[].Tf; open: far in the future) and its direction.
struct ResampleRow { int64_t slot, first, end, dir; };
// The buffers of one resampler call of n hops from the handle's hop a0: row r reads in + slot * in_pitch + in_col * hop_in
// and writes n * hop_out samples to out + slot * out_pitch + out_col * hop_out, then zeros up to sample out_w of its row
// (none when out_w ends before them); hist [rows][hist_pitch] are the rows' carried histories; tail: the hops a session's output runs past its end hop.
struct ResampleIO {
    const float *in;
    float *out, *hist;
    int64_t in_pitch, out_pitch, out_w, hist_pitch, in_col, out_col, n, a0, tail;
};
// One direction of a model's offline resampler (dfb_model_add_rate; DESIGN.md section 5i): torchaudio's sinc taps
// [nw][K = 2 width + og] for the gcd-reduced rates og -> nw.  Output t of a stream is sum_k taps[t % nw][k] x[(t / nw) og -
// width + k] over k = 0 .. K-1 in that order, taps outside the stream's input skipped: k_resample's sum, bit for bit.
struct RateDir { const float *taps; int og, nw, K, width; };
// A stream of a rated batch (dfb_enhance_ragged with rates) as a resampler launch sees it: in_len input samples at in + in_off,
// out_len outputs at out + out_off, its direction (-1: a 48 kHz stream, which no resampler touches) and its 48 kHz frame
// count tf (it has ended, every 48 kHz output written, once the chunk loop's DNN frames reach tf).
struct RateRow { int64_t in_off, in_len, out_off, out_len, tf; int dir; };
// The buffers and range of one launch.  Up (rate r -> 48 kHz): every row writes its outputs [lo, hi), clipped to its length.
// Down (48 kHz -> r): a row's input is written up to sample w, or entirely once it has ended; it writes the outputs whose
// taps all lie below w, from those complete at (w, d) = (lo, d_lo), which an earlier launch wrote, to those at (hi, d_hi).
struct RateIO { const float *in; float *out; int64_t lo, hi, d_lo, d_hi; };

// Down direction: the outputs of row r complete once its input is written up to w (all of them when it has ended).  Output
// block i's last tap is input i og + width + og - 1.
__host__ __device__ __forceinline__ int64_t rate_down_ready(const RateDir &d, const RateRow &r, int64_t w, bool ended) {
    if (ended || w >= r.in_len) return r.out_len;
    const int64_t span = (int64_t)d.width + d.og;
    if (w < span) return 0;
    const int64_t n = ((w - span) / d.og + 1) * d.nw;
    return n < r.out_len ? n : r.out_len;
}
// Up direction: the input samples the outputs below x read (their taps past the stream's end are skipped).
__host__ __device__ __forceinline__ int64_t rate_up_need(const RateDir &d, const RateRow &r, int64_t x) {
    if (x > r.out_len) x = r.out_len;
    if (x <= 0) return 0;
    const int64_t n = ((x - 1) / d.nw) * d.og + d.width + d.og;
    return n < r.in_len ? n : r.in_len;
}
// The outputs [*o0, *o1) row r writes in launch io.
__host__ __device__ __forceinline__ void rate_range(bool up, const RateDir &d, const RateRow &r, const RateIO &io, int64_t *o0,
                                                    int64_t *o1) {
    if (up) {
        *o0 = io.lo < r.out_len ? io.lo : r.out_len;
        *o1 = io.hi < r.out_len ? io.hi : r.out_len;
    } else {
        *o0 = rate_down_ready(d, r, io.lo, r.tf <= io.d_lo);
        *o1 = rate_down_ready(d, r, io.hi, r.tf <= io.d_hi);
    }
    if (*o1 < *o0) *o1 = *o0;
}

// Per-slot settings of a streaming handle (dfb_stream_set_atten_lim / _post_filter_beta): limit (0 = off) and post-filter
// beta (0 = off) from absolute frame sw on, and the previous ones before it.  Only the frame before sw, re-synthesised
// for its overlap-add tail, still reads the previous ones.  gate != 0: LSNR stage gating with the thresholds th_min /
// th_erb / th_df (tract.rs:658-672), which apply to every frame of the row; it takes effect only in launches that run the
// LSNR head (ApplyParams::lsnr).  Batch rows (dfb_enhance_ragged's settings) have sw = 0: one setting for the whole stream.
struct SlotCtl { float lim, beta, lim0, beta0; int64_t sw; float th_min, th_erb, th_df; int gate; };

// Streaming slots (dfb_stream_open_slots): `first` holds the absolute first frame of each stream of a launch, or is null.
// Window frame t (absolute w0 + t) of stream b exists from the returned window frame on; the kernels that look back in
// time read padding before it, as a fresh stream does before its frame 0.  Null: 0, every frame of the window exists.
__device__ __forceinline__ int stream_first(const int64_t *first, int b, int64_t w0) {
    if (!first) return 0;
    const int64_t d = first[b] - w0;
    return d > 0 ? (int)d : 0;
}

// Initial states of the feature normalisations (libDF/src/lib.rs: linspace(-60, -90, E) and linspace(1e-3, 1e-4, Fd)),
// explicitly rounded so that every kernel that starts a stream produces the same fp32 bits
__device__ __forceinline__ float erb_norm_init(int j, int E) {
    return (E == 1) ? -60.f : __fadd_rn(-60.f, __fmul_rn((float)j, __fdiv_rn(-30.f, (float)(E - 1))));
}
__device__ __forceinline__ float unit_norm_init(int k, int Fd) {
    return (Fd == 1) ? 0.001f : __fadd_rn(0.001f, __fmul_rn((float)k, __fdiv_rn(__fsub_rn(0.0001f, 0.001f), (float)(Fd - 1))));
}

// Parameters of the fused apply + synthesis kernel (dfb_dsp.cu).
// mode 0: plain ISTFT; 1: DeepFilterNet3 (DF on the noisy spectrum); 2: DeepFilterNet2 (DF on the
// masked spectrum).
struct ApplyParams {
    const float2 *spec;   // [B,Tf,F]
    const float *m;       // [B,Tf,E] or null
    const float *coefs;   // [B,Tf,nb_df,2*order] or null
    float *audio;         // [B, out_stride] or null
    float2 *spec_out;     // optional [B,Tf,F]: enhanced spectrum (dfb_apply) or null
    int64_t out_stride;
    int64_t out_offset;   // first synthesised sample that is written (n_fft - hop when pad)
    int64_t out_len;
    int Tf, mode, nb_df, order, lookahead;
    // time-chunked execution (0 = whole signal): the spectrum buffer holds spec_T frames per stream of which Tv exist
    // (rows >= Tv are the end of the stream: zero for the deep filter taps), m / coefs hold Tf; audio of frames < t_first
    // is not written (they belong to the previous window and are only re-synthesised for the overlap-add tail)
    int spec_T, Tv, t_first;
    int mc_T;             // frames per stream in m / coefs (0 = Tf)
    int frames_per_warp;  // consecutive frames one warp synthesises (set by the launcher)
    // optional stages: post filter (DFN3: on the enhanced spectrum, deepfilternet3.py:448-454; DFN2: on the ERB gains,
    // modules.py:234-245 with beta = 0.02) and mask_only (run_df = False: no deep filter, every bin takes the ERB gain)
    int pf, mask_only;
    float pf_beta;
    // LSNR stage gating of the streaming runtime (libDF/src/tract.rs:658-672), mode 1 only: lsnr [B][mc_T] or null;
    // lsnr < th_min -> zero gains, no DF; > th_erb -> frame passes unprocessed; > th_df -> gains only; else gains + DF
    const float *lsnr;
    float th_min, th_erb, th_df;
    // DeepFilterNet v1 (mode 2): alpha [B][mc_T] or null; DF bins <- alpha * deep filter + (1 - alpha) * masked bin
    // (assign_df, modules.py:470-478)
    const float *alpha;
    float atten_lim;      // 0 = off
    // carried ISTFT state (pyDF synthesis(reset=False), mode 0 only): channel 0 starts from init_tail,
    // channel c > 0 from the tail left by channel c - 1; the tail after the last frame goes to final_tail
    const float *init_tail;  // [hop] or null
    float *final_tail;       // [hop] or null
    int carry;
    // ragged batch (or null): row b reads rows[b] for its output row and its end.  Window frame t is absolute frame w0 + t;
    // spectrum rows >= rows[b].Tf - w0 do not exist, and the stream synthesises frames up to rows[b].Tf - w0 when that is
    // <= Tf (it ends in this window), else up to t_emit
    const RaggedRow *rows;
    int64_t w0;
    int t_emit;
    // streaming slots (with rows, or null): frames before stream b's first frame (stream_first) synthesise to zero.  Their
    // spectrum is zero, but the deep filter's look-ahead taps of the last of them reach the stream's first frames, which a
    // fresh stream never synthesises before.
    const int64_t *first;
    // linked channels (or null, specialised kernel with rows only): stream b applies the mask of its link group links[b] reduced
    // over the group's streams (reduce: kReduceMax or kReduceMean, tract.rs:868-902) wherever it applies m, and LSNR
    // gating reads the LSNR of the group's first stream.  Everything else -- deep filter, DeepFilterNet3's post filter,
    // the attenuation limit, the ISTFT -- stays per stream.
    const LinkRow *links;
    int reduce;
};

}  // namespace dfb

struct dfb_state;
namespace dfb {
// frame window of launch_analysis: frames [t_begin, t_begin + nf) of a signal of at most T samples per row go to rows
// out_t0 ... of buffers holding Tbuf frames per stream.  Stream b starts at audio + rows[b].in_off and its samples
// >= rows[b].len read as zero
struct AnaWindow { int t_begin, nf, out_t0, Tbuf; const RaggedRow *rows; };
int launch_analysis(dfb_state *st, const float *d_audio, int64_t C, int64_t T, float *d_spec, float *d_erb_db,
                    cudaStream_t s, const float *d_init_mem = nullptr, const AnaWindow *w = nullptr);
// Ts: frames per stream in the buffers (0 = Tf; pointers pre-offset to the first frame); *_state_out: EMA states after
// the last frame (may be null / alias the inputs); ref_bits: the reference loop's bits at any length (libdf.erb_norm /
// unit_norm): the one-thread scan, never the time-segmented one, with the reference's |x|
int launch_feat_norm(const float *d_erb, int E, int64_t erb_stride, const float *d_spec, int Fd, int64_t spec_stride,
                     int64_t C, int64_t Tf, float alpha, const float *d_erb_state, const float *d_unit_state,
                     float *d_feat_erb, float *d_feat_spec, cudaStream_t s, int64_t Ts = 0, float *d_erb_state_out = nullptr,
                     float *d_unit_state_out = nullptr, bool ref_bits = false);
// ctl (or null): per-stream settings of streaming slots (SlotCtl; specialised RG kernel only).  Stream b's attenuation limit
// and DeepFilterNet3 post-filter beta are ctl[b].lim / beta for absolute frames >= ctl[b].sw and lim0 / beta0 before it,
// in place of p.atten_lim / pf / pf_beta.  A kernel argument of its own after ApplyParams, so that the parameter layout
// of the other instantiations stays as it was.
int launch_apply_synthesis(dfb_state *st, const ApplyParams &p, int64_t B, cudaStream_t s, const SlotCtl *ctl = nullptr);
// One call of n hops through a streaming resampler (k_resample_up / k_resample_down), one CTA per row of rows[0, nb),
// each with the direction dirs.d[row.dir] and the buffers of io (up: a session's input ends at hop end - ext; io.in null:
// no input; down: zeros from hop end + tail on).
int launch_resample_stream(cudaStream_t s, bool up, const ResampleDirs &dirs, int n_dirs, const ResampleRow *rows, int nb,
                           const ResampleIO &io);
// One launch of the offline resampler (k_resample_rows) over the rows [0, nb) of a rated batch: d_dirs / d_rows on the
// device, max_out the most outputs any row writes in it.  A direction of at most smem_floats taps (<= kRateSmemFloats) is
// read from shared memory.
constexpr int kRateSmemFloats = 12288;   // 48 KB: no opt-in, and at least four CTAs per SM
int launch_resample_rows(cudaStream_t s, bool up, const RateDir *d_dirs, const RateRow *d_rows, int nb, const RateIO &io,
                         int64_t max_out, int smem_floats);
// time window of a recurrence launch: steps 0 .. T-1 are frames t0 .. of buffers holding Ts frames per stream; h0 (null:
// zeros) / hT (null: not stored) are the carried hidden states [B][H]
struct GruWindow {
    const float *h0; float *hT; int t0, Ts; const int64_t *first = nullptr; int64_t w0 = 0; /* stream_first */
    const unsigned char *run = nullptr;   /* or run flags [B][Ts]: a step whose flag is 0 keeps the state (k_gru_tc HOLD) */
};
// tensor-core GRU recurrence, H = 256 or 512 (dfb_tc.cu); hout may be null when the planes hout_hi / hout_lo are given.
// ns = 0, xg = -1: the production choice of instance; otherwise the instance <ns, H, xg> (dfb_debug_gru_tc)
int launch_gru_tc(cudaStream_t s, const float *xproj, const float *whh, const float *bhh, const float *res, float *hout,
                  unsigned short *hout_hi, unsigned short *hout_lo, int B, int T, long long *dbg = nullptr, int wide = 0,
                  int planes_res = 0, const GruWindow *w = nullptr, int H = 256, int ns = 0, int xg = -1);
// BF16x3 tensor-core GEMM on hi/lo planes (dfb_tc.cu)
int launch_gemm_bf16x3(cudaStream_t s, const void *x_hi, const void *x_lo, int64_t ldx, const void *w_hi, const void *w_lo,
                       const float *bias, float *y, int64_t ldy, int64_t M, int N, int K);
// BF16x3 tensor-core grouped linear on hi/lo planes + host-packed weight image (dfb_gl.cu); DFB_ERR_UNSUPPORTED when the
// shape is outside the kernel (the caller falls back to the FFMA kernel)
int launch_gl_bx(cudaStream_t s, const unsigned short *x_hi, const unsigned short *x_lo, int64_t ldx, const float *w_img,
                 const float *res, int64_t ldr, float *y, int64_t ldy, unsigned short *y_hi, unsigned short *y_lo, int64_t ldp,
                 int64_t M, int G, int Ig, int Hg, int act, float oscale, float ooffset);
bool gl_bx_geometry(int G, int Ig, int Hg, int *gpc_out, int *hgp_out, int *stages_out);
// df_conv1 -> df_fc_emb in one kernel, c1 kept on chip (dfb_gl.cu): emb_in planes = relu(GL(dwpw(c0))) (+ res)
bool df_emb_geometry(int Fd, int G, int Ig, int Hg, int kt, int *s_out, int *stages_out);
int launch_df_emb(cudaStream_t s, const float *c0, int64_t M, int T, int Fd, int kt, const float *dw, const float *bias,
                  const float *pw_sw, const float *w_img, int G, int Ig, int Hg, const float *res, int64_t ldr,
                  unsigned short *y_hi, unsigned short *y_lo, int64_t ldp, const int64_t *first, int64_t w0);
// DF pathway conv (df_convp) on tensor cores (dfb_tc.cu): df_convp_built says which (df_order, df_pathway_kt) have a
// kernel instance (df_order 5, kt 1 to 5); launch_df_convp_tc refuses the others with DFB_ERR_UNSUPPORTED
bool df_convp_built(int order, int kt);
int launch_df_convp_tc(cudaStream_t s, const float *c0, const float *w_sw, const float *w2, const float *bias, float *coefs, int B, int T,
                       int Fd, int order, int kt, const int64_t *first = nullptr, int64_t w0 = 0);
// fp32 [M][K] -> BF16 hi / lo planes [M][K]
int launch_to_planes(cudaStream_t s, const float *x, int64_t ldx, int64_t M, int K, unsigned short *hi, unsigned short *lo);
}  // namespace dfb

struct dfb_state {
    int device, sr, fft, hop, nb_erb, min_nb_erb_freqs;
    std::vector<int64_t> erb;
    std::vector<float> window;
    void *d_tables = nullptr;  // one slab holding every table
    dfb::DspTables tb{};
    dfb::GenFftPlan plan{};    // generic real FFT of fft_size (states other than fft 960 / hop 480); tw in d_tables
    dfb::Arena arena;          // scratch of the *_host entry points
    cudaStream_t stream = nullptr;
    // STFT / ISTFT memories carried between calls (libDF analysis_mem / synthesis_mem, lib.rs:60-62)
    std::vector<float> analysis_mem, synthesis_mem;
};
