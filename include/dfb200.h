/*
 * dfb200.h -- C ABI of libdfb200.so: the H100 (sm_90a) implementation of DeepFilterNet's
 * per-frame enhancement path (STFT -> ERB / complex features -> encoder / GRUs / decoders ->
 * gain mask + deep filter -> ISTFT).
 *
 * The reference has NO C ABI for this batched path: its boundary is the PyO3 module `libdf`
 * (pyDF/src/lib.rs) plus the Python functions in DeepFilterNet/df/enhance.py.  Each entry point
 * below names the reference interface it replaces; INTEGRATION.md shows the binding a reference
 * maintainer would add (ctypes stubs that stand in for pyDF's #[pymethods]).
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / numpy types cross this boundary.
 *   - every function returns 0 on success or a negative dfb_status; dfb_last_error() returns a
 *     thread-local human readable message for the last failure.
 *   - "_host" entry points take HOST pointers and do the host<->device copies themselves (on the
 *     handle's stream, synchronised before returning); the others take DEVICE pointers valid on
 *     the handle's device and are asynchronous on `stream` (a cudaStream_t passed as void*).
 *   - complex data are interleaved (re, im) float pairs, exactly numpy complex64 / Rust Complex32.
 *   - there is no CPU fallback: every function fails with DFB_ERR_CUDA when no sm_90 device is
 *     usable.
 */
#ifndef DFB200_H
#define DFB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    DFB_OK = 0,
    DFB_ERR_INVALID = -1,     /* bad argument (shape, null pointer, unsupported size) */
    DFB_ERR_CUDA = -2,        /* CUDA runtime / launch failure, or no usable device    */
    DFB_ERR_UNSUPPORTED = -3, /* configuration outside the built kernels               */
    DFB_ERR_OOM = -4
} dfb_status;

const char *dfb_last_error(void);
/* ABI / build info: "dfb200 <version> sm_90a" */
const char *dfb_version(void);
/* number of CUDA kernels this library has launched in the calling process (all handles) */
int64_t dfb_kernel_launches(void);

/* Per-kernel timing with CUDA events on the launching stream (used by bench.py for the roofline
 * numbers).  on != 0 enables it; only_kernel (may be NULL) restricts it to one kernel name.
 * dfb_profile_report synchronises the device, writes "name count total_ms\n" lines for everything
 * recorded since the previous report into buf and returns the number of bytes written. */
int dfb_profile_enable(int on, const char *only_kernel);
int64_t dfb_profile_report(char *buf, int64_t buflen);

/* ------------------------------------------------------------------ DSP state ------------
 * Replaces libDF `DFState` as exposed by pyDF `DF` (pyDF/src/lib.rs:14-136,
 * libDF/src/lib.rs:104-154).  Holds the vorbis window, FFT twiddles and ERB tables on the device.
 * The analysis / synthesis memories (lib.rs:60-62) are carried by the *_host_ex entry points exactly as
 * pyDF does with `reset=False`; the device-pointer entry points and the fused enhance path always start
 * each channel from the reset state (pyDF's default `reset=True`, pyDF/src/lib.rs:56-58, 91-93). */
typedef struct dfb_state dfb_state;

/* pyDF DF.__new__ (pyDF/src/lib.rs:22-39) -> DFState::new (libDF/src/lib.rs:104-154).
 * device: CUDA ordinal.  fft_size 2 ... 8192 (odd or even) and 1 <= hop_size <= fft_size / 2; fft_size > 8192 returns
 * DFB_ERR_UNSUPPORTED.  The STFT / ISTFT / feature entry points run at every such size (fft 960 / hop 480 on the
 * specialised kernels of the shipped models, every other size on the generic real FFT); the model path (dfb_enhance*,
 * dfb_apply, dfb_model_forward_full, dfb_stream_create) returns DFB_ERR_UNSUPPORTED for a state other than 960 / 480.
 * With reset == 0, the *_host_ex entry points carry fft_size - hop_size samples of memory, as DFState does. */
int dfb_state_create(dfb_state **out, int device, int sr, int fft_size, int hop_size, int nb_erb,
                     int min_nb_erb_freqs);
void dfb_state_free(dfb_state *st);
/* pyDF erb_widths / fft_window / sr / fft_size / hop_size / nb_erb (pyDF/src/lib.rs:109-131) */
int dfb_state_erb_widths(const dfb_state *st, int64_t *widths /* [nb_erb] host */);
int dfb_state_fft_window(const dfb_state *st, float *window /* [fft_size] host */);
int dfb_state_params(const dfb_state *st, int *sr, int *fft_size, int *hop_size, int *nb_erb);
/* ERB band widths only, no device needed: libDF erb_fb (libDF/src/lib.rs:68-100) */
int dfb_erb_widths(int sr, int fft_size, int nb_erb, int min_nb_freqs, int64_t *widths);

/* pyDF DF.analysis (pyDF/src/lib.rs:41-72) -> frame_analysis (libDF/src/lib.rs:356-394).
 * audio f32[C, T] (row stride T) -> spec c64[C, T / hop, F].  Trailing partial frame dropped. */
int dfb_analysis(dfb_state *st, const float *d_audio, int64_t C, int64_t T, float *d_spec, void *stream);
int dfb_analysis_host(dfb_state *st, const float *h_audio, int64_t C, int64_t T, float *h_spec);
/* same with pyDF's `reset` argument: reset == 0 carries the STFT memory across calls and channels exactly like
 * the shared DFState of the reference (channel 0 continues the previous call, channel c continues c - 1) */
int dfb_analysis_host_ex(dfb_state *st, const float *h_audio, int64_t C, int64_t T, int reset, float *h_spec);
/* pyDF DF.reset (pyDF/src/lib.rs:133-135): zero the carried analysis / synthesis memories */
int dfb_state_reset(dfb_state *st);

/* pyDF DF.synthesis (pyDF/src/lib.rs:74-107) -> frame_synthesis (libDF/src/lib.rs:396-427).
 * spec c64[C, Tf, F] -> audio f32[C, Tf * hop].  Does NOT clobber its input (the reference does). */
int dfb_synthesis(dfb_state *st, const float *d_spec, int64_t C, int64_t Tf, float *d_audio, void *stream);
int dfb_synthesis_host(dfb_state *st, const float *h_spec, int64_t C, int64_t Tf, float *h_audio);
int dfb_synthesis_host_ex(dfb_state *st, const float *h_spec, int64_t C, int64_t Tf, int reset, float *h_audio);

/* libdf.erb (pyDF/src/lib.rs:142-192) -> compute_band_corr (+dB) (libDF/src/lib.rs:280-295,
 * transforms.rs:236-253).  spec c64[n_frames, F] -> f32[n_frames, E]; widths host int64[E]. */
int dfb_erb_host(int device, const float *h_spec, int64_t n_frames, int64_t F, const int64_t *widths, int E,
                 int db, float *h_out);
/* libdf.erb_inv (pyDF/src/lib.rs:194-250) -> interp_band_gain (libDF/src/lib.rs:328-337). */
int dfb_erb_inv_host(int device, const float *h_gains, int64_t n_frames, const int64_t *widths, int E,
                     float *h_out /* [n_frames, sum(widths)] */);
/* libdf.erb_norm (pyDF/src/lib.rs:252-274) -> band_mean_norm_erb (libDF/src/lib.rs:244-251).
 * erb f32[C, T, E] -> out f32[C, T, E]; state f32[C, E] or NULL (linspace(-60,-90,E)). */
int dfb_erb_norm_host(int device, const float *h_erb, int64_t C, int64_t T, int64_t E, float alpha,
                      const float *h_state, float *h_out);
/* libdf.unit_norm (pyDF/src/lib.rs:276-298) -> band_unit_norm (libDF/src/lib.rs:253-259).
 * spec c64[C, T, F] -> out c64[C, T, F]; state f32[C, F] or NULL (linspace(1e-3,1e-4,F)). */
int dfb_unit_norm_host(int device, const float *h_spec, int64_t C, int64_t T, int64_t F, float alpha,
                       const float *h_state, float *h_out);
/* libdf.unit_norm_init (pyDF/src/lib.rs:300-307) */
int dfb_unit_norm_init(int64_t n, float *h_out);

/* df.enhance.df_features (DeepFilterNet/df/enhance.py:190-203) as ONE fused device pass:
 * audio f32[C,T] -> spec c64[C,Tf,F], feat_erb f32[C,Tf,E], feat_spec c64[C,Tf,nb_df]. */
int dfb_features(dfb_state *st, const float *d_audio, int64_t C, int64_t T, int nb_df, float alpha,
                 float *d_spec, float *d_feat_erb, float *d_feat_spec, void *stream);
int dfb_features_host(dfb_state *st, const float *h_audio, int64_t C, int64_t T, int nb_df, float alpha,
                      float *h_spec, float *h_feat_erb, float *h_feat_spec);

/* df.io.resample (DeepFilterNet/df/io.py:107-129 -> torchaudio.functional.resample): polyphase sinc resampling on the
 * device.  h_kernel f32[new][2 * width + orig] are the taps of torchaudio's _get_sinc_resample_kernel for the gcd-reduced
 * rates (orig, new); audio f32[C][T] -> out f32[C][T_out], T_out = ceil(new * T / orig). */
int dfb_resample_host(int device, const float *h_audio, int64_t C, int64_t T, const float *h_kernel, int orig, int new_rate,
                      int width, float *h_out, int64_t T_out);

/* ------------------------------------------------------------------ model ------------------
 * Replaces the forward pass of DeepFilterNet/df/deepfilternet3.py (DfNet :334-456) and
 * deepfilternet2.py (DfNet :374-505) for the shipped DeepFilterNet2 / 3 / 3_ll topologies. */
typedef struct dfb_model dfb_model;

typedef struct {
    int32_t model_kind;      /* 2 = DeepFilterNet2, 3 = DeepFilterNet3 (incl. _ll)          */
    int32_t nb_erb, nb_df, df_order, df_lookahead, conv_lookahead;
    int32_t conv_ch;         /* 64                                                           */
    int32_t conv_kt;         /* time taps of the `conv_kernel` layers (1; _ll: 2)            */
    int32_t inp_kt;          /* time taps of conv_kernel_inp (3)                             */
    int32_t emb_hidden, df_hidden;
    int32_t enc_gru_layers, erb_gru_layers, df_gru_layers;
    int32_t df_pathway_kt;   /* 5; 3 for DeepFilterNet2_ll; kernel instances for 1 to 5 at df_order 5 */
    int32_t enc_concat;      /* DFN2: 1 */
    int32_t g_df_fc_emb, g_enc_in, g_enc_out, g_erb_in, g_erb_out, g_df_in, g_df_skip, g_df_out;
    float lsnr_scale, lsnr_offset;
    float norm_alpha;        /* feature normalisation decay, df/utils.py:108-124 (0.99) */
} dfb_model_config;

/* One named fp32 tensor of the packed weight set (BatchNorm already folded, layouts as documented
 * in deepfilternet_b200/weights.py).  `data` is a HOST pointer; it is copied to the device. */
typedef struct {
    const char *name;
    const float *data;
    int64_t numel;
} dfb_tensor;

/* Replaces init_model + load_state_dict (deepfilternet3.py:80-87, checkpoint.py:46-104).  Rejects a weight set that
 * lacks a tensor, or has a tensor of the wrong size, for the layers the config runs (DFB_ERR_INVALID, naming the tensor).
 * Refuses with DFB_ERR_UNSUPPORTED, naming what is built, the shapes the kernels do not build: conv_ch != 64, nb_erb or
 * nb_df not a multiple of 8 or above 64 / 128, 2 * df_order > 16, conv_kt outside 1..2 or inp_kt outside 1..3, GRU
 * hidden sizes other than 256 / 512, a conv_lookahead or df_lookahead outside 0..3 (DeepFilterNet v1: conv_lookahead other
 * than 2), and (DeepFilterNet2 / 3) a grouped linear whose group width (inputs or outputs per group) is not a multiple of 4.  df_order != 5 and df_pathway_kt outside 1..5
 * are accepted here and refused by the first forward pass. */
int dfb_model_create(dfb_model **out, int device, const dfb_model_config *cfg, const dfb_tensor *tensors,
                     int n_tensors, const int64_t *erb_widths);
void dfb_model_free(dfb_model *m);

/* DfNet.forward without the spectral apply (deepfilternet3.py:407-441): features -> ERB mask m,
 * DF coefficients and local SNR.  feat_erb f32[B,T,E], feat_spec c64[B,T,nb_df]
 * -> m f32[B,T,E], coefs f32[B,T,nb_df,2*order], lsnr f32[B,T] (may be NULL), alpha f32[B,T]
 * (DeepFilterNet2's df_fc_a output, deepfilternet2.py:368; may be NULL, ignored for kind 3). */
int dfb_model_forward(dfb_model *m, const float *d_feat_erb, const float *d_feat_spec, int64_t B, int64_t T,
                      float *d_m, float *d_coefs, float *d_lsnr, float *d_alpha, void *stream);

/* Mask.forward + MF.DF.forward (modules.py:248-269, multiframe.py:169-180,
 * deepfilternet3.py:431-443 / deepfilternet2.py:494-503): spec c64[B,T,F], m, coefs -> spec_e. */
int dfb_apply(dfb_model *m, dfb_state *st, const float *d_spec, const float *d_m, const float *d_coefs,
              int64_t B, int64_t T, float *d_spec_e, void *stream);

/* Debug aid: one launch of the apply + ISTFT kernel with the row-level arguments the batch and slot executors pass, the
 * kernel instance chosen as they choose it.  Window frames t = 0 .. Tf-1 (absolute w0 + t) of B streams: spec c64[B][spec_T
 * (0: Tf)][F] of which the first Tv (0: all) rows exist; m f32[B][mc_T (0: Tf)][E], coefs f32[B][mc_T][nb_df][2 order],
 * alpha f32[B][mc_T] (DeepFilterNet v1 only, which needs it), lsnr f32[B][mc_T] or NULL (LSNR stage gating, DeepFilterNet3
 * only).  Frame t's samples [t hop - out_offset, + hop) are written for t >= t_first, and spec_out c64[B][Tf][F] (or NULL)
 * receives each synthesised frame's enhanced spectrum.  HOST tables, each NULL or B entries:
 *   rows   int64 [B][3]  out_off, out_len, Tf: stream b's output row audio[out_off, out_off + out_len) and its end (absolute
 *                        frame Tf; a stream that has not ended in the window synthesises up to t_emit).  NULL: row b is
 *                        audio[b out_len, (b + 1) out_len) and every stream ends at Tf;
 *   first  int64 [B]     streaming slots' first frames (absolute), frames before them synthesise to zero;
 *   links  int32 [B][2]  link group (first stream, n) of stream b, mask reduction `reduce` (DFB_REDUCE_MAX / _MEAN);
 *   ctl    f32 [B][7]    lim, beta, lim0, beta0, th_min, th_erb, th_df of stream b, with ctl_sw int64 [B] (absolute switch
 *                        frame) and ctl_gate int32 [B] (gate flag).
 * first, links and ctl need rows.  Without ctl the thresholds and atten_lim (a factor, 0 = off) apply to every row. */
int dfb_debug_apply_rows(dfb_model *m, dfb_state *st, const float *d_spec, int spec_T, int Tv, const float *d_m,
                         const float *d_coefs, const float *d_alpha, const float *d_lsnr, int mc_T, int64_t B, int Tf,
                         int t_first, int t_emit, int64_t w0, const int64_t *h_rows, const int64_t *h_first,
                         const int32_t *h_links, int reduce, const float *h_ctl, const int64_t *h_ctl_sw,
                         const int32_t *h_ctl_gate, float th_min, float th_erb, float th_df, float atten_lim,
                         int64_t out_offset, int64_t out_len, float *d_audio, float *d_spec_out, void *stream);

/* DfNet.forward (deepfilternet3.py:389-456): (spec, feat_erb, feat_spec) -> (spec_e, m, lsnr, coefs);
 * any of d_m / d_lsnr / d_coefs / d_alpha may be NULL. */
int dfb_model_forward_full(dfb_model *m, dfb_state *st, const float *d_spec, const float *d_feat_erb,
                           const float *d_feat_spec, int64_t B, int64_t T, float *d_spec_e, float *d_m,
                           float *d_lsnr, float *d_coefs, float *d_alpha, void *stream);

/* df.enhance.enhance (DeepFilterNet/df/enhance.py:206-250), the whole path in one call:
 * audio f32[B,T] -> enhanced f32[B,T_out].  pad != 0: zero-pad fft_size samples at the end and
 * crop the STFT delay (T_out = T); pad == 0: T_out = (T / hop) * hop, delayed by fft - hop.
 * atten_lim_db <= 0 disables the attenuation limit (enhance.py:238-240).
 * The apply + ISTFT stage is one fused kernel (gain x spectrum + deep filter + irFFT + OLA).
 * The signal is processed in time chunks with carried state (see "streaming" below), so the device workspace does
 * not grow with T; dfb_enhance_host additionally overlaps the H2D / D2H copies of neighbouring chunks with the compute.
 * An equal-length batch runs on the same executor as the ragged batch below, with stream b = {b * T, T, b * T_out}. */
int dfb_enhance(dfb_model *m, dfb_state *st, const float *d_audio, int64_t B, int64_t T, int pad,
                float atten_lim_db, float *d_out, void *stream);
int dfb_enhance_host(dfb_model *m, dfb_state *st, const float *h_audio, int64_t B, int64_t T, int pad,
                     float atten_lim_db, float *h_out);
/* output length of dfb_enhance for a given input length */
int64_t dfb_enhance_out_len(const dfb_state *st, int64_t T, int pad);
/* Rated batches: streams at their own sample rates, resampled to and from 48 kHz on the device (DESIGN.md section 5i).
 * dfb_model_add_rate registers rate r on the model, with the arguments of dfb_stream_add_slot_rate: up_taps / down_taps
 * [nw][2 width + og] (HOST arrays) are io.resample_kernel(r, 48000) / (48000, r) with the sinc_fast parameters, og / nw the
 * gcd-reduced rates (DFB_ERR_INVALID otherwise).  Every integer rate whose two tables hold at most 2^18 floats together is
 * supported (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 88200, 96000 among them; 11025 is the largest, 230,794);
 * any other is DFB_ERR_UNSUPPORTED.  48000 is the identity and registers nothing; registering a rate twice registers it once.
 * Synchronises the model's device. */
int dfb_model_add_rate(dfb_model *m, int rate, const float *up_taps, int up_og, int up_nw, int up_width,
                       const float *down_taps, int down_og, int down_nw, int down_width);
/* Ragged batch: B streams of different lengths in one call, optionally linked, at their own rates, with per-stream
 * settings and LSNR rows (DESIGN.md sections 5b, 5i, 5k).  group_sizes, rates, settings and d_lsnr / h_lsnr may each be
 * null, which turns that part off.
 *
 * Layout.  Stream b is lengths[b] samples at audio + in_offsets[b]; its result, dfb_enhance_out_len(st, lengths[b], pad)
 * samples, goes to out + out_offsets[b].  Nothing else in `out` is written.  in_offsets / lengths / out_offsets are HOST
 * arrays; in_numel / out_numel bound them.  Every stream's output equals dfb_enhance of that stream alone (fp32 reduction
 * order aside) -- which zero-padding the batch to its longest stream does not give: the padded frames would change the
 * look-ahead of every shorter stream's last frames.  Offsets cover a padded [B, S] tensor (in_offsets[b] = b * S) as well as
 * streams packed back to back.  The streams run longest first; a time chunk computes only the streams that have frames left
 * in it, so a batch of mixed lengths costs about its true frame count, not B times the longest.  DeepFilterNet v1 (one
 * window per signal) runs streams of the same frame count together, so a batch of v1 streams saves no frames.  The _host
 * variant takes host pointers (page-locked memory lets its copies overlap the compute), copies only the streams' own samples
 * and results, stages one stream group at a time on the device, and is synchronous.
 *
 * Link groups (group_sizes null: no links, and reduce_mask is ignored).  Linked channels: the Rust runtime's mask reduction
 * over the channels of one recording (libDF/src/tract.rs:95-99, 868-902; the default of its LADSPA plugin and, as
 * --reduce-mask, of its deep-filter binary).  A link group is C >= 1 streams of one length, the channels of one recording:
 * group g is the next group_sizes[g] streams in the caller's order (group_sizes is a HOST array of n_groups entries summing
 * to B).  Everything up to the model outputs stays per channel (STFT, features and their normalisation, encoder, GRU
 * states, m_c, coefs_c, lsnr_c).  The ERB mask is then shared:
 *   max:  m[t][e] = max_c m_c[t][e]
 *   mean: m[t][e] = (sum_c m_c[t][e], fp32 in channel order) * fl32(1 / C)
 * and every channel's apply stage uses it wherever it uses its own mask: the ERB gains (bins >= nb_df, or all bins with
 * mask_only), DeepFilterNet2's masked spectrum that feeds its deep filter, and DeepFilterNet2's post filter on the gains.
 * The deep-filter coefficients, DeepFilterNet3's post filter, the attenuation limit and the ISTFT stay per channel.
 * LSNR stage gating (streaming, DeepFilterNet3) makes one decision per group and frame, from the LSNR of the group's
 * FIRST channel: this library's reading of the single scalar the Rust runtime takes from its [ch] LSNR output.
 * With DFB_REDUCE_NONE, or groups of one stream, the result is the unlinked one.  A group is never split across stream
 * groups.  DeepFilterNet3, DeepFilterNet3_ll and DeepFilterNet2.
 *
 * Rates (rates null: every stream at 48 kHz).  With a HOST array rates[B], stream b is lengths[b] samples at rates[b] Hz
 * (48000 or a registered rate, dfb_model_add_rate), and lengths, offsets and in_numel / out_numel count each stream's own
 * samples.  A link group has one rate and one length.  Stream b's result, dfb_enhance_out_len_at(st, lengths[b], pad,
 * rates[b]) samples at out + out_offsets[b], is
 *     io.resample(enhance(io.resample(x_b, r_b, 48000), pad, atten_lim_db), 48000, r_b)
 * with io.resample's sinc_fast taps: the 48 kHz signal the analysis reads and the rate-r output are those of io.resample
 * (k_resample's sums) bit for bit, and the enhancement between them is that of the ragged batch (fp32 reduction order
 * aside).  A 48 kHz stream is enhanced as with rates null, untouched by any resampler.  Only rate-r samples cross PCIe in
 * the _host variant, whose copies overlap the compute as they do at 48 kHz.
 *
 * Settings (settings null: every stream takes atten_lim_db, the model's post filter and no gating).  settings / n_settings:
 * one dfb_enhance_settings per stream, in the caller's order (n_settings == B).  With a table, atten_lim_db is ignored and
 * stream b takes:
 *   atten_lim_db       the rule of the atten_lim_db argument: <= 0 turns the limit off, else lim = 10^(-db / 20); NaN is
 *                      invalid;
 *   post_filter_beta   the DeepFilterNet3 post filter (deepfilternet3.py:448-454) with this beta, finite and >= 0,
 *                      0 = off, in place of the model's option (dfb_model_set_options); DeepFilterNet2's own post filter
 *                      on the ERB gains still follows the model's option;
 *   lsnr_gating != 0   LSNR stage gating (tract.rs:658-672 apply_stages, as dfb_stream_set_lsnr_thresholds) with the
 *                      three thresholds, none NaN.
 * The streams of a link group take one setting: their entries must be equal.  Stream b's result equals that of the batch
 * with stream b's entry given to every stream, bit for bit.  What gating does to the network follows the model's gating mode
 * (dfb_model_set_gating_mode): in DFB_GATING_RUNTIME a gating stream's decoders run only on the frames its stages let
 * through, as in the Rust runtime; a stream that does not gate is computed as in DFB_GATING_APPLY.
 *
 * LSNR rows (d_lsnr / h_lsnr null: no LSNR output).  lsnr_offsets is a HOST array: stream b's LSNR row,
 * dfb_enhance_lsnr_len(st, lengths[b], pad, rates[b]) floats in dB, goes to lsnr + lsnr_offsets[b].  Value j is the LSNR of
 * the 48 kHz STFT frame that 10 ms output hop j carries: DfNet.forward's lsnr[j + 1] of the stream alone with pad != 0 (the
 * output drops the first fft - hop = 480 samples, frame 0's head), lsnr[j] with pad == 0.  The frames are those of the
 * 48 kHz signal at every rate, so a stream at rate r has one value per 10 ms of its output, the last one for the hop its
 * output's last partial hop falls in.  This is the rule of dfb_stream_process_lsnr: hop j carries frame f, and its value is
 * that frame's LSNR, the one gating reads.  The _host variant copies the LSNR rows back chunk by chunk, next to the audio.
 *
 * A table and LSNR rows run on the specialised apply kernel: a table needs df_order 5, nb_df 96 and 32 ERB bands (every
 * shipped model); post_filter_beta > 0 and lsnr_gating need a DeepFilterNet3 topology; DeepFilterNet v1 takes neither a
 * table nor LSNR rows.
 *
 * Errors.  A refused call changes nothing.
 *   DFB_ERR_INVALID      a null model, state, audio, out or layout array; a stream that reaches outside in_numel /
 *                        out_numel, has a length <= 0, or has no frame at 48 kHz (shorter than one hop with pad == 0); an
 *                        unregistered rate; group sizes < 1, above 65535 or not summing to B, a reduce_mask other than
 *                        DFB_REDUCE_*, or a link group whose streams differ in rate or length; n_settings != B, a NaN limit
 *                        or threshold, a beta < 0 or not finite, linked streams whose entries differ; LSNR rows without
 *                        offsets or outside lsnr_numel.
 *   DFB_ERR_UNSUPPORTED  a state other than 960 / 480; DeepFilterNet v1 with a link group of C > 1 (max / mean), a table
 *                        or LSNR rows; a table on a model shape other than the one above; a beta > 0 or gating on a
 *                        topology other than DeepFilterNet3.
 *   DFB_ERR_OOM          the workspace cap (dfb_model_set_max_workspace) cannot hold the largest link group. */
typedef enum { DFB_REDUCE_NONE = 0, DFB_REDUCE_MAX = 1, DFB_REDUCE_MEAN = 2 } dfb_reduce_mask;  /* tract.rs:95-99 */
/* What LSNR stage gating does to the network.  DFB_GATING_APPLY (the default): the stages select what is applied to a
 * frame and the network runs every frame.  DFB_GATING_RUNTIME, as the Rust runtime (tract.rs:478-503): wherever a stream
 * gates, the ERB decoder runs only on the frames with min <= lsnr <= max_erb (stages "gains" and "gains + deep filter"),
 * the DF decoder only on those that also have lsnr <= max_df.  A decoder that does not run on a frame leaves no trace of
 * it: its GRU layers keep their states, and its time-tap layers (the DF pathway conv; convt3 and the mask head of
 * conv_kt = 2 models) read the previous frames it ran on.  Each decoder computes what it would compute run alone on its
 * frames, from zero states, as tract's pulsed erb_dec / df_dec graphs.  The encoder and the LSNR are the same in both
 * modes, and so are the stage rule, the attenuation limit, the post filter and the mask reduction of link groups.  Not
 * built: the Rust runtime's skip of the network after silent hops (tract.rs:513-525) and its pass-through below an
 * attenuation limit of 0.01 dB (tract.rs:543-546).  Gated frames still cost decoder compute. */
typedef enum { DFB_GATING_APPLY = 0, DFB_GATING_RUNTIME = 1 } dfb_gating_mode;
/* The model's gating mode, read by every call that gates (dfb_enhance_ragged with a settings table, streaming and spectral
 * handles that follow the model); a mode other than DFB_GATING_* is DFB_ERR_INVALID and changes nothing.  DeepFilterNet v1
 * takes the mode and still refuses gating. */
int dfb_model_set_gating_mode(dfb_model *m, int mode);
typedef struct {
    float atten_lim_db;
    float post_filter_beta;
    int32_t lsnr_gating;
    float min_db_thresh, max_db_erb_thresh, max_db_df_thresh;
} dfb_enhance_settings;
int dfb_enhance_ragged(dfb_model *m, dfb_state *st, const float *d_audio, int64_t in_numel, const int64_t *in_offsets,
                       const int64_t *lengths, int64_t B, int pad, float atten_lim_db, float *d_out, int64_t out_numel,
                       const int64_t *out_offsets, const int64_t *group_sizes, int64_t n_groups, int reduce_mask,
                       const int32_t *rates, const dfb_enhance_settings *settings, int64_t n_settings, float *d_lsnr,
                       int64_t lsnr_numel, const int64_t *lsnr_offsets, void *stream);
int dfb_enhance_ragged_host(dfb_model *m, dfb_state *st, const float *h_audio, int64_t in_numel, const int64_t *in_offsets,
                            const int64_t *lengths, int64_t B, int pad, float atten_lim_db, float *h_out, int64_t out_numel,
                            const int64_t *out_offsets, const int64_t *group_sizes, int64_t n_groups, int reduce_mask,
                            const int32_t *rates, const dfb_enhance_settings *settings, int64_t n_settings, float *h_lsnr,
                            int64_t lsnr_numel, const int64_t *lsnr_offsets);
/* output length of a stream of T samples at `rate` in a rated batch: ceil(out48 rate / 48000), out48 =
 * dfb_enhance_out_len(st, ceil(T 48000 / rate), pad); -1 for a null state, T <= 0 or rate <= 0 */
int64_t dfb_enhance_out_len_at(const dfb_state *st, int64_t T, int pad, int rate);
/* LSNR values of a stream of T samples at `rate` in dfb_enhance_ragged: ceil(out48 / 480), out48 =
 * dfb_enhance_out_len(st, ceil(T 48000 / rate), pad) (T at 48 kHz); -1 for a null state, T <= 0 or rate <= 0 */
int64_t dfb_enhance_lsnr_len(const dfb_state *st, int64_t T, int pad, int rate);
/* Debug aid: one of a model's offline resamplers (up != 0: rate -> 48 kHz, else 48 kHz -> rate) alone over B rows (B <= 65535):
 * row b is in_lengths[b] samples at d_in + in_offsets[b] (at rates[b] going up, at 48 kHz going down; registered rates
 * only), and its resampled signal, io.resample's length, goes to d_out + out_offsets[b].  The launches are those of a chunk
 * loop with the bounds h_bounds[0 .. n_bounds) (HOST, increasing, > 0): going up, launch c writes the 48 kHz outputs
 * [h_bounds[c - 1], h_bounds[c]); going down, the outputs whose taps lie below input sample h_bounds[c], or all of them
 * once h_bounds[c] reaches the row's end.  Each output is written once, and nothing outside the rows' outputs. */
int dfb_debug_resample_rows(int up, const dfb_model *m, const float *d_in, const int64_t *in_offsets, const int64_t *in_lengths,
                            const int32_t *rates, int64_t B, float *d_out, const int64_t *out_offsets, const int64_t *h_bounds,
                            int64_t n_bounds, void *stream);
/* ------------------------------------------------------------------ streaming -----------------
 * Frame-incremental processing with carried per-stream state: the batched counterpart of the reference's
 * single-stream runtime `DfTract::process` (libDF/src/tract.rs:509-642) and its C ABI (libDF/src/capi.rs:83-253:
 * df_create / df_get_frame_length / df_process_frame / df_free).  The state carried between calls is SURVEY.md
 * Appendix D: STFT / ISTFT memories, normalisation EMAs, GRU hidden states, conv / deep-filter history.
 * Every call feeds n >= 1 hops per stream and returns n hops; the output trails the input by
 * dfb_stream_latency_frames() hops (the model's look-ahead) on top of the STFT's fft - hop samples: the concatenated
 * output equals dfb_enhance(pad = 0) of the concatenated input, delayed by latency * hop samples.  dfb_enhance itself
 * runs on the same time-chunked executor.  Optional stages: the post filter (dfb_model_set_options) and the Rust
 * runtime's LSNR stage gating (dfb_stream_set_lsnr_thresholds), with the decoders skipping gated frames as the runtime's do
 * in DFB_GATING_RUNTIME (dfb_stream_set_gating_mode); not built: its silent-frame skip (tract.rs:516-525). */
typedef struct dfb_stream dfb_stream;
/* capi.rs df_create: B independent streams on the model's device; atten_lim_db <= 0 disables the limit */
int dfb_stream_create(dfb_stream **out, dfb_model *m, dfb_state *st, int64_t B, float atten_lim_db);
void dfb_stream_free(dfb_stream *s);                       /* capi.rs df_free */
int dfb_stream_reset(dfb_stream *s);                       /* back to the initial state (all memories zero) */
int64_t dfb_stream_frame_length(const dfb_stream *s);      /* capi.rs df_get_frame_length: hop size in samples */
int64_t dfb_stream_latency_frames(const dfb_stream *s);    /* hops the output trails the input by */
/* The handle's gating mode (dfb_gating_mode), or -1 to follow the model's (dfb_model_set_gating_mode; the default).  It
 * takes effect from the next call's DNN frames.  A handle that switches to DFB_GATING_RUNTIME continues as if every frame
 * before the switch had been a run frame of both decoders.  Any other mode is DFB_ERR_INVALID and changes nothing. */
int dfb_stream_set_gating_mode(dfb_stream *s, int mode);
/* LSNR stage gating (libDF/src/tract.rs:658-672 apply_stages; defaults -10 / 30 / 20 dB, tract.rs:180-185): per frame,
 * lsnr < min_db_thresh -> zero gains, no deep filter; > max_db_erb_thresh -> the frame passes unprocessed;
 * > max_db_df_thresh -> ERB gains only; else gains + deep filter.  Off by default (the Python path never gates);
 * DeepFilterNet3 topologies only. */
int dfb_stream_set_lsnr_thresholds(dfb_stream *s, int enable, float min_db_thresh, float max_db_erb_thresh,
                                   float max_db_df_thresh);
/* Per-slot LSNR stage gating (the LADSPA plugin's per-instance thresholds): the listed slots gate with these thresholds
 * (enable != 0) or not at all (enable == 0), in place of the handle's setting above, from the next process / flush call on,
 * every frame of that call included.  `slots` as dfb_stream_set_atten_lim (a free slot or a partial group is
 * DFB_ERR_INVALID; DFB_ERR_UNSUPPORTED on linked handles and for models whose apply step is not the specialised kernel).
 * DeepFilterNet3 topologies only when enable != 0 (else DFB_ERR_UNSUPPORTED); a NaN threshold is DFB_ERR_INVALID; a
 * spectral handle, which gates in one pass for all rows, is DFB_ERR_UNSUPPORTED.  Opening a slot and dfb_stream_reset
 * return it to the handle's setting.  A refused call changes nothing. */
int dfb_stream_set_lsnr_thresholds_slots(dfb_stream *s, const int64_t *slots, int64_t n, int enable, float min_db_thresh,
                                         float max_db_erb_thresh, float max_db_df_thresh);
/* Linked channels (see dfb_enhance_ragged's link groups): streams g * channels + c form link group g; B % channels == 0.
 * Only on a new or reset handle (DFB_ERR_INVALID after the first frame: the frame re-synthesised for the overlap-add
 * tail would mix two settings) that has had no slot operation (DFB_ERR_UNSUPPORTED).  channels = 1 or DFB_REDUCE_NONE:
 * unlinked (the default); channels = 1 also records reduce_mask as the reduction of the slot groups that
 * dfb_stream_open_linked opens later (one mode per handle; it survives dfb_stream_reset, as the channel groups do). */
int dfb_stream_set_mask_reduce(dfb_stream *s, int channels, int reduce_mask);
/* capi.rs df_process_frame, batched and for n_frames hops at once: d_in / d_out f32[B][n_frames * hop] (device) */
int dfb_stream_process(dfb_stream *s, const float *d_in, int64_t n_frames, float *d_out, void *stream);
/* end of stream: the latency frames still in flight, d_out f32[B][latency * hop]; closes every open slot (below), so
 * afterwards every slot is free until it is opened or the handle is reset */
int dfb_stream_flush(dfb_stream *s, float *d_out, void *stream);
/* host pointers, synchronous; h_in == NULL flushes into h_out f32[B][latency * hop] (may be NULL when latency is 0) */
int dfb_stream_process_host(dfb_stream *s, const float *h_in, int64_t n_frames, float *h_out);

/* Streaming slots: each of a handle's B slots is one stream that starts and ends on its own (a service opens a slot when
 * a call starts, as capi.rs df_create, and closes it when the call ends, as df_free).  At creation and after
 * dfb_stream_reset every slot is open.  Slot operations take effect at the next process / flush call; `slots` is a HOST
 * array of n slot indices, each in [0, B) and listed once (DFB_ERR_INVALID otherwise).
 *   open:  each listed slot starts a new stream from the initial state, exactly as a fresh handle would; an open or
 *          closing slot's old stream is dropped without its tail.
 *   close: each listed open slot's stream ends after the input it has already been fed.  From the next call on its input
 *          rows are ignored, and over the next dfb_stream_latency_frames() hops its output rows carry what
 *          dfb_stream_flush would give that stream alone, whatever the call sizes; then the slot is free (at once when
 *          the latency is 0).  Closing a slot that is not open does nothing.
 *   free:  not computed; its input rows are ignored and its output rows are zeros.
 * Row b of process / flush is slot b.  Every session's output equals a single-stream handle fed the same audio in the
 * same call sizes and then flushed.  Only open and closing slots are computed, so the cost of a call follows the number
 * of live streams, not B.  Fixed channel groups (dfb_stream_set_mask_reduce with channels > 1) and slots do not combine:
 * every slot operation on such a handle is DFB_ERR_UNSUPPORTED; slot groups (below) are linked channels that take slot
 * operations.  The handle's clock counts frames since create / reset; calls need it below 2^31 - 2 frames (248 days). */
int dfb_stream_open_slots(dfb_stream *s, const int64_t *slots, int64_t n);
int dfb_stream_close_slots(dfb_stream *s, const int64_t *slots, int64_t n);
/* h_states i32[B] (host): 0 free, 1 open, 2 closing */
int dfb_stream_slot_states(const dfb_stream *s, int32_t *h_states);
/* Slot groups: one session of n channels in n slots, channel c in row slots[c] (n >= 1; DFB_ERR_INVALID for n = 0, and
 * for slots as dfb_stream_open_slots).  The channels share one ERB mask, reduced as the handle's mode says
 * (dfb_stream_set_mask_reduce(s, 1, mode)): the session's output equals a fresh handle with B = n and
 * dfb_stream_set_mask_reduce(s, n, mode), fed the same n rows in the same call sizes and then flushed.  With mode NONE, or
 * n = 1, the group is n unlinked channels.  LSNR stage gating reads the group's channel 0; the LSNR output is each
 * channel's own.  A group moves as a unit: a call that lists any member of a live group of more than one channel
 * (open_slots, open_linked, close_slots, set_atten_lim, set_post_filter_beta) must list all of its members, else it
 * returns DFB_ERR_INVALID and changes nothing.  dfb_stream_open_slots opens n groups of one channel.  Opening over a live
 * group drops its old session without its tail, as a re-opened slot does.  The members share their first and end
 * frames, so they close and become free together; settings made on all members are the group's.  Only the live rows are
 * computed; when a session ends, the rows behind it close up in two kernel launches whatever their number. */
int dfb_stream_open_linked(dfb_stream *s, const int64_t *slots, int64_t n);
/* h_first i64[B] (host): per slot, the slot holding channel 0 of its group (the slot itself for one channel), -1 if free */
int dfb_stream_slot_groups(const dfb_stream *s, int64_t *h_first);

/* Held sessions (DESIGN.md section 5p): a session that has no audio for a call (jitter, discontinuous transmission, a
 * participant on hold) sits the call out, as a libdeepfilter stream that df_process_frame is not called on.  A held
 * session behaves, for every call it is held through, as if that call had not happened: its state, age, settings, LSNR
 * start and drain do not change, its input rows are ignored, its output rows are zeros and its LSNR entries NaN (on a
 * spectral handle NaN rows with stage -1), as a free slot's.  It stays live: dfb_stream_slot_states reports it open or
 * closing, and it keeps its slot.  A session's outputs over the calls it advanced in, followed by its drain or flush,
 * equal a single-stream handle fed the same audio in those calls' sizes, bit for bit.
 *   dfb_stream_hold_slots   hold != 0 holds the listed live slots from the next call on, until hold == 0 lifts it.
 *                           Holding a held slot or lifting an unheld one does nothing.  `slots` as for
 *                           dfb_stream_open_slots; a free slot, or part of a linked group, is DFB_ERR_INVALID; a handle
 *                           with fixed channel groups DFB_ERR_UNSUPPORTED.  A refused call changes nothing.  Holding is a
 *                           slot operation (dfb_stream_set_sample_rate, dfb_stream_add_slot_rate, dfb_stream_set_mask_reduce).
 *   dfb_stream_held_slots   h_held i8[B] (host): 1 per held slot, else 0.
 * Every process entry point respects holds: device, host, _lsnr, spectral, resampled and mixed-rate.
 * Close while held: the session closes at the end of the input it has been fed and drains only in calls it advances in.
 * Settings made while held (dfb_stream_set_atten_lim, _post_filter_beta, _lsnr_thresholds_slots) take effect from the first
 * frame whose output starts in the first call the session advances in.  Holds are lifted by open / open_linked over the
 * slot, dfb_stream_reset, a released export and flush, which ends every session, held ones included, each exactly as its
 * own flush would; an import lands its sessions not held.  Export of a held session (snapshot or release) gives the blob
 * it would have given just before the hold.  DFB_GATING_RUNTIME: a held session keeps its decoder tails and whether its
 * last call kept them; if that call ran in the other gating mode it switches alone, as a handle does (DESIGN.md 5l).  An
 * export lists sessions whose tails agree (else DFB_ERR_INVALID).  DeepFilterNet2 LSNR rows: when the handle's LSNR output
 * first starts while a session is held, that session's first LSNR call after the hold may differ in its first df_lookahead
 * hops (NaN for a value), as after an import; its audio is exact.  Only the advancing rows are computed, so a held session
 * costs no compute; a change of hold state moves at most the rows whose state changed plus as many others, in the same two
 * row-move launches as open and close, at the next call. */
int dfb_stream_hold_slots(dfb_stream *s, const int64_t *slots, int64_t n, int hold);
int dfb_stream_held_slots(const dfb_stream *s, int8_t *h_held);
/* Debug aid: the state-slab rows the handle's last call moved or started fresh before computing (its row-move kernel) */
int dfb_debug_stream_rows_moved(const dfb_stream *s, int64_t *n);

/* Per-slot settings (capi.rs df_set_atten_lim / df_set_post_filter_beta, which each change one stream between two frames).
 * `slots` is validated as for dfb_stream_open_slots; naming a free slot is DFB_ERR_INVALID, an open or closing one is fine
 * (a closing slot's setting covers the rest of its tail).  A refused call changes nothing.  Linked handles:
 * DFB_ERR_UNSUPPORTED, as for every slot operation.  Models whose apply step is not the specialised kernel (df_order 5,
 * nb_df 96, 32 ERB bands, which every shipped model is): DFB_ERR_UNSUPPORTED.
 *   atten_lim_db: the library's rule, as dfb_stream_create: <= 0 turns the limit off, else lim = 10^(-db / 20); NaN is
 *          DFB_ERR_INVALID.  The Rust runtime instead takes |db|, treats >= 100 dB as off and < 0.01 dB as pass-through;
 *          here 100 dB is a limit of 1e-5 and 0.001 dB one of 0.99988.  DeepFilterNet2 and DeepFilterNet3 topologies.
 *   beta:  the DeepFilterNet3 post filter (deepfilternet3.py:448-454), finite and >= 0, 0 = off; anything else is
 *          DFB_ERR_INVALID.  DeepFilterNet2 (whose post filter acts on the ERB gains with a fixed beta, and which the Rust
 *          runtime does not run): DFB_ERR_UNSUPPORTED.
 * A slot without a setting of its own follows the handle: the atten_lim_db it was created with, and the model's
 * post_filter / pf_beta option (dfb_model_set_options) at the time of each call.  Opening a slot returns it to that; a
 * setting made after the open and before the next call applies from the new session's first frame.  dfb_stream_reset
 * drops every setting.  Several settings between the same two calls: the last one wins.
 * When a change takes effect: a setting made between two calls applies to every frame whose output starts in the next
 * process / flush call.  Output hop j of that call is the head of frame f0 + j plus the overlap-add tail of frame
 * f0 + j - 1, so hop 0 is the new setting's head of frame f0 plus the previous setting's tail of frame f0 - 1, as in the
 * Rust runtime, whose synthesis memory was computed in the previous call. */
int dfb_stream_set_atten_lim(dfb_stream *s, const int64_t *slots, int64_t n, float atten_lim_db);
int dfb_stream_set_post_filter_beta(dfb_stream *s, const int64_t *slots, int64_t n, float beta);

/* Local SNR output (capi.rs df_process_frame's return value).  d_lsnr / h_lsnr f32[B][n_frames] (flush: [B][latency]), or
 * NULL: entry [b][j] is the LSNR, in dB, of the frame that output hop j of row b carries -- the value LSNR stage gating
 * reads for that frame (gating itself reads the link group's first channel; linked handles return each channel's own).
 * NaN where the hop carries no frame: a free slot, the first `latency` hops of a handle or of a new session, a closing
 * slot past its tail.  Flush returns the tail frames' LSNR, computed with zero look-ahead like their audio.
 * Alignment: hop j of a call that starts at input hop k carries frame k + j - latency, latency = max(conv_lookahead,
 * df_lookahead) (+ df_lookahead for DeepFilterNet2): 2 for DeepFilterNet3, 4 for DeepFilterNet2, 0 for DeepFilterNet3_ll
 * and DeepFilterNet2_ll.  df_process_frame returns, for input frame k, the LSNR of frame
 * k - conv_lookahead (its encoder sees the features shifted by conv_lookahead, tract.rs:441-548), which is also the frame
 * its output carries.  For DeepFilterNet3 (conv_lookahead = df_lookahead = 2), DeepFilterNet3_ll and DeepFilterNet2_ll
 * (0 / 0) the two agree hop for hop.
 * The LSNR head runs only on handles that ask for it: from the first call with a non-NULL buffer until dfb_stream_reset,
 * every call computes it.  DeepFilterNet2's audio trails its DNN by df_lookahead frames, so at that first call the
 * frames whose DNN step ran in earlier calls have no LSNR and read NaN. */
int dfb_stream_process_lsnr(dfb_stream *s, const float *d_in, int64_t n_frames, float *d_out, float *d_lsnr, void *stream);
int dfb_stream_flush_lsnr(dfb_stream *s, float *d_out, float *d_lsnr, void *stream);
int dfb_stream_process_host_lsnr(dfb_stream *s, const float *h_in, int64_t n_frames, float *h_out, float *h_lsnr);

/* Sample rate of an audio handle: its slots, slot groups and fixed channel groups run at rate r in {8000, 12000, 16000,
 * 24000, 32000, 44100} -- the rates with a whole number of samples per 10 ms hop, h_r = r / 100 -- while inside them the
 * 48 kHz slot path runs unchanged between two resamplers with the taps of df.io.resample's default method, sinc_fast:
 *   R_up = io.resample(., r, 48000), R_down = io.resample(., 48000, r)   (torchaudio's resample; dfb_resample_host)
 * both over a session's audio zero-extended past its end.  up_* / down_* are io.resample_kernel's (kernel [nw][2 width +
 * og], width, og, nw) for (r, 48000) and (48000, r), passed as dfb_resample_host takes them.  Every slot carries its own
 * filter histories, and a new session starts from zero ones.
 * Frames are h_r samples: dfb_stream_process takes and returns [B][n * h_r]; flush, close and the _host variants keep
 * their meaning in units of h_r.  A session of calls n_1 .. n_c (a_1 = sum n_i hops) ended by flush, or by close and its
 * drain, outputs exactly:
 *   1. u' = D_r zeros followed by R_up(x)                                 (48 kHz)
 *   2. y48 = a 48 kHz handle fed u' in the calls n_1 .. n_c, one more call of 1 hop, then flushed
 *   3. E_r zeros followed by R_down(y48), cropped to (a_1 + L + 1) h_r samples   (L: the 48 kHz handle's latency)
 * D_r (48 kHz samples, a multiple of 48000 / gcd(r, 48000)) and E_r (rate-r samples) are the smallest delays with which every
 * call can form its n model hops from the input received so far and return its n h_r samples:
 *   D_r = ceil(width_up / og_up) nw_up,   E_r = ceil(width_down / og_down) nw_down.
 * So dfb_stream_latency_frames is L + 1 (the hops a flush returns and a closing slot drains for), and
 * dfb_stream_latency_samples the signal delay beyond the 48 kHz handle's, D_r r / 48000 + E_r, always below one hop.  The
 * same holds for every session at rate r: on a handle at r, and in a slot opened at r on a mixed-rate handle
 * (dfb_stream_add_slot_rate below):
 *      r    h_r  og/nw/width up  D_r   og/nw/width down  E_r   delay (samples / ms)
 *    8000    80     1/6/17       102       6/1/97         17     34 / 4.25
 *   12000   120     1/4/17        68       4/1/65         17     34 / 2.833
 *   16000   160     1/3/17        51       3/1/49         17     34 / 2.125
 *   24000   240     1/2/17        34       2/1/33         17     34 / 1.417
 *   32000   320     2/3/17        27       3/2/25         18     36 / 1.125
 *   44100   441   147/160/17     160     160/147/18      147    294 / 6.667
 * LSNR rows (NaN rows and stage gating included), per-slot settings, slot groups and re-opened slots behave as at 48 kHz
 * on the model frames of this composition.  Only on a new or reset handle before its first frame and any slot operation
 * (else DFB_ERR_INVALID); it survives dfb_stream_reset.  A spectral handle: DFB_ERR_INVALID (spectra have no rate).  Other
 * rates: DFB_ERR_UNSUPPORTED; 48000 is the plain 48 kHz handle (the taps are ignored and may be NULL).  Taps of other rates
 * or geometry: DFB_ERR_INVALID. */
int dfb_stream_set_sample_rate(dfb_stream *s, int rate, const float *up_taps, int up_og, int up_nw, int up_width,
                               const float *down_taps, int down_og, int down_nw, int down_width);
int64_t dfb_stream_latency_samples(const dfb_stream *s);   /* D_r r / 48000 + E_r; 0 at 48 kHz */
/* Debug aid: one of the two resamplers of a resampled handle on its own (up != 0: k_resample_up, r -> 48 kHz; else
 * k_resample_down, 48 kHz -> r), taps d_taps [nw][2 width + og] (device) as dfb_stream_set_sample_rate takes them.  C rows,
 * each one session from hop 0, run through the calls h_calls[0 .. n_calls) (HOST array of hop counts >= 1) with their
 * histories carried: d_in f32[C][H * hop_in] -> d_out f32[C][H * hop_out], H = sum of the calls, hop = 480 at 48 kHz and
 * h_r at r.  Row c of d_out is the resampled row delayed by D_r (up) or E_r (down) output samples, bit for bit. */
int dfb_debug_resample_stream(int up, int rate, const float *d_taps, int og, int nw, int width, const float *d_in, int64_t C,
                              const int64_t *h_calls, int64_t n_calls, float *d_out, void *stream);

/* Mixed-rate handle: a 48 kHz audio handle whose slots each run at their own rate, so that calls at different rates share
 * one pass through the slot path.  dfb_stream_add_slot_rate registers rate r (one of the rates above, with the arguments
 * of dfb_stream_set_sample_rate); a handle may register several.  Sessions then open at r with dfb_stream_open_slots_at /
 * dfb_stream_open_linked_at (a group at one rate, under the rules of dfb_stream_open_linked), and at 48 kHz with those
 * and rate 48000, or with dfb_stream_open_slots / dfb_stream_open_linked; dfb_stream_reset reopens every slot at 48 kHz.
 *   Row layout: rows stay 480 samples per hop.  dfb_stream_process takes and returns [B][n * 480], and
 *   dfb_stream_frame_length is 480.  A slot at rate r reads the first n h_r samples of its input row and ignores the
 *   rest; its output row carries n h_r samples followed by exact zeros.  The _host and _lsnr variants keep these
 *   meanings, and LSNR rows are one value per hop as on every handle.
 *   Composition: a slot at r outputs, over the first n h_r samples of each call, exactly what a handle at r
 *   (dfb_stream_set_sample_rate) with one slot outputs for that session: the composition above, ended by its close and
 *   L + 1 drain hops or by flush.  A 48 kHz slot outputs what a 48 kHz handle with one slot does (its resamplers copy
 *   its rows value for value: a -0 comes out as +0), and drains for L hops after its close.  Linked groups, per-slot settings, LSNR rows and stage
 *   gating behave as on a handle at the session's rate.
 *   Drain: dfb_stream_latency_frames is L + 1, the longest drain of any slot, and dfb_stream_latency_samples is 0 (a
 *   48 kHz slot's); a session at r has the latency of a handle at r, from the table above.  dfb_stream_flush returns
 *   [B][(L + 1) * 480]: a 48 kHz slot's L tail hops, then one hop of zeros; a slot at r its L + 1 tail hops of h_r
 *   samples each, each row followed by zeros to its end.
 * Errors (DFB_ERR_INVALID unless said otherwise): registering after the handle's first frame or a slot operation (the
 * registrations themselves survive dfb_stream_reset), on a spectral handle, or on a handle set to another rate than
 * 48000; taps of another rate or geometry; a rate outside the list (DFB_ERR_UNSUPPORTED).  Opening at a rate the handle has
 * not registered, or on a handle without slot rates; opening at a rate outside the list and 48000 (DFB_ERR_UNSUPPORTED).
 * dfb_stream_set_sample_rate of a mixed-rate handle to another rate than 48000 (48000 changes nothing).  Registering a
 * rate twice registers it once. */
int dfb_stream_add_slot_rate(dfb_stream *s, int rate, const float *up_taps, int up_og, int up_nw, int up_width,
                             const float *down_taps, int down_og, int down_nw, int down_width);
int dfb_stream_open_slots_at(dfb_stream *s, const int64_t *slots, int64_t n, int rate);
int dfb_stream_open_linked_at(dfb_stream *s, const int64_t *slots, int64_t n, int rate);
/* h_rates [B]: the rate of each live slot's session (the handle's rate on a handle at one rate, 48000 on a 48 kHz one),
 * 0 for a free slot.  A spectral handle: DFB_ERR_INVALID. */
int dfb_stream_slot_rates(const dfb_stream *s, int32_t *h_rates);
/* Debug aid: both resamplers of a handle on their own, with its own taps (up != 0: k_resample_up, else k_resample_down),
 * row c in the direction of rate h_rates[c] (HOST array; a rate the handle runs: its registered rates and 48000 on a
 * mixed-rate handle, its rate on a handle at one rate; else DFB_ERR_INVALID).  Every row is one session from hop 0, run
 * through the calls h_calls[0 .. n_calls) (HOST array of hop counts >= 1) with its histories carried: d_in f32[C][H * 480]
 * -> d_out f32[C][H * 480], H = sum of the calls.  Row c reads its first H hop_in samples and writes H hop_out samples
 * (hop = 480 at 48 kHz and h_r at r) followed by zeros: its row resampled and delayed by D_r (up) or E_r (down) output
 * samples, bit for bit, and a 48 kHz row copied (a -0 as +0). */
int dfb_debug_resample_slots(int up, const dfb_stream *s, const int32_t *h_rates, const float *d_in, int64_t C,
                             const int64_t *h_calls, int64_t n_calls, float *d_out, void *stream);

/* Session export / import (DESIGN.md section 5o): take live sessions out of an audio handle as one blob and resume them in
 * free slots of any compatible handle -- the same one, another one with other neighbours, batch size and clock, one in
 * another process or on another GPU.  A resumed session's next process / flush calls return exactly the hops the source
 * would have returned next, bit for bit for the same neighbour counts (the kernels' fp32 reduction order can follow the
 * number of live rows, as for every session of a slot handle), then it closes and drains as any session does.
 *
 * `slots` is a HOST array of n slot indices (each in [0, B), listed once).  Export lists open sessions only (a free or
 * closing slot is DFB_ERR_INVALID), each linked group whole, from its channel 0 and in channel order (else
 * DFB_ERR_INVALID).  Import lists n free slots (else DFB_ERR_INVALID), one per channel of the blob in blob order; a group
 * lands as a linked group.  A refused call changes nothing.  Spectral handles: DFB_ERR_UNSUPPORTED (DeepFilterNet v1 has
 * no streaming handle).
 *   dfb_stream_session_bytes      the blob's size in bytes for these sessions (checks `slots` as export does).
 *   dfb_stream_export_sessions    packs the sessions into d_blob (device, 4-byte aligned, >= session_bytes) on `stream`
 *                                 and synchronises it: the blob is complete when the call returns.
 *                                 release = 0: a snapshot, the sessions and every other slot continue unchanged, bit for
 *                                 bit.  release != 0: the slots are free at once, without a look-ahead tail: the sessions
 *                                 now live only in the blob.  One kernel launch, whatever the number of sessions.
 *   dfb_stream_import_sessions    resumes the blob at d_blob (device, 4-byte aligned, the whole blob) in free slots of
 *                                 this handle: reads the header, then its records, then one kernel launch, each on
 *                                 `stream`, which it synchronises before returning.  The blob may come from another
 *                                 device: copy it to this handle's first.
 *   _host variants                the blob in host memory: one device copy of the rows per call, on the handle's own
 *                                 stream, synchronised, as dfb_stream_process_host.
 * Every variant returns with its device work done, so the handle's next call may run on any stream.  Work of earlier
 * calls on another stream than the export's / import's must have finished first (synchronise that stream), as for the
 * handle's other calls.
 * Import refuses with DFB_ERR_INVALID, naming the mismatch: another model (fingerprint of dfb_model_create's config, ERB
 * band widths and weight bytes) or DSP state; another gating mode (dfb_stream_set_gating_mode / the model's); a session rate this handle
 * does not run (its rate on a handle at one rate, 48000 and its registered rates on a mixed-rate one); a group whose mask
 * reduction is not the handle's (dfb_stream_set_mask_reduce); a bad magic or version, a size too small for its records,
 * records that do not describe the header's size, or a device blob that is not 4-byte aligned; and, on a handle with live sessions, a clock that has not settled (fewer than 8 + look-ahead
 * frames since its creation, reset or flush) or, in DFB_GATING_RUNTIME, decoder tails kept by the blob's last call where
 * this handle's last call kept none or the reverse.  A handle with no live session takes any blob: its clock moves ahead
 * to where it has settled, as calls with no live slot would move it.
 * What travels: each session's age (frames since its open), rate, group, its settings pinned (the limit, post-filter beta
 * and LSNR gating its next call would resolve, own or the source handle's; the destination's defaults do not reach it;
 * change them with the per-slot setters) with the previous call's settings and switch frame, and the frame its LSNR
 * output starts at.  LSNR rows of DeepFilterNet2 (whose audio trails its DNN by df_lookahead frames): the first LSNR call
 * after an import where exactly one of the two handles had computed LSNR before may differ from the source's in its
 * first df_lookahead hops (NaN for a value or the reverse); every other LSNR value, and the audio, is exact.
 *
 * Blob layout (little-endian, version 1): a header of 192 bytes, n_sessions records of 112 bytes, then the rows.
 *   header   0 u32 magic 0x53424644 ("DFBS")  4 u32 version  8 u64 model fingerprint
 *           16 i32 sr, fft_size, hop_size, nb_erb (the DSP state)  32 i32 gating mode (0 apply, 1 runtime)
 *           36 i32 gate tails (runtime gating: the decoder tails were kept by the last call)  40 i32 n_sessions
 *           44 i32 n_rows (channels)  48 i64 total bytes  56 i64 floats per row of each of the 17 state arrays
 *           (arrays 15 / 16, the resampler histories: the source handle's width)
 *   session  0 i64 age  8 i64 LSNR start frame relative to the session's frame 0 (INT64_MIN: none)  16 i64 switch frame
 *           of the last call's settings (relative)  24 i32 rate  28 i32 channels  32 i32 mask reduction  36 i32 0
 *           40 f32 atten limit (linear, 0 off)  44 f32 beta  48 i32 gate  52 f32 thresholds[3] (min, max erb, max df)
 *           64 f32 last call's limit, beta, previous limit, previous beta  80 i32 last gate  84 f32 last thresholds[3]
 *           96 i32 own up / 100 down resampler history floats  104 i64 byte offset of its rows
 *   rows     per channel: arrays 0 .. 14 (layer-major, as many floats as the header says), then its own up and down
 *           histories (an import pads them with zeros to the handle's width). */
int dfb_stream_session_bytes(const dfb_stream *s, const int32_t *slots, int n, int64_t *bytes);
int dfb_stream_export_sessions(dfb_stream *s, const int32_t *slots, int n, int release, void *d_blob, void *stream);
int dfb_stream_export_sessions_host(dfb_stream *s, const int32_t *slots, int n, int release, void *h_blob);
int dfb_stream_import_sessions(dfb_stream *s, const int32_t *slots, int n, const void *d_blob, void *stream);
int dfb_stream_import_sessions_host(dfb_stream *s, const int32_t *slots, int n, const void *h_blob);

/* Spectral streaming handle (capi.rs df_process_frame_raw, DfTract::process_raw, tract.rs:441-506): the caller runs its own
 * filter bank, passes spectrum frames in and gets the network's outputs back -- ERB gains, deep-filter coefficients, LSNR
 * and the stage LSNR gating picks -- with the features' normalisation, the GRU, conv and norm states carried between
 * calls.  No STFT, nothing applied: dfb_apply and the audio handle do that.  The mode is fixed at creation; a spectral
 * handle takes only the *_spec calls below (dfb_stream_process* / flush* are DFB_ERR_INVALID, and the *_spec calls on an
 * audio handle too), and dfb_stream_set_atten_lim / set_post_filter_beta, which are apply-stage settings, are
 * DFB_ERR_UNSUPPORTED.  Slots, slot groups, dfb_stream_set_mask_reduce, dfb_stream_reset and the LSNR thresholds work as
 * on audio handles (the thresholds also for DeepFilterNet2).  DeepFilterNet v1: DFB_ERR_UNSUPPORTED.
 *   d_spec f32[B][n_frames][F][2]: complex64 rows as dfb_analysis returns them (F = fft / 2 + 1 of the state, 481).
 *   Outputs, [B][n_frames] rows (flush: [B][latency]); every pointer except d_gains may be NULL:
 *     d_gains f32[..][nb_erb]            the ERB mask (dfb_apply's `m` layout)
 *     d_coefs f32[..][nb_df][2 * order]  the network's c[t][k][o * 2 + re/im] (dfb_apply's `coefs` layout; the [nb_df][order]
 *                                        complex layout tract.rs's df() reads -- not [order][nb_df][2] as capi.rs's comment says)
 *     d_lsnr  f32[..]                    dB
 *     d_stage i8 [..]                    see below
 * Alignment: row j of a call that starts at input frame k carries frame k + j - latency, latency = conv_lookahead (2 for
 * DeepFilterNet3 and DeepFilterNet2, 0 for DeepFilterNet3_ll; dfb_stream_latency_frames returns it).  As df_process_frame
 * (see the LSNR note above); for DeepFilterNet2 this is NOT the audio handle's latency: the outputs do not wait for the deep
 * filter's own look-ahead.  Flush returns the last `latency` frames, computed with zero look-ahead features.
 * Rows that carry no frame (the first `latency` rows of a handle or of a session, free slots, a closing slot past its tail):
 * NaN gains, coefs and LSNR, stage -1.
 * Stages (tract.rs:658-672 apply_stages on the frame's LSNR, the link group's channel 0's for a slot group; every frame is
 * stage 1 while gating is off):
 *   0  lsnr < min_db_thresh        gains 0, coefs 0
 *   3  else lsnr > max_db_erb      gains 1 (unprocessed), coefs 0
 *   2  else lsnr > max_db_df       network gains, coefs 0
 *   1  otherwise                   network gains and coefs
 * On a mask_only model stage 1 is stage 2.  Where the Rust runtime returns NULL for a skipped output, the values here are
 * defined, so a caller can apply every row as it comes.  Linked channels: each member's gains are the group's reduced mask
 * (max / mean as dfb_enhance_ragged's link groups); coefs and LSNR stay per channel.  In DFB_GATING_RUNTIME
 * (dfb_stream_set_gating_mode) the network gains of stages 1 / 2 and the coefs of stage 1 come from decoders that ran
 * only on such frames, as df_process_frame_raw's do; this holds for DeepFilterNet2 and DeepFilterNet2_ll too. */
int dfb_stream_create_spec(dfb_stream **out, dfb_model *m, dfb_state *st, int64_t B);
int dfb_stream_process_spec(dfb_stream *s, const float *d_spec, int64_t n_frames, float *d_gains, float *d_coefs,
                            float *d_lsnr, int8_t *d_stage, void *stream);
/* end of stream: closes every open slot, as dfb_stream_flush */
int dfb_stream_flush_spec(dfb_stream *s, float *d_gains, float *d_coefs, float *d_lsnr, int8_t *d_stage, void *stream);
/* host pointers, synchronous; h_spec == NULL flushes into [B][latency] rows (h_gains may be NULL when latency is 0) */
int dfb_stream_process_spec_host(dfb_stream *s, const float *h_spec, int64_t n_frames, float *h_gains, float *h_coefs,
                                 float *h_lsnr, int8_t *h_stage);

/* Chunk pipeline of dfb_enhance (device_chunks) / dfb_enhance_host (host_chunks): a signal of >= 64 * chunks frames is cut
 * into at least that many time chunks; lanes = 2 overlaps the encoder phase of chunk c + 1 with the decoder phase (the
 * recurrences) of chunk c on a second set of streams and a second workspace, lanes = 1 runs them back to back.
 * Defaults 0 (auto: 3 chunks up to 8 streams, 2 up to 256, else 1) / 4 / 2.  The output
 * does not depend on these settings beyond fp32 reduction order (tests compare them). */
int dfb_model_set_chunking(dfb_model *m, int device_chunks, int host_chunks, int lanes);
/* init_df(post_filter=..., mask_only=...) (DeepFilterNet/df/enhance.py:101-187).  post_filter: Valin's post filter -- for
 * DeepFilterNet3 on the enhanced spectrum with beta = pf_beta (deepfilternet3.py:448-454), for DeepFilterNet2 on the ERB
 * gains with beta = 0.02 (Mask.pf, modules.py:234-245).  mask_only: the model as built with run_df = False
 * (checkpoint.py:32): no deep-filter stage, every bin takes the ERB gain. */
int dfb_model_set_options(dfb_model *m, int post_filter, float pf_beta, int mask_only);
/* Cap (bytes) of the per-call device workspace of dfb_enhance: the batch is processed in time chunks (and, for very
 * large batches, stream groups) that fit below it (default 40 GB, or DFB_MAX_WORKSPACE_MB in the environment at
 * dfb_model_create). */
int dfb_model_set_max_workspace(dfb_model *m, int64_t bytes);
/* Debug aid: steps > 0 with h_out == NULL arms clock64() phase stamps ([steps][8]) for the following
 * GRU launches of at most `steps` time steps (longer ones are not stamped); a second call with h_out != NULL copies
 * min(steps, armed steps) rows of the stamps (of the last stamped launch) and disarms. */
int dfb_debug_gru_timing(dfb_model *m, int steps, long long *h_out);
/* Debug aid: one launch of the tensor-core GRU recurrence on device pointers, on `stream` (NULL = default).  For steps
 * t = 0 .. T-1 (frame t0 + t of buffers holding Ts frames per stream): xproj [B][Ts][3H] (W_ih x + b_ih), whh [3H][H],
 * bhh [3H]; hout [B][Ts][H] = h + res and / or the BF16 hi / lo planes of h (planes_res = 0) or of h + res (1); res may
 * be NULL.  h0 [B][H] carried state (NULL: zeros), hT [B][H] final state (may alias h0, may be NULL).  first (NULL or
 * [B]): stream b's first frame is first[b] - w0 of the window; h stays 0 before it.  ns = 0, xg = -1: the instance the
 * library picks for B; otherwise the instance of ns streams per cluster and exchange xg (0: DSMEM copies, 1: L2 multicast):
 * H = 256 with (16|32, 0|1) or (48, 1), H = 512 with (16, 0|1); others return DFB_ERR_UNSUPPORTED. */
int dfb_debug_gru_tc(const float *xproj, const float *whh, const float *bhh, const float *res, float *hout, void *hout_hi,
                     void *hout_lo, int planes_res, const float *h0, float *hT, const int64_t *first, int64_t w0, int t0,
                     int Ts, int B, int T, int H, int ns, int xg, void *stream);
/* Debug aid: dfb_debug_gru_tc with run flags run [B][Ts] (bytes, not NULL), the recurrence of the runtime gating mode:
 * at a step whose flag is 0 the state keeps its value, is carried on and is written out (plus res) as that step's output. */
int dfb_debug_gru_tc_hold(const float *xproj, const float *whh, const float *bhh, const float *res, float *hout, void *hout_hi,
                          void *hout_lo, int planes_res, const float *h0, float *hT, const int64_t *first, int64_t w0,
                          const unsigned char *run, int t0, int Ts, int B, int T, int H, int ns, int xg, void *stream);
/* Debug aid: one launch of the BF16x3 projection GEMM on device pointers: y [M][N] (pitch ldy) = x w^T + bias with x
 * given as BF16 hi / lo planes [M][K] (pitch ldx) and w as BF16 hi / lo planes [N][K]; bias may be NULL. */
int dfb_debug_gemm_bf16x3(const void *x_hi, const void *x_lo, int64_t ldx, const void *w_hi, const void *w_lo,
                          const float *bias, float *y, int64_t ldy, int64_t M, int N, int K, void *stream);
/* Debug aid: one launch of the tensor-core grouped linear on device pointers, on `stream` (a cudaStream_t, NULL = default):
 * y / (y_hi, y_lo) [M][G*Hg] = act(GL(x)) * oscale + ooffset + res, x given as BF16 hi / lo planes [M][G*Ig] (pitch ldx)
 * and w_img the weight image of weights.py gl_bx_image.  y or the planes may be NULL; res may alias y.  act: 0 none,
 * 1 ReLU, 2 tanh. */
int dfb_debug_gl_bx(const void *x_hi, const void *x_lo, int64_t ldx, const float *w_img, const float *res, int64_t ldr,
                    float *y, int64_t ldy, void *y_hi, void *y_lo, int64_t ldp, int64_t M, int G, int Ig, int Hg, int act,
                    float oscale, float ooffset, void *stream);
/* Debug aid: one launch of the tensor-core DF pathway conv on device pointers, on `stream` (NULL = default):
 * coefs [B][T][Fd][2 order] = relu(w2^T (grouped (2) temporal conv of c0 [B][T][Fd][64] with kt taps) + bias), w_sw the
 * operand image of weights.py (df_dec.df_convp.w_sw), w2 [2 order][2 order] (in, out), bias [2 order].  Frames before
 * frame 0 of a stream, and (first != NULL, [B]) before frame first[b] - w0, read as zeros.  order 5 with kt 1 to 5 are
 * built; others return DFB_ERR_UNSUPPORTED. */
int dfb_debug_df_convp_tc(const float *c0, const float *w_sw, const float *w2, const float *bias, float *coefs, int B, int T,
                          int Fd, int order, int kt, const int64_t *first, int64_t w0, void *stream);
/* Debug aids for the spectral handle's input kernel.  dfb_debug_analysis_erb: the time-chunked analysis kernel on audio
 * f32[C][T] with its ERB epilogue: spec c64[C][T / hop][F], erb_db f32[C][T / hop][E] (dB, before normalisation).
 * dfb_debug_spec_ingest: k_spec_ingest over n frames of nb live rows, row b reading caller row h_src[b] of spec
 * c64[..][n][F] and zeros from frame h_len[b] on (h_src / h_len HOST arrays of nb entries, or NULL: row b, n frames):
 * erb_db f32[nb][n][E] and the first nb_df bins c64[nb][n][nb_df].  fft 960 / hop 480 states only. */
int dfb_debug_analysis_erb(dfb_state *st, const float *d_audio, int64_t C, int64_t T, float *d_spec, float *d_erb_db,
                           void *stream);
int dfb_debug_spec_ingest(dfb_state *st, const float *d_spec, int64_t n, const int64_t *h_src, const int64_t *h_len, int64_t nb,
                          int nb_df, float *d_erb_db, float *d_bins, void *stream);
/* Debug aid for parity tests: copies the named activation of the LAST forward pass on this handle
 * (e0,e1,e2,e3,c0,c1,emb_in,emb,dec_emb,d3,d2,d1,dfc) to the host; returns the element count
 * (or a negative dfb_status).  Valid until the next call on the handle.
 * A window run in runtime gating mode (dfb_model_set_gating_mode) adds, for its B rows of T frames (M = B T):
 *   lsnr [B][T], m [B][T][nb_erb], coefs [B][T][nb_df][2 df_order]: the window's outputs;
 *   gate_erb_run, gate_df_run: run flags, one byte per frame [B][T], fetched as ceil(M / 4) floats;
 *   gate_erb_src, gate_df_pos: int32 [B][T] (the last ERB run frame, -1: none; DF run frames before t);
 *   gate_df_n: int32 [B];  gate_erb_first: int64 [B] (2 B floats), the first frame the kt = 2 layers read;
 *   gate_P [B][Tp][nb_df * 64], gate_Q [B][Tp][nb_df][2 df_order]: the compacted DF pathway rows and their conv, with
 *   Tp = df_pathway_kt - 1 + new frames;
 *   erb_gru_hi, erb_gru_lo: the ERB recurrence's output [B][T][emb_hidden] as BF16 planes (M emb_hidden / 2 floats each). */
int64_t dfb_model_debug_fetch(dfb_model *m, const char *name, float *h_out, int64_t max_numel);
/* bytes of device workspace the model handle currently owns (grow-only arena) */
int64_t dfb_model_workspace_bytes(const dfb_model *m);

/* ------------------------------------------------------------------ metrics -------------------
 * Speech-quality metrics of a ragged batch on the device (DESIGN.md section 5j), each equal to the reference function
 * applied to one entry alone:
 *   DFB_METRIC_SISDR  DeepFilterNet/df/evaluation_utils.py si_sdr_speechmetrics(clean, degraded) at the input rate
 *                     (fp64 sums, float32 eps);
 *   DFB_METRIC_STOI   df/stoi.py stoi(clean[None], degraded[None], sr)[0]: io.resample to 10 kHz (sinc_fast), silent
 *                     frames removed, 15 third-octave bands, 30-frame segments; NaN when fewer than 512 samples remain;
 *   DFB_METRIC_SSNR   df/sepm.py SNRseg(c16, d16, 16000) after io.resample to 16 kHz (sinc_fast); NaN when no frame is left;
 *   DFB_METRIC_LLR    df/sepm.py llr(c16, d16, 16000): the log-likelihood ratio of order-16 LPC models of the T =
 *                     (L16 - 480) / 120 frames of 480 samples at hop 120, averaged over the round(0.95 T) smallest;
 *   DFB_METRIC_WSS    df/sepm.py wss(c16, d16, 16000): Klatt's weighted spectral slope over 25 critical bands on the same
 *                     frames, averaged the same way.  LLR and WSS are NaN when T = 0.
 * With PESQ-WB (not provided) they make df/sepm.py's composite measure: CSIG, CBAK and COVL are Hu & Loizou's (IEEE TASLP
 * 16(1), 2008) linear regressions on PESQ, LLR, WSS and SSNR.
 *   DFB_METRIC_PYSTOI pystoi.stoi(x10, y10, 10000) (pystoi 0.4.1), which df/evaluation_utils.py stoi reports, on the
 *                     same 10 kHz rows as STOI: F = ceil((L10 - 256) / 128) frames of 256 samples at hop 128, those
 *                     within 40 dB of the loudest kept and overlap-added (K of them), K - 1 STFT frames, J = K - 30
 *                     segments of 30 frames, all in fp64 (DESIGN.md section 5n);
 *   DFB_METRIC_ESTOI  pystoi.stoi(x10, y10, 10000, extended=True) on the same segments, without pystoi's eps-scaled
 *                     random noise: a centred row or column of norm 0 normalises to 0.
 *                     Both are NaN when L10 <= 256 (no frame: pystoi raises) and 1e-5 when K - 1 < 30 (pystoi's value).
 * Bits 8 and 64 are not metrics.  DFB_METRIC_STOI is df/stoi.py's STOI, which removes silence and frames differently from pystoi's. */
enum {
    DFB_METRIC_SISDR = 1, DFB_METRIC_STOI = 2, DFB_METRIC_SSNR = 4, DFB_METRIC_LLR = 16, DFB_METRIC_WSS = 32,
    DFB_METRIC_PYSTOI = 128, DFB_METRIC_ESTOI = 256
};
typedef struct dfb_metrics dfb_metrics;
/* A metrics handle on `device` for inputs at `sr` Hz: taps10 / taps16 [nw][2 width + og] (HOST arrays) are
 * io.resample_kernel(sr, 10000) / (sr, 16000) with the sinc_fast parameters, og / nw the gcd-reduced rates (DFB_ERR_INVALID
 * otherwise); NULL when sr is that rate.  DFB_ERR_UNSUPPORTED when the two tables hold more than 2^18 floats together (as
 * dfb_model_add_rate).  The handle owns the tables, a stream and a workspace that grows when a call needs more. */
int dfb_metrics_create(dfb_metrics **out, int device, int sr, const float *taps10, int og10, int nw10, int width10,
                       const float *taps16, int og16, int nw16, int width16);
void dfb_metrics_free(dfb_metrics *h);
/* One call scores B <= 32767 entries: entry b is clean_lengths[b] samples of clean at d_clean + offsets[b] and as many of
 * degraded at d_degraded + offsets[b] (offsets / lengths HOST arrays, in_numel bounding both buffers).  d_out [n][B] fp32
 * gets one row per bit of `metrics`, in the order SI-SDR, STOI, SSNR, LLR, WSS, PYSTOI, ESTOI.  DFB_ERR_INVALID for a length <= 0, different clean
 * and degraded lengths, an entry outside in_numel, no metric or an unknown metric bit.  Asynchronous on `stream`; the
 * handle's workspace serves one call at a time. */
int dfb_metrics_compute(dfb_metrics *h, const float *d_clean, const float *d_degraded, int64_t in_numel, const int64_t *offsets,
                        const int64_t *clean_lengths, const int64_t *degraded_lengths, int64_t B, int metrics, float *d_out,
                        void *stream);
int dfb_metrics_compute_host(dfb_metrics *h, const float *h_clean, const float *h_degraded, int64_t in_numel,
                             const int64_t *offsets, const int64_t *clean_lengths, const int64_t *degraded_lengths, int64_t B,
                             int metrics, float *h_out);
/* bytes of device workspace the metrics handle owns */
int64_t dfb_metrics_workspace_bytes(const dfb_metrics *h);
/* Debug aid: the STOI of a dfb_metrics_host call, then h_counts [B][3] = each entry's kept frames, its length after silence
 * removal and its STFT frames (0 when that length is below 512). */
int dfb_debug_metrics_counts(dfb_metrics *h, const float *h_clean, const float *h_degraded, int64_t in_numel,
                             const int64_t *offsets, const int64_t *lengths, int64_t B, int64_t *h_counts);
/* Debug aid: the LLR and WSS of a dfb_metrics_host call, then h_frames [B] = each entry's frame count T and h_llr / h_wss
 * = every entry's per-frame distortions before the 0.95 trim (fp64), entries back to back.  DFB_ERR_INVALID when the
 * frames of all entries exceed `capacity` doubles. */
int dfb_debug_metrics_frames(dfb_metrics *h, const float *h_clean, const float *h_degraded, int64_t in_numel,
                             const int64_t *offsets, const int64_t *lengths, int64_t B, int64_t *h_frames, double *h_llr,
                             double *h_wss, int64_t capacity);
/* Debug aid: the PYSTOI and ESTOI of a dfb_metrics_host call, then h_counts [B][5] = each entry's pystoi frames F, kept
 * frames K, silence-free length, STFT frames nf and segments J (all 0 when F = 0).  When h_bands is not NULL it gets every
 * entry's band magnitudes (fp64), entries back to back, each [2][15][nf] (clean, then degraded); DFB_ERR_INVALID when
 * they exceed `capacity` doubles. */
int dfb_debug_metrics_pystoi(dfb_metrics *h, const float *h_clean, const float *h_degraded, int64_t in_numel,
                             const int64_t *offsets, const int64_t *lengths, int64_t B, int64_t *h_counts, double *h_bands,
                             int64_t capacity);

#ifdef __cplusplus
}
#endif
#endif /* DFB200_H */
