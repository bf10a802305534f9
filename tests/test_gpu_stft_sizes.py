"""GPU: the STFT, ISTFT and feature extraction of DSP states at fft / hop sizes other than 960 / 480 (the generic real FFT
of dfb_fft_generic.cuh and the k_analysis_gen / k_synthesis_gen kernels), element by element against float64.

Bounds follow tests/dsp_ref64.py (|fp32 result - float64 reference| <= bound per element), with an FFT bound for the
generic stage structure (fft_rounds: roundings along one input -> output path of the plan, the same table as
tests/host/fft_generic_host_test.cu) and an ISTFT for every overlap, not only N = 2 H.  Inputs come from seeds only."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import dsp_ref64 as R
import libdf_oracle as LO
from tests_common import synth_audio

from deepfilternet_b200 import DfNet, _lib, libdf
from deepfilternet_b200._lib import DfbError
from deepfilternet_b200.config import ModelConfig
from deepfilternet_b200.enhance import df_features
from deepfilternet_b200.features import fft_features
from deepfilternet_b200.weights import random_state_dict

U = R.U
ALPHA = 0.99
SIZES = [(24000, 96, 24), (16000, 320, 160), (16000, 512, 128), (48000, 512, 256), (48000, 960, 240), (48000, 1024, 512),
         (48000, 2048, 512), (48000, 8192, 2048), (8000, 97, 48), (48000, 2018, 1009)]


# ------------------------------------------------------------------ float64 references ----
def fft_rounds(N):
    """Roundings along one input -> output path of the generic real FFT of length N (gen_fft_plan's factorisation of
    M = N / 2 or N: fours, twos, threes, fives, sevens, then the other primes): per stage 6 (the rounded twiddle and
    its complex product, with slack) plus the butterfly's depth; a direct length-p DFT adds p + 1; the split / merge
    step of even N 4 more."""
    M = N // 2 if N % 2 == 0 else N
    rad, m = [], M
    for p in (4, 2, 3, 5, 7):
        while m % p == 0:
            rad.append(p)
            m //= p
    p = 11
    while m > 1:
        while m % p == 0:
            rad.append(p)
            m //= p
        p += 2
    return (4 if N % 2 == 0 else 0) + sum(6 + {2: 1, 4: 2, 3: 4, 5: 6, 7: 8}.get(r, r + 1) for r in rad)


def stft64(x, window, hop, mem=None):
    """frame_analysis over a whole signal (lib.rs:356-394): frame t = window x samples [t hop - (N - hop), t hop + hop),
    the N - hop samples before sample 0 from `mem` [C, N - hop] (zeros when None).  -> (X [C, Tf, N // 2 + 1], bound)."""
    x = np.asarray(x, np.float64)
    w = np.asarray(window, np.float64)
    N = len(w)
    C, T = x.shape
    Tf = T // hop
    m0 = np.zeros((C, N - hop)) if mem is None else np.asarray(mem, np.float64)
    xp = np.concatenate([m0, x[:, :Tf * hop]], 1)
    frames = np.lib.stride_tricks.sliding_window_view(xp, N, axis=1)[:, ::hop][:, :Tf] * w
    wn = R.wnorm_f32(N, hop)
    X = np.fft.rfft(frames, axis=-1) * wn
    bound = (wn * R.gamma(fft_rounds(N) + 1) * np.abs(frames).sum(-1))[..., None] + U * np.abs(X)
    return X, np.broadcast_to(bound, X.shape).copy()


def istft64(X, window, hop):
    """frame_synthesis (lib.rs:396-427) from zero memory, any overlap: out[t hop + i] = sum over the frames t' that
    cover the sample of w[j] x_t'[j], j = t hop + i - t' hop (imaginary parts of DC and, for even N, Nyquist ignored).
    X [C, Tf, F] -> ([C, Tf hop], bound)."""
    X = np.array(X, np.complex128)
    w = np.asarray(window, np.float64)
    N = len(w)
    C, Tf, F = X.shape
    X[..., 0] = X[..., 0].real
    if N % 2 == 0:
        X[..., -1] = X[..., -1].real
    yw = np.fft.irfft(X, n=N, axis=-1) * N * w
    herm = np.full(F, 2.0)
    herm[0] = 1.0
    if N % 2 == 0:
        herm[-1] = 1.0
    by = (R.gamma(fft_rounds(N) + 1) * (np.abs(X) @ herm))[..., None] * w + U * np.abs(yw)
    out, bout, asum = (np.zeros((C, Tf * hop + N)) for _ in range(3))
    for t in range(Tf):
        out[:, t * hop:t * hop + N] += yw[:, t]
        bout[:, t * hop:t * hop + N] += by[:, t]
        asum[:, t * hop:t * hop + N] += np.abs(yw[:, t])
    bout += R.gamma(math.ceil(N / hop)) * asum
    return out[:, :Tf * hop], bout[:, :Tf * hop]


# ------------------------------------------------------------------ helpers ----
def frames_per_cta(N):
    """Frames per CTA of the generic kernels (dfb_dsp.cu gen_frames)."""
    M = N // 2 if N % 2 == 0 else N
    return max(1, min(32, 2048 // M))


def chunk_of(N, H):
    """Frames per CTA of the generic synthesis kernel (launch_synthesis_gen)."""
    G, K = frames_per_cta(N), -(-(N - H) // H)
    return G * max(2, -(-8 * K // G))


def frame_counts(N, H):
    G, ch = frames_per_cta(N), chunk_of(N, H)
    return sorted({1, G + 1, max(1, ch - 1), ch + 1, 1000})


def assert_within(name, got, ref, bound, k=1.0):
    r = R.err_ratio(got, ref, bound)
    print(f"err/bound {name}: {r:.3g}")
    assert r <= k, (name, r)


def signal(C, T, seed, sr):
    return np.ascontiguousarray(synth_audio(C, T, seed=seed, sr=sr).numpy())


def complex_of(t):
    return torch.view_as_complex(t.contiguous()).cpu().numpy().astype(np.complex128)


_STATES = {}


def state(sr, N, H):
    if (sr, N, H) not in _STATES:
        _STATES[(sr, N, H)] = libdf.DF(sr, N, H, 32, 1)
    return _STATES[(sr, N, H)]


CASES = [(s, tf) for s in SIZES for tf in frame_counts(s[1], s[2])]


# ------------------------------------------------------------------ 1. element-wise bounds ----
@pytest.mark.parametrize("size,Tf", CASES, ids=[f"{s[1]}-{s[2]}-Tf{tf}" for s, tf in CASES])
def test_stft_istft_features_against_ref64(size, Tf):
    """DF.analysis, DF.synthesis, df_features and fft_features (spectrum, ERB features, DF features) at every size and at
    frame counts 1, around the analysis CTA tile and the synthesis chunk, and many; the signal length is not a multiple
    of the hop.  K = 1."""
    sr, N, H = size
    st = state(sr, N, H)
    F = N // 2 + 1
    T = Tf * H + (37 * Tf + 11) % H
    x = signal(2, T, seed=Tf + N, sr=sr)
    w = st.fft_window()
    X, bX = stft64(x, w, H)
    assert_within("analysis", st.analysis(x), X, bX)
    # synthesis of a random spectrum with non-zero imaginary parts at DC / Nyquist (ignored)
    rng = np.random.default_rng(N + Tf)
    S = ((rng.standard_normal((2, Tf, F)) + 1j * rng.standard_normal((2, Tf, F))) * 0.01).astype(np.complex64)
    y, by = istft64(S, w, H)
    assert_within("synthesis", st.synthesis(S), y, by)
    nb_df = min(96, F)
    sp, fe, fs = df_features(torch.from_numpy(x), st, nb_df, alpha=ALPHA)
    assert_within("df_features spec", complex_of(sp[:, 0]), X, bX)
    db, bdb = R.erb_db(X, bX, st.erb_widths())
    ref_e, b_e = R.mean_norm(db, ALPHA, None, bdb)
    assert_within("df_features erb", fe[:, 0].numpy(), ref_e, b_e)
    ref_u, b_u = R.unit_norm(X[..., :nb_df], ALPHA, None, bX[..., :nb_df])
    assert_within("df_features unit", complex_of(fs[:, 0]), ref_u, b_u)
    out = fft_features(st, torch.from_numpy(x).cuda(), torch.from_numpy(x[::-1].copy()).cuda(), nb_spec=nb_df, norm_alpha=ALPHA)
    torch.cuda.synchronize()
    assert_within("fft_features noisy", complex_of(out["noisy"][:, 0]), X, bX)
    assert_within("fft_features erb", out["feat_erb"][:, 0].cpu().numpy(), ref_e, b_e)
    assert_within("fft_features unit", complex_of(out["feat_spec"][:, 0]), ref_u, b_u)
    Xs, bXs = stft64(x[::-1], w, H)
    assert_within("fft_features speech", complex_of(out["speech"][:, 0]), Xs, bXs)


def test_large_unit_norm_features():
    """df_features with every bin as a DF feature at fft 8192 (E + Fd = 4129 values per stream: the wide scan)."""
    sr, N, H = 48000, 8192, 2048
    st = state(sr, N, H)
    x = signal(2, 40 * H + 5, seed=3, sr=sr)
    X, bX = stft64(x, st.fft_window(), H)
    sp, fe, fs = df_features(torch.from_numpy(x), st, N // 2 + 1, alpha=ALPHA)
    ref_u, b_u = R.unit_norm(X, ALPHA, None, bX)
    assert_within("unit 4097", complex_of(fs[:, 0]), ref_u, b_u)
    db, bdb = R.erb_db(X, bX, st.erb_widths())
    ref_e, b_e = R.mean_norm(db, ALPHA, None, bdb)
    assert_within("erb", fe[:, 0].numpy(), ref_e, b_e)


# ------------------------------------------------------------------ 2. carried memories ----
CARRY = [(24000, 96, 24), (16000, 320, 160), (8000, 97, 48), (16000, 500, 200)]


@pytest.mark.parametrize("size", CARRY, ids=[f"{s[1]}-{s[2]}" for s in CARRY])
def test_carried_memories_match_oracle(size):
    """reset=False chains (two calls of three channels each, the second call shorter than N - H where N / H > 2) against
    the CPU oracle LO.DF, whose dfo_analysis / dfo_synthesis carry N - H samples like the reference's DFState; then a
    reset call.  Bound: the float64 bound of any frame of the calls (every frame's L1 norm is at most sum |w| max |x|),
    which is far below what a wrong sample of memory would move."""
    sr, N, H = size
    st, lo = libdf.DF(sr, N, H, 32, 1), LO.DF(sr, N, H, 32, 1)
    w = st.fft_window()
    wn = R.wnorm_f32(N, H)
    for T, seed, reset in ((5 * H + 7, 1, False), (H + 3, 2, False), (3 * H, 3, False), (4 * H + 1, 4, True)):
        x = signal(3, T, seed=seed * 100 + N, sr=sr)
        got, ref = st.analysis(x, reset=reset), lo.analysis(x, reset=reset)
        bound = wn * R.gamma(fft_rounds(N) + 1) * np.abs(w).sum() * np.abs(x).max() + 2 * U * np.abs(ref)
        assert_within(f"analysis T={T} reset={reset}", got, ref.astype(np.complex128), bound)
    rng = np.random.default_rng(N)
    K = math.ceil(N / H)
    for Tf, reset in ((5, False), (1, False), (2, False), (3, True)):
        S = ((rng.standard_normal((3, Tf, N // 2 + 1)) + 1j * rng.standard_normal((3, Tf, N // 2 + 1))) * 0.01).astype(np.complex64)
        got, ref = st.synthesis(S, reset=reset), lo.synthesis(S, reset=reset)
        l1 = 2 * np.abs(S).sum(-1).max()
        bound = K * (R.gamma(fft_rounds(N) + 1) * l1 + 2 * U * np.abs(ref).max()) + R.gamma(K + 1) * K * np.abs(ref).max()
        assert_within(f"synthesis Tf={Tf} reset={reset}", got, ref.astype(np.float64), np.full(ref.shape, bound))


# ------------------------------------------------------------------ 3. the reference's STFT test ----
def test_reference_stft_test_and_round_trip():
    """test_analysis_synthesis_stft (DeepFilterNet/tests/test_dflib.py) at sr 24000, fft 96, hop 24: the analysis is
    torch.stft(center=False, window=fft_window()) times wnorm after N - H zeros of left padding; and at every size where
    2 H divides N, synthesis(analysis(x)) is x delayed by N - H to fp32 accuracy."""
    sr, N, H = 24000, 96, 24
    st = state(sr, N, H)
    x = signal(1, 2400 * 5 + 13, seed=9, sr=sr)
    w = st.fft_window()
    xp = torch.from_numpy(np.concatenate([np.zeros((1, N - H)), x.astype(np.float64)], 1))
    ref = torch.stft(xp, n_fft=N, hop_length=H, window=torch.from_numpy(w.astype(np.float64)), center=False,
                     return_complex=True).transpose(1, 2).numpy() * R.wnorm_f32(N, H)
    Tf = x.shape[1] // H
    _, bX = stft64(x, w, H)
    assert_within("torch.stft", st.analysis(x), ref[:, :Tf], bX)
    for sr, N, H in SIZES:
        if N % (2 * H):
            continue
        st = state(sr, N, H)
        x = signal(2, 50 * H, seed=N, sr=sr)
        y = st.synthesis(st.analysis(x))
        err = np.abs(y[:, N - H:] - x[:, :x.shape[1] - (N - H)]).max()
        print(f"round trip {N}/{H}: max err {err:.3g}")
        assert err <= 1e-5 * np.abs(x).max(), (N, H, err)


# ------------------------------------------------------------------ 4. large spectra ----
@pytest.mark.parametrize("F", [1025, 4097])
def test_norms_of_large_spectra_match_oracle(F):
    """libdf.unit_norm / erb_norm over 1025 and 4097 values per frame (more than one block of the scan), with and
    without a state: the reference loop's bits (ref_bits)."""
    rng = np.random.default_rng(F)
    spec = ((rng.standard_normal((2, 150, F)) + 1j * rng.standard_normal((2, 150, F))) * 0.1).astype(np.complex64)
    state_u = (rng.random((2, F)) * 1e-3).astype(np.float32)
    np.testing.assert_array_equal(libdf.unit_norm(spec, ALPHA), LO.unit_norm(spec, ALPHA))
    np.testing.assert_array_equal(libdf.unit_norm(spec, ALPHA, state_u), LO.unit_norm(spec, ALPHA, state_u))
    erb = (rng.standard_normal((2, 150, F)) * 20 - 60).astype(np.float32)
    state_e = (rng.standard_normal((2, F)) * 10 - 70).astype(np.float32)
    np.testing.assert_array_equal(libdf.erb_norm(erb, ALPHA), LO.erb_norm(erb, ALPHA))
    np.testing.assert_array_equal(libdf.erb_norm(erb, ALPHA, state_e), LO.erb_norm(erb, ALPHA, state_e))


# ------------------------------------------------------------------ 5. refusals ----
def test_refusals():
    """fft_size above 8192 is refused with DFB_ERR_UNSUPPORTED; the model path refuses a DSP state that is not 960 / 480
    at every C entry point (and in Python before it gets there)."""
    with pytest.raises(DfbError) as e:
        libdf.DF(48000, 16384, 4096)
    assert e.value.code == _lib.DFB_ERR_UNSUPPORTED and "8192" in str(e.value)
    with pytest.raises(NotImplementedError):
        DfNet(ModelConfig(model="deepfilternet3", fft_size=320, hop_size=160, sr=16000), {})
    cfg = ModelConfig(model="deepfilternet3", conv_ch=64, conv_lookahead=2, df_lookahead=2, emb_num_layers=3, df_num_layers=2,
                      lin_groups=16, enc_lin_groups=32, df_gru_skip="groupedlinear", df_pathway_kernel_size_t=5)
    model = DfNet(cfg, random_state_dict(cfg, seed=0))
    st = state(16000, 320, 160)
    L = _lib.lib()
    buf = torch.zeros(1 << 20, device="cuda")
    hbuf = np.zeros(1 << 16, np.float32)
    d, h = buf.data_ptr(), hbuf.ctypes.data
    s = torch.cuda.current_stream().cuda_stream
    offs = np.zeros(1, np.int64)
    lens = np.full(1, 1600, np.int64)
    op, lp = offs.ctypes.data, lens.ctypes.data
    handle = C.c_void_p()
    calls = {
        "dfb_enhance": lambda: L.dfb_enhance(model.handle, st.handle, d, 1, 1600, 1, C.c_float(0.0), d, s),
        "dfb_enhance_host": lambda: L.dfb_enhance_host(model.handle, st.handle, h, 1, 1600, 1, C.c_float(0.0), h),
        "dfb_enhance_ragged_host": lambda: L.dfb_enhance_ragged_host(model.handle, st.handle, h, 1600, op, lp, 1, 1, C.c_float(0.0),
                                                                     h, 1600, op, None, 0, 0, None, None, 0, None, 0, None),
        "dfb_apply": lambda: L.dfb_apply(model.handle, st.handle, d, d, d, 1, 4, d, s),
        "dfb_model_forward_full": lambda: L.dfb_model_forward_full(model.handle, st.handle, d, d, d, 1, 4, d, d, d, d, None, s),
        "dfb_stream_create": lambda: L.dfb_stream_create(C.byref(handle), model.handle, st.handle, 1, C.c_float(0.0)),
    }
    for name, call in calls.items():
        rc = call()
        assert rc == _lib.DFB_ERR_UNSUPPORTED, (name, rc, L.dfb_last_error())
        assert b"960" in L.dfb_last_error(), name
    torch.cuda.synchronize()
