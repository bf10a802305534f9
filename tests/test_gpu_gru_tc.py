"""GPU: the tensor-core GRU recurrence (k_gru_tc) and its input projection (k_gemm_bf16x3) on their own, through
dfb_debug_gru_tc / dfb_debug_gemm_bf16x3, against torch.nn.GRU in float64 on the CPU.

The recurrence-only tests feed the kernel's input `xproj` (= W_ih x + b_ih) to a float64 torch.nn.GRU whose W_ih is the
identity I(3H) and whose b_ih is 0, so the reference is torch's own cell.  Weights are torch's default init U(+-1/sqrt(H))
or the W_hh / b_hh that weights.py packs from random_state_dict of the DeepFilterNet3 (H = 256) and DeepFilterNet3_ll
(H = 512) configurations.

Element-wise accuracy, teacher-forced step check.  Step t is checked on its own: the kernel's fp32 h[t-1] goes through one
float64 cell step and the result is compared with the kernel's h[t].  For unit j, with P_g = sum_k |W_hh[g,j,k]| |h_k| +
|b_hh[g,j]| the product part of gate g (r, z, n) and X_g = |xproj[g,j]|, the kernel's pre-activations carry
  e_g <= c1 (P_g + X_g):  W_hh and h each carried to ~2^-16 relative by their BF16 hi + lo split, the dropped lo * lo term
      (~2^-16), the fp32 accumulation of the K-partial sums over K = H and the fp32 additions of x, W_hh h and b.
Through the gates (sigma' <= 1/4, tanh' <= 1, |a_n + b_n| <= P_n, |h_prev - n| <= 2):
  |dr| <= c1 (P_r + X_r) / 4,   |dz| <= c1 (P_z + X_z) / 4,
  |dn| <= |dr| P_n + c1 (P_n + X_n),   |dh| <= (1 - z) |dn| + 2 |dz|,
so |h_kernel - h_ref| <= c1 S + c2 with S = (P_n + X_n) + (P_r + X_r) P_n / 4 + (P_z + X_z) / 2, and c2 the absolute error
of the MUFU __expf / __fdividef gates and of the final fp32 combine.  Because every step restarts from the kernel's own
state, the bound does not grow with T.  C1 / C2 are set from an H100 measurement (see the constants); each check prints
its measured max of |err| / bound.  A kernel that drops the lo * hi term of the MMA errs by ~2^-9 of the products and fails.

Free-running trajectories over the full sequence (T = 3002 at H = 256, 1002 at H = 512, and a long-memory case with the
z-gate bias raised by 3) are compared with a max-abs bound measured on an H100.

Bit-exact invariants that follow from the code (mma.sync N columns are independent, the K-partial sums are added in the
same order for a given H, bf16_split of a carried fp32 h equals the in-kernel split): a stream's rows do not depend on
its batch position, on B or on the instance; a launch split in two with the state carried through h0 / hT (aliased) equals
one launch; a slot's rows before its first frame are 0 and from it on equal a fresh launch; the outputs are h + res, the
round-to-nearest-even BF16 hi / lo split of h or of h + res, and hT the residual-free last state; nothing outside the
launch's frames and rows is written; concurrent launches on two CUDA streams equal serial ones."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

INST = {256: [(16, 0), (16, 1), (32, 0), (32, 1), (48, 1)], 512: [(16, 0), (16, 1)]}   # (ns, xg) built per H
# Teacher-forced bound |err| <= C1 * S + C2 (module docstring).  Measured on an H100 80GB HBM3 (700 W): max |err| / S
# 3.7e-7 over all cases, max |err| 4.7e-6 (saturated gates); the bound is about 4x the worst case.
C1, C2 = 1.5e-6, 5e-7
SENT = 1234.5          # fp32 sentinel of frames / rows a launch must not write
SENT16 = 0x5A5A        # BF16 plane sentinel


def lib():
    from deepfilternet_b200 import _lib
    return _lib.lib()


def ptr(t):
    return None if t is None else t.data_ptr()


def gru_call(xp, whh, bhh, B, T, H, res=None, hout=None, hi=None, lo=None, planes_res=0, h0=None, hT=None, first=None,
             w0=0, t0=0, Ts=None, ns=0, xg=-1, stream=None):
    """one dfb_debug_gru_tc call on device tensors; returns the status"""
    st = (stream or torch.cuda.current_stream()).cuda_stream
    return lib().dfb_debug_gru_tc(ptr(xp), ptr(whh), ptr(bhh), ptr(res), ptr(hout), ptr(hi), ptr(lo), planes_res, ptr(h0),
                                  ptr(hT), ptr(first), w0, t0, T if Ts is None else Ts, B, T, H, ns, xg, st)


def gru_run(xp, whh, bhh, B, T, H, stream=None, sync=True, **kw):
    """fp32 output [B][Ts][H] (+ hT) of one launch; xp [B][Ts][3H] on the device"""
    Ts = kw.get("Ts") or T
    hout = torch.zeros((B, Ts, H), dtype=torch.float32, device="cuda")
    if stream is not None:
        torch.cuda.synchronize()   # inputs and the zero fill are complete before another stream reads / writes them
    rc = gru_call(xp, whh, bhh, B, T, H, hout=hout, stream=stream, **kw)
    assert rc == 0, (rc, lib().dfb_last_error())
    if sync:
        torch.cuda.synchronize()
    return hout


def default_weights(H, seed, z_bias=0.0):
    """torch.nn.GRU's default init U(+-1/sqrt(H)) of W_hh / b_hh (fp32, CPU)"""
    g = torch.Generator().manual_seed(seed)
    k = H ** -0.5
    whh = (torch.rand(3 * H, H, generator=g) * 2 - 1) * k
    bhh = (torch.rand(3 * H, generator=g) * 2 - 1) * k
    bhh[H:2 * H] += z_bias
    return whh.contiguous(), bhh.contiguous()


_MODEL_W = {}


def model_weights(model, name):
    """W_hh / b_hh that weights.py packs from random_state_dict of a shipped configuration"""
    if model not in _MODEL_W:
        import bench
        from deepfilternet_b200.weights import pack_state_dict, random_state_dict
        cfg = bench.model_config(model)
        _MODEL_W[model] = pack_state_dict(random_state_dict(cfg, seed=0), cfg)[0]
    w = _MODEL_W[model]
    return torch.from_numpy(w[name + ".w_hh"]).reshape(-1), torch.from_numpy(w[name + ".b_hh"])


def weights(src, H, seed=0):
    if src == "default":
        return default_weights(H, seed)
    model, name = {256: ("DeepFilterNet3", "enc.emb_gru.l0"), 512: ("DeepFilterNet3_ll", "df_dec.df_gru.l2")}[H]
    whh, bhh = model_weights(model, name)
    return whh.reshape(3 * H, H).contiguous(), bhh.contiguous()


def rand_x(B, T, H, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, T, 3 * H, generator=g) * scale).contiguous()


def ref_gru(whh, bhh, H, w_ih=None, b_ih=None):
    """float64 torch.nn.GRU; W_ih = I(3H), b_ih = 0 unless given"""
    in_dim = 3 * H if w_ih is None else w_ih.shape[1]
    g = torch.nn.GRU(in_dim, H, batch_first=True, dtype=torch.float64)
    with torch.no_grad():
        g.weight_ih_l0.copy_(torch.eye(3 * H, dtype=torch.float64) if w_ih is None else w_ih.double())
        g.bias_ih_l0.copy_(torch.zeros(3 * H, dtype=torch.float64) if b_ih is None else b_ih.double())
        g.weight_hh_l0.copy_(whh.double())
        g.bias_hh_l0.copy_(bhh.double())
    return g


def check_teacher_forced(xp, whh, bhh, h, h0=None, label=""):
    """every element of the kernel's h [B][T][H] (CPU) against one float64 cell step from its own h[t-1]; returns
    max |err| / bound"""
    B, T, H = h.shape
    prev = torch.cat([torch.zeros(B, 1, H) if h0 is None else h0.reshape(B, 1, H), h[:, :-1]], 1).double()
    with torch.no_grad():
        ref, _ = ref_gru(whh, bhh, H)(xp.double().reshape(B * T, 1, 3 * H), prev.reshape(1, B * T, H))
    ref = ref.reshape(B, T, H)
    P = torch.einsum("gjk,btk->gbtj", whh.double().abs().reshape(3, H, H), prev.abs()) + bhh.double().abs().reshape(3, 1, 1, H)
    X = xp.double().abs().reshape(B, T, 3, H).permute(2, 0, 1, 3)
    S = (P[2] + X[2]) + (P[0] + X[0]) * P[2] / 4 + (P[1] + X[1]) / 2
    err = (h.double() - ref).abs()
    bound = C1 * S + C2
    ratio = float((err / bound).max())
    print(f"teacher-forced {label}: max|err| {float(err.max()):.3e}  max err/S {float((err / S).max()):.3e}  "
          f"measured / bound {ratio:.3f}")
    assert torch.isfinite(h).all()
    bad = err > bound
    assert not bad.any(), (label, int(bad.sum()), float(err.max()), ratio)
    return ratio


# ------------------------------------------------------------------------------------------- accuracy -----------------

@pytest.mark.parametrize("H,T", [(256, 1), (256, 2), (256, 3), (256, 64), (256, 1002), (256, 3002),
                                 (512, 1), (512, 2), (512, 3), (512, 64), (512, 1002), (512, 3002)])
@pytest.mark.parametrize("src", ["default", "model"])
def test_teacher_forced(H, T, src):
    """every step of one launch from its own previous state, element by element; a non-zero h0 enters step 0"""
    B = 3 if T <= 64 else 2
    whh, bhh = weights(src, H, seed=H + T)
    xp = rand_x(B, T, H, seed=T)
    h0 = torch.rand(B, H, generator=torch.Generator().manual_seed(5)) * 2 - 1
    h = gru_run(xp.cuda(), whh.cuda(), bhh.cuda(), B, T, H, h0=h0.cuda()).cpu()
    check_teacher_forced(xp, whh, bhh, h, h0, f"H{H} T{T} {src}")


@pytest.mark.parametrize("H", [256, 512])
def test_teacher_forced_saturated(H):
    """pre-activations up to +-100: __expf overflows to inf inside the gates, the outputs stay finite and in the bound"""
    B, T = 3, 64
    whh, bhh = default_weights(H, seed=7)
    xp = rand_x(B, T, H, seed=8, scale=40.0).clamp(-100, 100)
    xp[:, ::4, : H] = 100.0       # r saturated open
    xp[:, 1::4, H: 2 * H] = -100.0   # z saturated shut: h = n
    xp[:, 2::4, 2 * H:] = 100.0   # n saturated at +1
    h = gru_run(xp.cuda(), whh.cuda(), bhh.cuda(), B, T, H).cpu()
    assert torch.isfinite(h).all() and float(h.abs().max()) <= 1.0
    check_teacher_forced(xp, whh, bhh, h, None, f"saturated H{H}")


# free-running max |h_kernel - h_float64| over the whole sequence: (H, T, z-gate bias) -> bound, about 4x what an H100
# 80GB HBM3 (700 W) measured: 2.7e-6, 3.1e-6 and 6.0e-7 (the saturated-open z gate carries h with little new rounding)
FREE = {(256, 3002, 0.0): 1e-5, (512, 1002, 0.0): 1.2e-5, (256, 3002, 3.0): 2.5e-6}


@pytest.mark.parametrize("H,T,zb", list(FREE), ids=lambda v: str(v))
def test_free_running(H, T, zb):
    """the kernel's own trajectory against the float64 GRU's over the full sequence (z bias +3: long memory, drift
    accumulates)"""
    B = 2
    whh, bhh = default_weights(H, seed=11, z_bias=zb)
    xp = rand_x(B, T, H, seed=12)
    h = gru_run(xp.cuda(), whh.cuda(), bhh.cuda(), B, T, H).cpu().double()
    with torch.no_grad():
        ref, _ = ref_gru(whh, bhh, H)(xp.double())
    err = float((h - ref).abs().max())
    print(f"free-running H{H} T{T} z+{zb}: max|err| {err:.3e}  bound {FREE[(H, T, zb)]:.1e}")
    assert err <= FREE[(H, T, zb)], err


# ------------------------------------------------------------------------------------------- bit-exact ----------------

def pool(H, P, T, seed):
    whh, bhh = default_weights(H, seed)
    return rand_x(P, T, H, seed + 1).cuda(), whh.cuda(), bhh.cuda()


@pytest.mark.parametrize("H", [256, 512])
def test_instances_batch_positions(H):
    """a stream's rows are identical whatever its batch position, B and instance (ragged last clusters included)"""
    T, P = 5, 2 * 48 + 3
    xp, whh, bhh = pool(H, P, T, seed=20)
    canon = gru_run(xp, whh, bhh, P, T, H, ns=16, xg=1)
    for ns, xg in INST[H]:
        for B in (1, ns - 1, ns, ns + 1, 2 * ns + 3):
            k = (7 * B + ns) % P      # batch row i holds pool stream (i + k) % P
            idx = (torch.arange(B) + k) % P
            h = gru_run(xp[idx.cuda()].contiguous(), whh, bhh, B, T, H, ns=ns, xg=xg)
            assert torch.equal(h, canon[idx.cuda()]), (H, ns, xg, B)
    # the production choice (ns = 0, xg = -1) as well
    assert torch.equal(gru_run(xp, whh, bhh, P, T, H), canon)


@pytest.mark.parametrize("H", [256, 512])
@pytest.mark.parametrize("inst", ["xg0", "xg1"])
def test_split_window(H, inst):
    """[0, T) split at s into two launches (the second from h0 = hT of the first, hT aliasing h0) equals one launch"""
    B, T = 5, 40
    ns, xg = 16, int(inst[-1])
    xp, whh, bhh = pool(H, B, T, seed=30)
    h0 = (torch.rand(B, H, generator=torch.Generator().manual_seed(31)) * 2 - 1).cuda()
    hT_one = torch.empty(B, H, device="cuda")
    one = gru_run(xp, whh, bhh, B, T, H, h0=h0, hT=hT_one, ns=ns, xg=xg)
    assert torch.equal(hT_one, one[:, -1])
    for s in (1, 7, T - 1):
        state = torch.empty(B, H, device="cuda")
        out = torch.zeros(B, T, H, device="cuda")
        assert gru_call(xp, whh, bhh, B, s, H, hout=out, h0=h0, hT=state, t0=0, Ts=T, ns=ns, xg=xg) == 0
        assert gru_call(xp, whh, bhh, B, T - s, H, hout=out, h0=state, hT=state, t0=s, Ts=T, ns=ns, xg=xg) == 0
        torch.cuda.synchronize()
        assert torch.equal(out, one), (H, inst, s)
        assert torch.equal(state, hT_one), (H, inst, s)


@pytest.mark.parametrize("H", [256, 512])
@pytest.mark.parametrize("inst", ["xg0", "xg1"])
def test_slot_first_frames(H, inst):
    """first frames before the window, at its start, inside it, at its last step and past its end, with w0 != 0 and a
    non-zero h0.  Before the first frame the rows are exactly 0; from it on they equal a fresh launch (h0 = NULL) from
    that frame.  A first frame at or before the window start means the stream was already running when the window
    began: its state entering the window is h0 (slots that open there start from zeroed state rows)."""
    Ts, t0, T, w0 = 40, 8, 24, 5
    steps = [-3, 0, 9, T - 1, T + 4]        # first frame, in steps of this window
    B = 2 * len(steps)
    ns, xg = 16, int(inst[-1])
    xp, whh, bhh = pool(H, B, Ts, seed=40)
    h0 = (torch.rand(B, H, generator=torch.Generator().manual_seed(41)) * 2 - 1).cuda()
    tf = [steps[b // 2] for b in range(B)]
    first = torch.tensor([w0 + t0 + v for v in tf], dtype=torch.int64, device="cuda")
    hT = torch.empty(B, H, device="cuda")
    h = gru_run(xp, whh, bhh, B, T, H, h0=h0, hT=hT, first=first, w0=w0, t0=t0, Ts=Ts, ns=ns, xg=xg)
    carried = gru_run(xp, whh, bhh, B, T, H, h0=h0, t0=t0, Ts=Ts, ns=ns, xg=xg)
    for b in range(B):
        f = tf[b]
        win = h[b, t0:t0 + T]
        if f <= 0:
            assert torch.equal(win, carried[b, t0:t0 + T]), (b, f)
            continue
        assert torch.equal(win[:min(f, T)], torch.zeros_like(win[:min(f, T)])), (b, f)
        if f >= T:
            assert torch.equal(hT[b], torch.zeros_like(hT[b])), (b, f)
            continue
        fresh_hT = torch.empty(B, H, device="cuda")
        fresh = gru_run(xp, whh, bhh, B, T - f, H, hT=fresh_hT, t0=t0 + f, Ts=Ts, ns=ns, xg=xg)
        assert torch.equal(win[f:], fresh[b, t0 + f:t0 + T]), (b, f)
        assert torch.equal(hT[b], fresh_hT[b]), (b, f)


def bf16_planes(x):
    """round-to-nearest-even BF16 hi / lo split of fp32 x (as int16)"""
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi.view(torch.int16), lo.view(torch.int16)


@pytest.mark.parametrize("H", [256, 512])
@pytest.mark.parametrize("out", ["fp32", "planes", "both"])
@pytest.mark.parametrize("planes_res", [0, 1])
def test_outputs_and_untouched(H, out, planes_res):
    """hout = h + res, the planes are the BF16 split of h (planes_res 0) or of h + res (1), hT is the residual-free last
    state; frames outside [t0, t0 + T) of the Ts-frame buffers and rows past B keep their sentinels"""
    if out == "fp32" and planes_res:
        pytest.skip("planes_res selects the planes' content")
    B, Bbuf, Ts, t0, T = 19, 21, 30, 6, 17
    xp, whh, bhh = pool(H, Bbuf, Ts, seed=50)
    res = torch.randn(Bbuf, Ts, H, generator=torch.Generator().manual_seed(51)).cuda()
    h0 = (torch.rand(Bbuf, H, generator=torch.Generator().manual_seed(52)) * 2 - 1).cuda()
    h = gru_run(xp, whh, bhh, B, T, H, h0=h0, t0=t0, Ts=Ts)      # residual-free reference launch
    fp32, planes = out in ("fp32", "both"), out in ("planes", "both")
    hout = torch.full((Bbuf, Ts, H), SENT, device="cuda") if fp32 else None
    hi = torch.full((Bbuf, Ts, H), SENT16, dtype=torch.int16, device="cuda") if planes else None
    lo = torch.full((Bbuf, Ts, H), SENT16, dtype=torch.int16, device="cuda") if planes else None
    hT = torch.full((Bbuf, H), SENT, device="cuda")
    rc = gru_call(xp, whh, bhh, B, T, H, res=res, hout=hout, hi=hi, lo=lo, planes_res=planes_res, h0=h0, hT=hT, t0=t0, Ts=Ts)
    assert rc == 0, lib().dfb_last_error()
    torch.cuda.synchronize()
    w = slice(t0, t0 + T)
    hw = h[:B, w]
    assert torch.equal(hT[:B], hw[:, -1]) and (hT[B:] == SENT).all()
    inside = torch.zeros(Bbuf, Ts, dtype=torch.bool, device="cuda")
    inside[:B, w] = True
    if fp32:
        assert torch.equal(hout[:B, w], hw + res[:B, w])
        assert (hout[~inside] == SENT).all()
    if planes:
        ph, pl = bf16_planes(hw + res[:B, w] if planes_res else hw)
        assert torch.equal(hi[:B, w], ph) and torch.equal(lo[:B, w], pl)
        assert (hi[~inside] == SENT16).all() and (lo[~inside] == SENT16).all()


def test_two_streams_and_exchange_scratch():
    """recurrences of H = 256 and 512 launched concurrently on two CUDA streams equal the same launches run serially;
    the exchange scratch of a stream grows (small B, large B, small B) without changing any result"""
    T = 300
    xa, wa, ba = pool(256, 64, T, seed=60)
    xb, wb, bb = pool(512, 32, T, seed=61)
    sa, sb = gru_run(xa, wa, ba, 64, T, 256), gru_run(xb, wb, bb, 32, T, 512)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    ca = gru_run(xa, wa, ba, 64, T, 256, stream=s1, sync=False)
    cb = gru_run(xb, wb, bb, 32, T, 512, stream=s2, sync=False)
    torch.cuda.synchronize()
    assert torch.equal(ca, sa) and torch.equal(cb, sb)
    # scratch growth on a fresh stream: 3 streams, then 16 * 20 + 5 (21 clusters), then 3 again
    T, P = 20, 325
    xp, whh, bhh = pool(256, P, T, seed=62)
    small, big = gru_run(xp[:3].contiguous(), whh, bhh, 3, T, 256, ns=16, xg=1), gru_run(xp, whh, bhh, P, T, 256, ns=32, xg=0)
    s3 = torch.cuda.Stream()
    for B, want in ((3, small), (P, big), (3, small)):
        got = gru_run(xp[:B].contiguous(), whh, bhh, B, T, 256, ns=16, xg=1, stream=s3)
        assert torch.equal(got, want), B


# ------------------------------------------------------------------------------------------- projection GEMM ----------

def gemm_shapes():
    """(N, K) of every k_gemm_bf16x3 launch of the shipped models: 3H x in_dim of each GRU layer (and a BF16x3 df_fc_out
    when its width is a multiple of 128 -- DeepFilterNet v1's 960 is not, it runs on the FFMA kernel)"""
    import bench
    from deepfilternet_b200.weights import pack_state_dict, pack_state_dict_v1, random_state_dict, random_state_dict_v1
    seen = set()
    for model in ("DeepFilterNet3", "DeepFilterNet2", "DeepFilterNet3_ll", "DeepFilterNet"):
        cfg = bench.model_config(model)
        if model == "DeepFilterNet":
            w, _ = pack_state_dict_v1(random_state_dict_v1(cfg, seed=0), cfg)
        else:
            w, _ = pack_state_dict(random_state_dict(cfg, seed=0), cfg)
        for k, v in w.items():
            if (k.endswith(".w_ih_hi") or k.endswith(".w_hi")) and v.shape[0] % 128 == 0:
                seen.add((v.shape[0], 2 * v.shape[1]))
    return sorted(seen)


def bench_m(H):
    import bench
    import bench_gl
    model = {256: "DeepFilterNet3", 512: "DeepFilterNet3_ll"}[H]
    return bench_gl.bench_rows(bench.model_config(model), *bench_gl.BENCH[model])


# |y - ref| <= GEMM_C1 * sum_k |x_k| |w_k| + 2^-23 |ref| (BF16x3 products to ~2^-16, fp32 accumulation over K, the fp32
# bias add); an H100 80GB HBM3 (700 W) measured at most 0.074 of the bound at GEMM_C1 = 3e-5, i.e. about 2.2e-6
GEMM_C1 = 8e-6
GEMM_BLOCK = 1024


def gemm_case(N, K, M, bias, seed):
    """x [M][K] (rows repeat a seeded block of GEMM_BLOCK), w [N][K], bias [N] on the CPU"""
    g = torch.Generator().manual_seed(seed)
    xb = torch.randn(min(M, GEMM_BLOCK), K, generator=g)
    w = torch.randn(N, K, generator=g) * K ** -0.5
    b = torch.randn(N, generator=g) if bias else None
    return xb, w, b


def gemm_run(xb, w, b, M, ldx_pad=64, ldy_pad=6, stream=None):
    """planes in buffers of pitch K + ldx_pad (garbage in the pad columns), y [M + 3][N + ldy_pad] with sentinels"""
    N, K = w.shape
    ldx, ldy = K + ldx_pad, N + ldy_pad
    reps = -(-M // xb.shape[0])
    x = xb.repeat(reps, 1)[:M]
    xfull = torch.full((M, ldx), 1e3)
    xfull[:, :K] = x
    xh, xl = (t.contiguous().cuda() for t in bf16_planes(xfull))
    wh, wl = (t.contiguous().cuda() for t in bf16_planes(w))
    y = torch.full((M + 3, ldy), SENT, device="cuda")
    bd = None if b is None else b.cuda()
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = lib().dfb_debug_gemm_bf16x3(ptr(xh), ptr(xl), ldx, ptr(wh), ptr(wl), ptr(bd), ptr(y), ldy, M, N, K, st)
    assert rc == 0, lib().dfb_last_error()
    torch.cuda.synchronize()
    return y


def gemm_check(xb, w, b, y, M, label):
    N, K = w.shape
    ref = xb.double() @ w.double().T + (0 if b is None else b.double())
    absdot = xb.double().abs() @ w.double().abs().T
    tol = (GEMM_C1 * absdot + 2.0 ** -23 * ref.abs()).cuda()
    ref = ref.cuda()
    assert (y[:, N:] == SENT).all() and (y[M:] == SENT).all(), label
    nb = xb.shape[0]
    worst = 0.0
    for r0 in range(0, M, nb):   # rows repeat the seeded block
        blk = y[r0:min(r0 + nb, M), :N].double()
        assert torch.isfinite(blk).all()
        worst = max(worst, float(((blk - ref[:blk.shape[0]]).abs() / tol[:blk.shape[0]]).max()))
    print(f"gemm {label}: measured / bound {worst:.3f}")
    assert worst <= 1.0, (label, worst)


@pytest.mark.parametrize("NK", gemm_shapes(), ids=lambda s: "N%d_K%d" % s)
@pytest.mark.parametrize("M", [1, 127, 128, 129, 300, "bench"])
@pytest.mark.parametrize("bias", [True, False])
def test_gemm_bf16x3(NK, M, bias):
    """element-wise bound; pad columns of x are ignored, columns past N and rows past M of y keep their sentinels"""
    N, K = NK
    M = bench_m(N // 3) if M == "bench" else M
    xb, w, b = gemm_case(N, K, M, bias, seed=N + M)
    y = gemm_run(xb, w, b, M)
    gemm_check(xb, w, b, y, M, f"N{N} K{K} M{M} bias{int(bias)}")


# max |h - h_float64| of projection + recurrence over 200 steps; an H100 80GB HBM3 (700 W) measured 7.8e-6 (H = 256) and
# 8.8e-6 (H = 512)
FREE_CHAINED = 3e-5


@pytest.mark.parametrize("H", [256, 512])
def test_projection_then_recurrence(H):
    """k_gemm_bf16x3 (W_ih x + b_ih from BF16 planes) then k_gru_tc against torch.nn.GRU(in_dim, H) in float64 with the
    real W_ih of a shipped configuration"""
    import bench
    from deepfilternet_b200.weights import pack_state_dict, random_state_dict
    model, name = {256: ("DeepFilterNet3", "enc.emb_gru.gru"), 512: ("DeepFilterNet3_ll", "df_dec.df_gru.gru")}[H]
    sd = random_state_dict(bench.model_config(model), seed=0)
    w_ih, b_ih = sd[name + ".weight_ih_l0"].float(), sd[name + ".bias_ih_l0"].float()
    whh, bhh = sd[name + ".weight_hh_l0"].float().contiguous(), sd[name + ".bias_hh_l0"].float().contiguous()
    in_dim = w_ih.shape[1]
    B, T = 3, 200
    x = torch.randn(B, T, in_dim, generator=torch.Generator().manual_seed(70))
    xproj = gemm_run(x.reshape(B * T, in_dim), w_ih, b_ih, B * T, ldx_pad=0, ldy_pad=0)[:B * T]
    h = gru_run(xproj.reshape(B, T, 3 * H).contiguous(), whh.cuda(), bhh.cuda(), B, T, H).cpu().double()
    with torch.no_grad():
        ref, _ = ref_gru(whh, bhh, H, w_ih, b_ih)(x.double())
    err = float((h - ref).abs().max())
    print(f"projection + recurrence H{H}: max|err| {err:.3e}  bound {FREE_CHAINED:.1e}")
    assert err <= FREE_CHAINED, err


# ------------------------------------------------------------------------------------------- errors -------------------

def test_errors_launch_nothing():
    """unbuilt instances, null outputs, T <= 0, a window past the buffer and unsupported GEMM shapes return their status
    and launch nothing"""
    from deepfilternet_b200._lib import DFB_ERR_INVALID, DFB_ERR_UNSUPPORTED
    L = lib()
    H, B, T = 256, 4, 8
    xp, whh, bhh = pool(512, B, T, seed=80)
    hout = torch.zeros(B, T, 512, device="cuda")
    hi = torch.zeros(B, T, 512, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    n0 = L.dfb_kernel_launches()
    cases = [
        (DFB_ERR_UNSUPPORTED, dict(H=512, ns=32, xg=1)), (DFB_ERR_UNSUPPORTED, dict(H=512, ns=48, xg=1)),
        (DFB_ERR_UNSUPPORTED, dict(H=H, ns=48, xg=0)), (DFB_ERR_UNSUPPORTED, dict(H=H, ns=24, xg=1)),
        (DFB_ERR_UNSUPPORTED, dict(H=H, ns=16, xg=2)), (DFB_ERR_UNSUPPORTED, dict(H=384)),
        (DFB_ERR_INVALID, dict(H=H, hout=None)), (DFB_ERR_INVALID, dict(H=H, hout=None, hi=hi)),
        (DFB_ERR_INVALID, dict(H=H, T=0)), (DFB_ERR_INVALID, dict(H=H, T=-1)), (DFB_ERR_INVALID, dict(H=H, B=0)),
        (DFB_ERR_INVALID, dict(H=H, t0=1)), (DFB_ERR_INVALID, dict(H=H, xp=None)),
    ]
    for want, kw in cases:
        a = dict(xp=xp, B=B, T=T, hout=hout, t0=0)
        a.update(kw)
        rc = gru_call(a.pop("xp"), whh, bhh, a.pop("B"), a.pop("T"), a.pop("H"), Ts=T, **a)
        assert rc == want, (kw, rc, L.dfb_last_error())
    st = torch.cuda.current_stream().cuda_stream
    w = torch.zeros(1536 * 512, dtype=torch.int16, device="cuda")
    y = torch.zeros(300 * 1536, device="cuda")
    # DeepFilterNet v1's df_fc_out (N = 960) is not a multiple of the 128-column tile
    assert L.dfb_debug_gemm_bf16x3(ptr(hi), ptr(hi), 512, ptr(w), ptr(w), None, ptr(y), 960, 32, 960, 512, st) == DFB_ERR_UNSUPPORTED
    assert L.dfb_debug_gemm_bf16x3(ptr(hi), ptr(hi), 512, ptr(w), ptr(w), None, ptr(y), 768, 0, 768, 512, st) == DFB_ERR_UNSUPPORTED
    assert L.dfb_debug_gemm_bf16x3(ptr(hi), ptr(hi), 512, ptr(w), ptr(w), None, None, 768, 32, 768, 512, st) == DFB_ERR_INVALID
    assert L.dfb_kernel_launches() == n0
    # and a valid launch counts exactly one
    assert gru_call(xp, whh, bhh, B, T, 512, hout=hout) == 0
    torch.cuda.synchronize()
    assert L.dfb_kernel_launches() == n0 + 1


# ------------------------------------------------------------------------------------------- dfb_debug_gru_timing -----

def test_gru_timing_fewer_steps_than_launch():
    """stamps armed for fewer steps than the recurrences run: no launch is stamped and the call succeeds; armed for
    enough steps, the first rows carry clock64 stamps of the five phases and the rest stay 0"""
    from deepfilternet_b200 import DfNet, _lib, enhance_device, libdf
    from deepfilternet_b200.weights import random_state_dict
    import bench
    cfg = bench.model_config("DeepFilterNet3")
    st = libdf.DF(cfg.sr, cfg.fft_size, cfg.hop_size, cfg.nb_erb, cfg.min_nb_erb_freqs)
    model = DfNet(cfg, random_state_dict(cfg, 0), st)
    model.set_chunking(1, 1, 1)
    audio = (torch.randn(1, 48000, generator=torch.Generator().manual_seed(90)) * 0.05).cuda()
    frames = (48000 + cfg.fft_size) // cfg.hop_size
    L = _lib.lib()
    for armed in (8, 4 * frames):
        _lib.check(L.dfb_debug_gru_timing(model.handle, armed, None))
        enhance_device(model, st, audio)
        torch.cuda.synchronize()
        buf = np.full((armed, 8), -1, dtype=np.int64)
        _lib.check(L.dfb_debug_gru_timing(model.handle, armed, buf.ctypes.data))
        assert (buf[:, 5:] == 0).all()
        if armed < frames:
            assert (buf == 0).all()
        else:
            n = int((buf[:, 0] != 0).sum())
            assert 0 < n < armed and (buf[:n, :5] > 0).all() and (buf[n:] == 0).all(), n
