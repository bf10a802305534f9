"""GPU: the tensor-core grouped linear (k_gl_bx) on its own, through dfb_debug_gl_bx, element by element against a float64
restatement of y = act(GL(x)) * oscale + ooffset + res, at every (G, Ig, Hg) that DeepFilterNet3, DeepFilterNet2 and
DeepFilterNet3_ll run on it.  Row counts below, at and past the 128-row tile and one bench-sized count; fp32 output, BF16
hi / lo planes or both; no residual, a separate one and one added in place (res = y, as df_out does).

The output bits are also pinned: tests/golden/gl_bx_bits.json holds SHA-256 digests of y, y_hi and y_lo for one seeded
case per shape, written by the kernel as it was before its epilogue moved to TMA loads and stores
(`python tests/test_gpu_gl_bx.py --write-golden` regenerates the file; only do that on purpose)."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench_gl  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden", "gl_bx_bits.json")
MODELS = ("DeepFilterNet3", "DeepFilterNet2", "DeepFilterNet3_ll")


def model_calls():
    """(model, call) for every k_gl_bx launch of the three models' forward passes"""
    import bench
    from deepfilternet_b200.weights import pack_state_dict, random_state_dict
    out = []
    for model in MODELS:
        cfg = bench.model_config(model)
        _, g = pack_state_dict(random_state_dict(cfg, seed=0), cfg)
        out += [(model, c) for c in bench_gl.gl_calls(cfg, g)]
    return out


def shapes():
    seen = []
    for _, c in model_calls():
        s = (c["G"], c["Ig"], c["Hg"])
        if s not in seen:
            seen.append(s)
    return seen


def bench_m():
    import bench
    return bench_gl.bench_rows(bench.model_config("DeepFilterNet3"), *bench_gl.BENCH["DeepFilterNet3"])


def reference(case, act, res, oscale, ooffset):
    """float64: act(x W) * oscale + ooffset (+ res), per group"""
    G, Ig, Hg, M = case.G, case.Ig, case.Hg, case.M
    x = case.x.astype(np.float64).reshape(M, G, Ig)
    y = np.einsum("mgi,gih->mgh", x, case.w.astype(np.float64)).reshape(M, G * Hg)
    if act == bench_gl.ACT_RELU:
        y = np.maximum(y, 0.0)
    elif act == bench_gl.ACT_TANH:
        y = np.tanh(y)
    y = y * oscale + ooffset
    if res is not None:
        y = y + case.r.astype(np.float64)
    return y


def bf16_pair_to_f64(hi, lo):
    f = lambda u: (u.astype(np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return f(hi) + f(lo)


def run(G, Ig, Hg, M, fp32, planes, res, act, oscale, ooffset, seed=3):
    """res: None, "sep" (a separate tensor) or "y" (in place).  Returns (case, y or None, (hi, lo) or None)"""
    import torch
    case = bench_gl.GlCase(G, Ig, Hg, M, fp32=fp32 or res == "y", planes=planes, seed=seed)
    rt = None
    if res == "y":
        case.set_residual()
        rt = "y"
    elif res == "sep":
        rt = torch.from_numpy(case.r).cuda()
    case.launch(act, rt, oscale, ooffset)
    torch.cuda.synchronize()
    y = case.y.cpu().numpy() if case.y is not None else None
    pl = (case.y_hi.cpu().numpy(), case.y_lo.cpu().numpy()) if planes else None
    return case, y, pl


def check(case, y, pl, act, res, oscale, ooffset):
    ref = reference(case, act, res, oscale, ooffset)
    # BF16x3 products (x and w each carried to ~2^-17 by hi + lo, lo * lo dropped) accumulated in fp32 over K = Ig: bounded
    # by sum |x| |w| (act is 1-Lipschitz); tanh on the MUFU units (~1e-6 absolute); planes: hi + lo carries ~2^-17 of y
    G, Ig, Hg, M = case.G, case.Ig, case.Hg, case.M
    absdot = np.einsum("mgi,gih->mgh", np.abs(case.x.astype(np.float64)).reshape(M, G, Ig),
                       np.abs(case.w.astype(np.float64))).reshape(M, G * Hg)
    tol = 3e-5 * absdot * abs(oscale) + 2e-5 * np.abs(ref) + 2e-6
    for got in ([y] if y is not None else []) + ([bf16_pair_to_f64(*pl)] if pl is not None else []):
        assert got.shape == ref.shape and np.isfinite(got).all()
        bad = np.abs(got - ref) > tol
        assert not bad.any(), (int(bad.sum()), float(np.abs(got - ref).max()), float(np.abs(ref).max()))


SHAPES = shapes()


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "G%d_Ig%d_Hg%d" % s)
@pytest.mark.parametrize("M", [1, 127, 128, 129, 300])
def test_gl_bx_rows(shape, M):
    """every shape at row counts around the tile: both outputs, residual in place, tanh, non-trivial scale / offset"""
    case, y, pl = run(*shape, M, True, True, "y", bench_gl.ACT_TANH, 0.75, -0.125)
    check(case, y, pl, bench_gl.ACT_TANH, "y", 0.75, -0.125)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "G%d_Ig%d_Hg%d" % s)
@pytest.mark.parametrize("out", ["fp32", "planes", "both"])
@pytest.mark.parametrize("res", [None, "sep", "y"])
@pytest.mark.parametrize("act", [bench_gl.ACT_NONE, bench_gl.ACT_RELU, bench_gl.ACT_TANH])
def test_gl_bx_modes(shape, out, res, act):
    if res == "y" and out == "planes":
        pytest.skip("an in-place residual is read from the fp32 output")
    fp32, planes = out in ("fp32", "both"), out in ("planes", "both")
    case, y, pl = run(*shape, 300, fp32, planes, res, act, 1.0, 0.0)
    check(case, y, pl, act, res, 1.0, 0.0)


@pytest.mark.parametrize("model,call", [(m, c) for m, c in model_calls() if m == "DeepFilterNet3"],
                         ids=lambda v: v if isinstance(v, str) else v["name"])
def test_gl_bx_bench_rows(model, call):
    """each DeepFilterNet3 call as forward_body makes it, at the bench config's row count"""
    res = "y" if call["res"] else None
    case, y, pl = run(call["G"], call["Ig"], call["Hg"], bench_m(), call["fp32"] or call["res"], call["planes"], res,
                      call["act"], 1.0, 0.0)
    check(case, y, pl, call["act"], res, 1.0, 0.0)


GOLDEN_M, GOLDEN_SCALE, GOLDEN_OFFSET = 300, 0.75, -0.125


def golden_case(shape):
    case, y, pl = run(*shape, GOLDEN_M, True, True, "y", bench_gl.ACT_TANH, GOLDEN_SCALE, GOLDEN_OFFSET, seed=11)
    d = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    return {"y": d(y.view(np.uint32)), "y_hi": d(pl[0]), "y_lo": d(pl[1]), "y_row0": [int(v) for v in y.view(np.uint32)[0, :8]]}


def test_gl_bx_golden_bits():
    """the output bits of one seeded case per shape (in-place residual, tanh, scale / offset, both outputs) equal those
    the kernel produced before its data movement was reworked"""
    with open(GOLDEN) as f:
        gold = json.load(f)
    assert sorted(gold) == sorted("G%d_Ig%d_Hg%d" % s for s in SHAPES)
    for s in SHAPES:
        key = "G%d_Ig%d_Hg%d" % s
        assert golden_case(s) == gold[key], key


if __name__ == "__main__":
    if sys.argv[1:] != ["--write-golden"]:
        raise SystemExit("usage: python tests/test_gpu_gl_bx.py --write-golden")
    out = {"G%d_Ig%d_Hg%d" % s: golden_case(s) for s in SHAPES}
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {GOLDEN}: {len(out)} shapes")
