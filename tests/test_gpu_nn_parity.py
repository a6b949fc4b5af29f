"""GPU parity tests (H100): the CUDA path THROUGH THE C ABI against the numpy oracle, the committed golden fixtures
(reference PyTorch model outputs), and size-independent properties at BASELINE.json's full sizes.

Tolerances (written here on purpose):
  * fp32-equivalent mode (useFP16=false: 3-term split-fp16 on the tensor pipe, fp32 accumulate and streams):
      |logit - oracle| <= 1e-3  (north_star: "policy/value logits within 1e-3 fp32")
  * fp16 mode (fp16 operands, fp32 accumulate): relative to the largest logit of the row set, <= 1.5e-2
    (the reference's own fp16 GPU path is compared with its fp32 path by distribution thresholds, not bitwise:
     cpp/tests/testnnevalcanary.cpp:256-470)
"""
import os

import numpy as np
import pytest

import kg_nn_oracle as orc
from katago_b200 import NeuralNet, modelgen

pytestmark = pytest.mark.gpu

FP32_TOL = 1e-3
FP16_REL = 1.5e-2


def run_cuda(path, sp, gl, sym, opt, fp16, X=19, Y=19, nhwc=True, max_batch=None):
    lm = NeuralNet.loadModelFile(path)
    ctx = NeuralNet.createComputeContext([0], X, Y, fp16, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, max_batch or max(4, sp.shape[0]), False, nhwc, 0)
    assert NeuralNet.isUsingFP16(h) == bool(fp16)
    flat = sp.reshape(sp.shape[0], -1) if nhwc else np.ascontiguousarray(sp.transpose(0, 3, 1, 2)).reshape(sp.shape[0], -1)
    out = NeuralNet.getOutput(h, flat, gl, sym, opt)
    h.free(); ctx.free(); lm.free()
    return out


def check(got, ref, fp16):
    for k in ("policy", "value", "score_value", "ownership"):
        err = np.abs(got[k] - ref[k]).max()
        assert np.isfinite(got[k]).all()
        if fp16:
            assert err <= FP16_REL * max(1.0, np.abs(ref[k]).max()), (k, err)
        else:
            assert err <= FP32_TOL, (k, err)


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("ky,cin,cout,n,X,Y", [(1, 64, 64, 2, 19, 19), (3, 22, 96, 3, 9, 9), (5, 22, 96, 3, 9, 9), (3, 192, 192, 5, 19, 19),
                                               (1, 384, 192, 9, 19, 19), (1, 192, 384, 4, 19, 19), (3, 128, 192, 8, 13, 7), (3, 40, 320, 2, 19, 19)])
def test_conv_layer(ky, cin, cout, n, X, Y, fp16):
    """NeuralNet::testEvaluateConv analogue (cpp/tests/testnn.cpp:107-341 tests the same hook with fixed tensors)."""
    rng = np.random.default_rng(ky * 1000 + cin)
    w = (rng.standard_normal((ky, ky, cin, cout)) * np.sqrt(1.0 / (ky * ky * cin))).astype(np.float32)
    x = rng.standard_normal((n, Y, X, cin)).astype(np.float32)
    if fp16:  # operands exactly representable -> only accumulation order differs
        w, x = w.astype(np.float16).astype(np.float32), x.astype(np.float16).astype(np.float32)
    ref = orc.conv2d(x, orc.Conv("t", ky, ky, cin, cout, w))
    got = NeuralNet.testEvaluateConv(ky, ky, cin, cout, w, n, X, Y, fp16, x)
    assert np.abs(got - ref).max() < (2e-4 if not fp16 else 1e-4)


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("kind", [1, 2, 3])
@pytest.mark.parametrize("ky,cin,cout,n,X,Y,act", [(3, 192, 192, 5, 19, 19, 2), (1, 384, 192, 9, 19, 19, 2), (1, 192, 384, 7, 19, 19, 2),
                                                   (3, 256, 256, 3, 19, 19, 2), (3, 64, 128, 4, 13, 7, 1), (5, 22, 64, 3, 9, 9, 0),
                                                   (3, 96, 96, 70, 9, 9, 2)])
def test_conv_fused_epilogues(ky, cin, cout, n, X, Y, act, kind, fp16):
    """The three production epilogues of a trunk convolution (kgb_conv.cuh): kind 1 = next layer's BN + activation + mask as an fp16
    operand; 2 = + the residual stream, read and rewritten in place; 3 = raw stream + operand.  Reference: NormActConv / residual add of
    ResidualBlock::apply and NestedBottleneckResidualBlock::apply (eigenbackend.cpp:1065-1077, 1127-1160, 1295-1314).  Pad rows of the
    operand must come back as zeros (checked inside the hook).  (3, 96, 96, 70, 9, 9): more than one CTA-pair tile per cluster."""
    from katago_b200 import nn_backend
    rng = np.random.default_rng(ky * 100 + cin + kind)
    w = (rng.standard_normal((ky, ky, cin, cout)) * np.sqrt(1.0 / (ky * ky * cin))).astype(np.float16).astype(np.float32)
    x = rng.standard_normal((n, Y, X, cin)).astype(np.float16).astype(np.float32)
    res = rng.standard_normal((n, Y, X, cout)).astype(np.float16).astype(np.float32) if kind == 2 else None
    sc = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    bi = rng.uniform(-0.5, 0.5, cout).astype(np.float32)
    raw_ref = orc.conv2d(x, orc.Conv("t", ky, ky, cin, cout, w))
    if res is not None:
        raw_ref = raw_ref + res
    z = raw_ref * sc + bi
    if act == 2:
        act_ref = z * np.tanh(np.log1p(np.exp(np.minimum(z, 30.0))))
    elif act == 1:
        act_ref = np.maximum(z, 0.0)
    else:
        act_ref = z
    raw, a = nn_backend.test_conv_epilogue(ky, ky, cin, cout, w, n, X, Y, fp16, kind, x, res, sc, bi, act)
    # fp16 mode stores both tensors as fp16 (relative 2^-11); fp32-equivalent mode stores raw as fp32 and the operand as hi + lo halves
    tol_raw = 4e-3 if fp16 else 3e-4
    tol_act = 4e-3 if fp16 else 3e-4
    if raw is not None:
        assert np.abs(raw - raw_ref).max() <= tol_raw * max(1.0, np.abs(raw_ref).max()), np.abs(raw - raw_ref).max()
    assert np.abs(a - act_ref).max() <= tol_act * max(1.0, np.abs(act_ref).max()), np.abs(a - act_ref).max()


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("cfg", ["b2c16", "b2c32nbt", "b4c32"])
def test_golden_reference_pytorch_outputs(golden_dir, cfg, fp16):
    d = np.load(os.path.join(golden_dir, f"torchref_{cfg}.npz"))
    sp, gl = d["spatial_nhwc"].astype(np.float32), d["global_"]
    n = sp.shape[0]
    on = sp[..., 0].reshape(n, -1) > 0
    path = os.path.join(golden_dir, "models", f"torchref_{cfg}.bin.gz")
    for opt, key in ((0.0, "policy0"), (1.0, "policy_opt")):
        got = run_cuda(path, sp, gl, None, np.full(n, opt, np.float32), fp16)
        tol = FP32_TOL if not fp16 else FP16_REL
        assert np.abs(got["policy"][:, :361] - d[key][:, :361])[on].max() < tol
        assert np.abs(got["policy"][:, 361] - d[key][:, 361]).max() < tol
        assert np.abs(got["value"] - d["value"]).max() < tol
        assert np.abs(got["score_value"] - d["score_value"]).max() < tol
        assert np.abs(got["ownership"] - d["ownership"])[on].max() < tol


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("key,n,X,Y,sizes", [
    ("tiny_reg", 3, 9, 9, None),
    ("tiny_nbt", 5, 19, 19, [(19, 19), (9, 9), (13, 13), (19, 19), (7, 11)]),   # mixed board sizes: pad + mask (config 4)
    ("mid_nbt", 9, 19, 19, None),
    ("tiny_relu_v8", 2, 13, 13, None),
    ("tiny_nbt", 1, 19, 19, None),
    ("tiny_reg", 4, 11, 7, None),                                                # rectangular nnXLen != nnYLen
])
def test_synthetic_nets_vs_oracle(tmp_models, key, n, X, Y, sizes, fp16):
    sp, gl = modelgen.synthetic_inputs(n, X, Y, seed=n + X, board_sizes=sizes)
    sym = (np.arange(n) * 3 + 1) % 8
    opt = np.linspace(0.0, 1.0, n).astype(np.float32)
    ref = orc.get_output(orc.load_model(tmp_models[key]), sp, gl, sym, opt)
    check(run_cuda(tmp_models[key], sp, gl, sym, opt, fp16, X, Y), ref, fp16)


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("X", [19, 9])
def test_real_g170_net_vs_oracle(golden_dir, X, fp16):
    """A trained net from the reference's test suite (5x5 first conv, relu, v8, trunk-level gpool blocks)."""
    path = os.path.join(golden_dir, "models", "g170-b6c96-s175395328-d26788732.bin.gz")
    sp, gl = modelgen.synthetic_inputs(4, X, X, seed=21)
    sym = np.array([0, 2, 5, 7])
    ref = orc.get_output(orc.load_model(path), sp, gl, sym)
    got = run_cuda(path, sp, gl, sym, None, fp16, X, X)
    if fp16:
        check(got, ref, True)
    else:  # logits reach |52| on this net: 1e-3 absolute is 2e-5 relative
        check(got, ref, False)


def test_nchw_and_nhwc_inputs_agree(tmp_models):
    sp, gl = modelgen.synthetic_inputs(3, 19, 19, seed=9)
    a = run_cuda(tmp_models["tiny_nbt"], sp, gl, None, None, False, nhwc=True)
    b = run_cuda(tmp_models["tiny_nbt"], sp, gl, None, None, False, nhwc=False)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_rows_are_independent_of_batch_composition(tmp_models):
    """Size-independent property: a row's result does not depend on which other rows share its batch (bit-exact),
    and repeated calls on one handle are deterministic."""
    sp, gl = modelgen.synthetic_inputs(7, 19, 19, seed=12, board_sizes=[(19, 19)] * 3 + [(9, 9)] * 4)
    lm = NeuralNet.loadModelFile(tmp_models["mid_nbt"])
    ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 16, False, True, 0)
    full = NeuralNet.getOutput(h, sp.reshape(7, -1), gl)
    again = NeuralNet.getOutput(h, sp.reshape(7, -1), gl)
    for k in full:
        assert np.array_equal(full[k], again[k])
    perm = np.array([4, 0, 6, 2])
    sub = NeuralNet.getOutput(h, sp[perm].reshape(4, -1), gl[perm])
    for k in full:
        assert np.array_equal(full[k][perm], sub[k]), k
    one = NeuralNet.getOutput(h, sp[5:6].reshape(1, -1), gl[5:6])
    for k in full:
        assert np.array_equal(full[k][5:6], one[k]), k
    h.free(); ctx.free()


def test_symmetry_equivariance_on_device(tmp_models):
    m = tmp_models["tiny_reg"]
    sp, gl = modelgen.synthetic_inputs(1, 9, 9, seed=5)
    base = {s: run_cuda(m, sp, gl, [s], None, False, 9, 9) for s in range(8)}
    for s in range(8):
        rot = orc.apply_symmetry_nhwc(sp[0], s, False)[None]
        b = run_cuda(m, rot, gl, [0], None, False, 9, 9)
        back = orc.apply_symmetry_nhwc(b["policy"][0, :81].reshape(9, 9), s, True).reshape(-1)
        assert np.abs(base[s]["policy"][0, :81] - back).max() < 1e-5
        assert np.abs(base[s]["value"] - b["value"]).max() < 1e-5


def test_bad_arguments_are_reported(tmp_models):
    from katago_b200 import KGBError
    lm = NeuralNet.loadModelFile(tmp_models["tiny_reg"])
    ctx = NeuralNet.createComputeContext([0], 9, 9, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 2, False, True, 0)
    sp, gl = modelgen.synthetic_inputs(3, 9, 9, seed=1)
    with pytest.raises(KGBError, match="batch size"):
        NeuralNet.getOutput(h, sp.reshape(3, -1), gl)
    with pytest.raises(KGBError, match="symmetry"):
        NeuralNet.getOutput(h, sp[:1].reshape(1, -1), gl[:1], [9])
    with pytest.raises(KGBError):
        NeuralNet.createComputeHandle(ctx, lm, 4, False, True, 99)


@pytest.mark.parametrize("cfg", ["b18c384nbt"])
def test_full_size_b18_batch256(cfg, tmp_path):
    """BASELINE.json configs[1] shape: b18c384nbt, 19x19, 256 rows.  The oracle would need ~2 min for 256 rows, so it
    checks 6 of them; all 256 go through the size-independent properties (finite; rows repeated at different batch
    positions give identical results; fp32-equivalent and fp16 modes agree to fp16 accuracy)."""
    path = modelgen.write_model(str(tmp_path / f"{cfg}.bin"), cfg, seed=0)
    n = 256
    sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=77)
    sp[128:] = sp[:128][::-1]; gl[128:] = gl[:128][::-1]          # second half = first half reversed
    sym = np.zeros(n, np.int32)
    got16 = run_cuda(path, sp, gl, sym, None, True, max_batch=n)
    got32 = run_cuda(path, sp, gl, sym, None, False, max_batch=n)
    for k in got16:
        assert np.isfinite(got16[k]).all() and np.isfinite(got32[k]).all()
        assert np.array_equal(got16[k][128:], got16[k][:128][::-1]), k
        assert np.abs(got16[k] - got32[k]).max() <= FP16_REL * max(1.0, np.abs(got32[k]).max()), k
    idx = np.array([0, 17, 101, 127, 200, 255])
    ref = orc.get_output(orc.load_model(path), sp[idx], gl[idx], sym[idx])
    for k in ref:
        assert np.abs(got32[k][idx] - ref[k]).max() <= FP32_TOL, (k, np.abs(got32[k][idx] - ref[k]).max())
        assert np.abs(got16[k][idx] - ref[k]).max() <= FP16_REL * max(1.0, np.abs(ref[k]).max()), k


@pytest.mark.parametrize("fp16", [False, True])
def test_reference_tiny_net_known_answers_on_device(golden_dir, fp16):
    """The reference's own known-answer test for the NN path (cpp/tests/tinymodel.cpp; fixture tests/golden/tinymodel.json.gz) through the
    C ABI: its two embedded nets, three positions (one 13x6 on the 19x19 frame), the symmetries it fixes, the outputs it expects and
    its own tolerances."""
    import gzip, json
    from test_oracle_nn import _post_process
    blocks = json.loads(gzip.open(os.path.join(golden_dir, "tinymodel.json.gz"), "rb").read())
    for b in blocks:
        path = os.path.join(golden_dir, "models", b["model"] + ".bin.gz")
        version = orc.load_model(path).version
        sp = np.array(b["spatial"], np.float32).reshape(1, 19, 19, 22)
        gl = np.array(b["global"], np.float32).reshape(1, 19)
        out = run_cuda(path, sp, gl, np.array([b["symmetry"]], np.int32), None, fp16)
        got = _post_process({k: np.asarray(v)[0] for k, v in out.items()}, b["legal"], version, black_to_move=True, ko_simple=bool(b["koRuleSimple"]))
        for name, (expected, tol) in b["scalars"].items():
            assert abs(got[name] - expected) <= tol, (b["model"], b["symmetry"], name, got[name], expected, tol)
        X, Y = b["X"], b["Y"]
        idx = np.array([(i % X) + (i // X) * 19 for i in range(X * Y)])
        k = 0.1 if b["model"] == "tinymodel" else 0.15
        cap = 120.0 if (X, Y) == (13, 6) else 60.0
        own_tol = 300.0 if b["model"] == "tinymodel" else 600.0
        for e, p in zip(b["arrays"]["expectedPolicy"], got["policy"][idx]):
            if e >= 0:
                assert abs(p * 10000 - e) <= min(cap, e * k + 2.0) + min(10.0, e * k), (b["model"], e, p * 10000)
        for e, o in zip(b["arrays"]["expectedOwnership"], got["ownership"][idx]):
            assert abs(o * 10000 - e) <= own_tol, (b["model"], e, o * 10000)
