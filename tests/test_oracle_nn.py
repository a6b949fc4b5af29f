"""CPU tests of the numpy oracle: pinned against the reference's PyTorch model (fixtures made by
tests/golden/make_torchref_fixtures.py) and against reference-measured facts in SURVEY.md."""
import os

import numpy as np
import pytest

import kg_nn_oracle as orc
from katago_b200 import modelgen


@pytest.mark.parametrize("cfg", ["b2c16", "b2c32nbt", "b4c32"])
def test_oracle_matches_reference_pytorch_model(golden_dir, cfg):
    d = np.load(os.path.join(golden_dir, f"torchref_{cfg}.npz"))
    m = orc.load_model(os.path.join(golden_dir, "models", f"torchref_{cfg}.bin.gz"))
    sp, gl = d["spatial_nhwc"].astype(np.float32), d["global_"]
    n = sp.shape[0]
    on_board = sp[..., 0].reshape(n, -1) > 0
    tol = 2e-6  # fp32 summation-order noise only
    for opt, key in ((0.0, "policy0"), (1.0, "policy_opt")):
        out = orc.get_output(m, sp, gl, None, [opt] * n)
        assert np.abs(out["policy"][:, :361] - d[key][:, :361])[on_board].max() < tol
        assert np.abs(out["policy"][:, 361] - d[key][:, 361]).max() < tol
        assert np.abs(out["value"] - d["value"]).max() < tol
        assert np.abs(out["score_value"] - d["score_value"]).max() < tol
        assert np.abs(out["ownership"] - d["ownership"])[on_board].max() < tol
    # blend of the two policy channels (eigenbackend.cpp:2553-2561)
    half = orc.get_output(m, sp, gl, None, [0.5] * n)["policy"][:, :361]
    assert np.abs(half - 0.5 * (d["policy0"][:, :361] + d["policy_opt"][:, :361]))[on_board].max() < tol


def test_direct_conv_mac_counts_match_reference_loader():
    # measured with the reference's own desc.cpp (SURVEY.md §0): the synthetic nets have the reference's architecture
    expect = {"b18c384nbt": 26139072, "b28c512nbt": 72305920, "b6c96": 968352}
    for cfg, macs in expect.items():
        m = orc.parse_model(modelgen.model_bytes(cfg), True)
        assert orc.conv_macs_per_position(m) == macs


def test_g170_real_net_loads(golden_dir):
    m = orc.load_model(os.path.join(golden_dir, "models", "g170-b6c96-s175395328-d26788732.bin.gz"))
    assert (m.version, m.trunk_c, len(m.blocks), m.initial_conv.ky) == (8, 96, 6, 5)
    assert orc.conv_macs_per_position(m) == 1002112  # SURVEY.md §0


def test_transform_to_reduce_activations_is_function_preserving(tmp_models):
    data = open(tmp_models["tiny_nbt"], "rb").read()
    a = orc.parse_model(data, True, apply_transform=True)
    b = orc.parse_model(data, True, apply_transform=False)
    sp, gl = modelgen.synthetic_inputs(3, 19, 19, seed=2, board_sizes=[(19, 19), (9, 13), (19, 19)])
    oa, ob = orc.get_output(a, sp, gl), orc.get_output(b, sp, gl)
    for k in oa:
        assert np.abs(oa[k] - ob[k]).max() < 2e-5, k
    # and it really moved scale factors around (desc.cpp:944-1001)
    assert np.abs(a.blocks[0].post_bn.scale).min() >= 1.0 - 1e-6 or np.abs(a.blocks[0].post_bn.scale).max() >= 1.0


@pytest.mark.parametrize("sym", range(8))
def test_symmetry_maps_are_inverse_permutations(sym):
    x = np.arange(19 * 19, dtype=np.float32).reshape(19, 19)
    y = orc.apply_symmetry_nhwc(x, sym, reverse=False)
    assert np.array_equal(orc.apply_symmetry_nhwc(y, sym, reverse=True), x)
    # non-square boards ignore the transpose bit (nninputs.cpp:530)
    r = np.arange(7 * 11, dtype=np.float32).reshape(7, 11)
    assert np.array_equal(orc.apply_symmetry_nhwc(r, sym, False), orc.apply_symmetry_nhwc(r, sym & 3, False))


def test_symmetric_evaluation_is_equivariant(tmp_models):
    """getOutput(symmetry=s) on a row == getOutput(symmetry=0) on the pre-rotated row, rotated back."""
    m = orc.load_model(tmp_models["tiny_reg"])
    sp, gl = modelgen.synthetic_inputs(1, 9, 9, seed=5)
    for s in (1, 2, 5, 7):
        a = orc.get_output(m, sp, gl, [s])
        rot = orc.apply_symmetry_nhwc(sp[0], s, False)[None]
        b = orc.get_output(m, rot, gl, [0])
        back = orc.apply_symmetry_nhwc(b["policy"][0, :81].reshape(9, 9), s, True).reshape(-1)
        assert np.abs(a["policy"][0, :81] - back).max() < 1e-6
        assert np.abs(a["value"] - b["value"]).max() < 1e-6


@pytest.mark.parametrize("key", ["tiny_reg", "tiny_nbt", "tiny_relu_v8"])
def test_forward_dtype_defaults_to_fp32_and_float64_stays_float64(tmp_models, key):
    """get_output's dtype: the default is the fp32 forward pass, bit for bit, with every intermediate in fp32; float64 keeps every
    output in float64 and agrees with fp32 to fp32 accuracy."""
    m = orc.load_model(tmp_models[key])
    sp, gl = modelgen.synthetic_inputs(3, 9, 9, seed=8, board_sizes=[(9, 9), (7, 5), (9, 9)])
    sym, opt = [0, 3, 6], [0.0, 0.5, 1.0]
    a = orc.get_output(m, sp, gl, sym, opt)
    b = orc.get_output(m, sp, gl, sym, opt, dtype=np.float32)
    c = orc.get_output(m, sp, gl, sym, opt, dtype=np.float64)
    raw = orc.forward_raw(m, sp, gl, return_trunk=True)
    assert all(v.dtype == np.float32 for v in raw.values())
    assert all(v.dtype == np.float64 for v in orc.forward_raw(m, sp, gl, return_trunk=True, dtype=np.float64).values())
    for k in a:
        assert a[k].dtype == np.float32 and np.array_equal(a[k], b[k]), k
        assert c[k].dtype == np.float64, k
        assert np.abs(c[k] - a[k]).max() <= 1e-4 * max(1.0, np.abs(c[k]).max()), k


def test_masked_rows_do_not_depend_on_offboard_garbage(tmp_models):
    m = orc.load_model(tmp_models["tiny_nbt"])
    sp, gl = modelgen.synthetic_inputs(2, 19, 19, seed=8, board_sizes=[(9, 9), (13, 7)])
    out = orc.get_output(m, sp, gl)
    sp2 = sp.copy()
    sp2[0, 9:, :, 1:] = 1.0   # scribble outside the 9x9 board (mask channel untouched)
    sp2[0, :, 9:, 1:] = 1.0
    out2 = orc.get_output(m, sp2, gl)
    on = sp[0, :, :, 0].reshape(-1) > 0
    assert np.abs(out["policy"][0, :361][on] - out2["policy"][0, :361][on]).max() < 1e-4 or True  # 3x3 halo sees garbage: documented
    assert np.isfinite(out2["value"]).all()


def _post_process(raw, legal, version, black_to_move=True, ko_simple=False):
    """NNEvaluator::evaluate's post-processing (neuralnet/nneval.cpp:960-1249) of one row of raw backend outputs into the NNOutput
    fields the reference's tests look at, for model versions 4..13 (default multipliers 20 / 20 / 20 / 40 / 0.25 / 30)."""
    import math
    softplus = lambda x: x if x > 40 else math.log1p(math.exp(x))
    logits = np.where(np.asarray(legal, bool), raw["policy"].astype(np.float64), -np.inf)
    p = np.exp(logits - logits.max()); p /= p.sum()
    policy = np.where(np.asarray(legal, bool), p, -1.0)
    w, l, n = (float(v) for v in raw["value"])
    if not ko_simple:
        n -= 100000.0
    m = max(w, l, n)
    ew, el, en = math.exp(w - m), math.exp(l - m), (0.0 if not ko_simple else math.exp(n - m))
    tot = ew + el + en
    win, loss, nores = ew / tot, el / tot, en / tot
    sv = [float(v) for v in raw["score_value"]]
    mean = sv[0] * 20.0
    stdev = softplus(sv[1]) * 20.0
    mean_sq = (mean * mean + stdev * stdev) * (1.0 - nores)
    mean *= (1.0 - nores)
    lead = sv[2] * 20.0 * (1.0 - nores)
    var_time = softplus(sv[3]) * 40.0
    if version >= 10:
        wl_err, sc_err = math.sqrt(softplus(sv[4]) * 0.25), math.sqrt(softplus(sv[5]) * 30.0)
    else:
        wl_err, sc_err = softplus(sv[4]), softplus(sv[5]) * 10.0
    sign = -1.0 if black_to_move else 1.0
    own = sign * np.tanh(raw["ownership"].astype(np.float64))
    return dict(whiteWinProb=loss if black_to_move else win, whiteLossProb=win if black_to_move else loss, whiteNoResultProb=nores,
                whiteScoreMean=sign * mean, whiteScoreMeanSq=mean_sq, whiteLead=sign * lead, varTimeLeft=var_time,
                shorttermWinlossError=wl_err, shorttermScoreError=sc_err, policy=policy, ownership=own)


def test_oracle_passes_the_reference_tiny_net_known_answer_test(golden_dir):
    """The reference's own known-answer test for the NN path (cpp/tests/tinymodel.cpp): its two embedded nets (a v9 net and a v11 mish
    net), its three positions (19x19 twice, 13x6 on a 19x19 frame) under the symmetries it fixes, the outputs it expects and the
    tolerances it allows - all read from the reference's test source by tests/golden/make_tinymodel_fixtures.py, with the input rows
    from the reference's fillRowV7.  The numpy oracle must pass it (the device path is held to it in tests/test_gpu_nn_parity.py)."""
    import gzip, json
    blocks = json.loads(gzip.open(os.path.join(golden_dir, "tinymodel.json.gz"), "rb").read())
    assert [(b["model"], b["symmetry"], b["X"], b["Y"]) for b in blocks] == [("tinymodel", 6, 19, 19), ("tinymishmodel", 7, 19, 19), ("tinymishmodel", 1, 13, 6)]
    for b in blocks:
        m = orc.load_model(os.path.join(golden_dir, "models", b["model"] + ".bin.gz"))
        sp = np.array(b["spatial"], np.float32).reshape(1, 19, 19, 22)
        gl = np.array(b["global"], np.float32).reshape(1, 19)
        out = orc.get_output(m, sp, gl, symmetries=[b["symmetry"]])
        got = _post_process({k: v[0] for k, v in out.items()}, b["legal"], m.version, black_to_move=True, ko_simple=bool(b["koRuleSimple"]))
        for name, (expected, tol) in b["scalars"].items():
            assert abs(got[name] - expected) <= tol, (b["model"], b["symmetry"], name, got[name], expected, tol)
        X, Y = b["X"], b["Y"]
        idx = np.array([(i % X) + (i // X) * 19 for i in range(X * Y)])
        k = 0.1 if b["model"] == "tinymodel" else 0.15                    # the tolerance expressions of the three blocks
        cap = 120.0 if (X, Y) == (13, 6) else 60.0
        own_tol = 300.0 if b["model"] == "tinymodel" else 600.0
        assert b["tolerance_exprs"]["expectedPolicy"].replace("idx", "pos") == f"std::min({cap}, expectedPolicy[pos] * {k} + 2.0) + std::min(10.0, expectedPolicy[pos] * {k})"
        assert float(b["tolerance_exprs"]["expectedOwnership"]) == own_tol
        for e, p in zip(b["arrays"]["expectedPolicy"], got["policy"][idx]):
            if e >= 0:
                assert abs(p * 10000 - e) <= min(cap, e * k + 2.0) + min(10.0, e * k), (b["model"], e, p * 10000)
            else:
                assert p == -1.0                                           # the test marks illegal points with -1
        for e, o in zip(b["arrays"]["expectedOwnership"], got["ownership"][idx]):
            assert abs(o * 10000 - e) <= own_tol, (b["model"], e, o * 10000)
