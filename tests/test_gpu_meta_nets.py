"""GPU tests (H100) of SGF-metadata (human SL) nets: the encoder on the device against the metadata oracle (tests/meta_oracle.py) on
real metadata rows (tests/golden/metarows.npz, SGFMetadata::fillMetadataRow of the reference), its error paths, weight staging, and
the reference's kata-raw-human-nn through boundary 1.  Tolerances are those of test_gpu_nn_parity.py."""
import os
import subprocess

import numpy as np
import pytest

import meta_oracle as mo
from conftest import ROOT
from katago_b200 import KGBError, NeuralNet, modelgen
from test_gpu_net_fp64 import KEYS, _err
from test_gpu_nn_parity import FP16_REL, FP32_TOL, check

pytestmark = pytest.mark.gpu

META_CFGS = ["b2c16_meta", "b2c32nbt_meta", "b1c64nbt_meta"]
SIZES = [(19, 19), (9, 9), (13, 13), (19, 19), (13, 7), (11, 11), (19, 19), (7, 7)]


@pytest.fixture(scope="module")
def metarows():
    d = np.load(os.path.join(ROOT, "tests", "golden", "metarows.npz"))
    return d["rows"], d["names"], d["players"], d["areas"]


def rows_for(metarows, n, seed):
    rows = metarows[0]
    return rows[np.random.default_rng(seed).choice(len(rows), n)].astype(np.float32)


class Net:
    def __init__(self, path, fp16, X=19, Y=19, nhwc=True, max_batch=8):
        self.lm = NeuralNet.loadModelFile(path)
        self.ctx = NeuralNet.createComputeContext([0], X, Y, fp16, self.lm)
        self.h = NeuralNet.createComputeHandle(self.ctx, self.lm, max_batch, False, nhwc, 0)
        self.nhwc = nhwc

    def __call__(self, sp, gl, meta, sym=None, opt=None):
        flat = sp.reshape(sp.shape[0], -1) if self.nhwc else np.ascontiguousarray(sp.transpose(0, 3, 1, 2)).reshape(sp.shape[0], -1)
        return NeuralNet.getOutput(self.h, flat, gl, sym, opt, meta=meta)

    def free(self):
        self.h.free(); self.ctx.free(); self.lm.free()


def _same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in KEYS)


@pytest.mark.parametrize("nhwc", [True, False])
@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("cfg", META_CFGS)
def test_meta_nets_vs_oracle_every_symmetry(golden_dir, metarows, cfg, fp16, nhwc):
    path = os.path.join(golden_dir, "models", f"torchref_{cfg}.bin.gz")
    m = mo.load_meta_model(path)
    n = 8
    sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=5, board_sizes=SIZES)
    meta = rows_for(metarows, n, 6)
    sym = np.arange(8, dtype=np.int32)
    opt = np.linspace(0.0, 1.0, n).astype(np.float32)
    net = Net(path, fp16, nhwc=nhwc)
    check(net(sp, gl, meta, sym, opt), mo.get_output(m, sp, gl, meta, sym, opt), fp16)
    net.free()


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("cfg", META_CFGS)
def test_meta_nets_vs_reference_pytorch_outputs(golden_dir, cfg, fp16):
    d = np.load(os.path.join(golden_dir, f"torchref_{cfg}.npz"))
    sp, gl, meta = d["spatial_nhwc"].astype(np.float32), d["global_"], d["meta"]
    n = sp.shape[0]
    on = sp[..., 0].reshape(n, -1) > 0
    net = Net(os.path.join(golden_dir, "models", f"torchref_{cfg}.bin.gz"), fp16)
    tol = FP16_REL if fp16 else FP32_TOL
    for opt, key in ((0.0, "policy0"), (1.0, "policy_opt")):
        got = net(sp, gl, meta, None, np.full(n, opt, np.float32))
        assert np.abs(got["policy"][:, :361] - d[key][:, :361])[on].max() < tol * (max(1.0, np.abs(d[key][:, :361][on]).max()) if fp16 else 1)
        assert np.abs(got["value"] - d["value"]).max() < tol * (max(1.0, np.abs(d["value"]).max()) if fp16 else 1)
        assert np.abs(got["ownership"] - d["ownership"])[on].max() < tol
    net.free()


def test_b18c384nbt_meta_against_fp64(tmp_path, metarows):
    """The error model of test_gpu_net_fp64.py: the fp32-equivalent mode's error against float64 at most 1/32 of fp16 mode's."""
    path = modelgen.write_model(str(tmp_path / "b18m.bin"), "b18c384nbt", seed=0, meta_channels=384)
    n = 8
    sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=39, board_sizes=[(19, 19), (9, 9), (13, 13), (7, 11)] * 2)
    meta = rows_for(metarows, n, 7)
    sym = (np.arange(n) * 3 + 1) % 8
    m = mo.load_meta_model(path)
    ref64 = mo.get_output(m, sp, gl, meta, sym, dtype=np.float64)
    e_or = _err(mo.get_output(m, sp, gl, meta, sym), ref64)
    errs = []
    for fp16 in (False, True):
        net = Net(path, fp16)
        errs.append(_err(net(sp, gl, meta, sym), ref64))
        net.free()
    e32, e16 = errs
    print(f"b18c384nbt-meta: E32 {e32:.3g}  E16 {e16:.3g}  Eor {e_or:.3g}  E16/E32 {e16 / max(e32, 1e-30):.3g}")
    assert e32 <= e16 / 32, (e32, e16, e_or)


@pytest.mark.parametrize("fp16", [False, True])
def test_ragged_rows_batch_position_and_other_rows(tmp_path, metarows, fp16, monkeypatch):
    path = modelgen.write_model(str(tmp_path / "m.bin"), "mid_nbt", seed=2, meta_channels=96)
    rng = np.random.default_rng(3)
    sizes = [SIZES[i] for i in rng.integers(0, len(SIZES), 256)]
    sp, gl = modelgen.synthetic_inputs(256, 19, 19, seed=4, board_sizes=sizes)
    meta = rows_for(metarows, 256, 8)
    sym = rng.integers(0, 8, 256).astype(np.int32)
    net = Net(path, fp16, max_batch=256)
    monkeypatch.setenv("KGB_RAGGED_ROWS", "0")
    full = Net(path, fp16, max_batch=256)
    monkeypatch.delenv("KGB_RAGGED_ROWS")
    for n in (1, 7, 256):
        a, b = net(sp[:n], gl[:n], meta[:n], sym[:n]), full(sp[:n], gl[:n], meta[:n], sym[:n])
        assert _same(a, b), n
        # row 0 alone, and row 0 among rows of other metadata, in another batch position
        other = rows_for(metarows, n, 100 + n)
        perm = np.roll(np.arange(n), 1)   # row 0 moves to position 1 (n > 1)
        meta2 = other.copy()
        meta2[0] = meta[0]
        c = net(sp[:n][perm], gl[:n][perm], meta2[perm], sym[:n][perm])
        pos = 1 if n > 1 else 0
        for k in KEYS:
            assert np.array_equal(c[k][pos], a[k][0]), (n, k)
    net.free(); full.free()


@pytest.mark.parametrize("fp16", [False, True])
def test_metadata_changes_outputs_and_zero_encoder_matches_its_twin(tmp_path, metarows, fp16):
    meta_path = modelgen.write_model(str(tmp_path / "m.bin"), "tiny_nbt", seed=5, meta_channels=64)
    zero_path = modelgen.write_model(str(tmp_path / "z.bin"), "tiny_nbt", seed=5, meta_channels=64, meta_out_gain=0.0)
    twin_path = modelgen.write_model(str(tmp_path / "t.bin"), "tiny_nbt", seed=5)
    sp, gl = modelgen.synthetic_inputs(5, 19, 19, seed=9, board_sizes=SIZES[:5])
    meta = rows_for(metarows, 5, 9)
    sym = np.array([0, 1, 2, 5, 7], np.int32)
    net = Net(meta_path, fp16)
    a = net(sp, gl, meta)
    meta2 = meta.copy()
    meta2[2] = next(r for r in metarows[0] if not np.array_equal(r, meta[2]))
    b = net(sp, gl, meta2)
    assert not np.array_equal(a["value"][2], b["value"][2]) and not np.array_equal(a["policy"][2], b["policy"][2])
    for i in (0, 1, 3, 4):
        assert all(np.array_equal(a[k][i], b[k][i]) for k in KEYS)
    net.free()
    zero, twin = Net(zero_path, fp16), Net(twin_path, fp16)
    z, t = zero(sp, gl, meta, sym), twin(sp, gl, None, sym)
    assert _same(z, t)
    assert zero.h.launches_per_forward == twin.h.launches_per_forward + 3
    zero.free(); twin.free()


@pytest.mark.parametrize("fp16", [False, True])
def test_staging_a_second_meta_net(tmp_path, metarows, fp16):
    p1 = modelgen.write_model(str(tmp_path / "a.bin"), "tiny_nbt", seed=1, meta_channels=64)
    p2 = modelgen.write_model(str(tmp_path / "b.bin.gz"), "tiny_nbt", seed=2, meta_channels=64)
    plain = modelgen.write_model(str(tmp_path / "p.bin"), "tiny_nbt", seed=3)
    other_width = modelgen.write_model(str(tmp_path / "w.bin"), "tiny_nbt", seed=4, meta_channels=32)
    sp, gl = modelgen.synthetic_inputs(4, 19, 19, seed=12, board_sizes=SIZES[:4])
    meta = rows_for(metarows, 4, 12)
    fresh = Net(p2, fp16)
    want = fresh(sp, gl, meta)
    fresh.free()
    net = Net(p1, fp16)
    net(sp, gl, meta)
    lm2 = NeuralNet.loadModelFile(p2)
    net.h.stage_weights(lm2)
    net.h.commit_weights()
    assert _same(net(sp, gl, meta), want)
    for path in (plain, other_width):
        with pytest.raises(KGBError, match="architecture"):
            net.h.stage_weights(NeuralNet.loadModelFile(path))
    net.free()
    # and the other way: a net without an encoder refuses a metadata net
    pnet = Net(plain, fp16)
    with pytest.raises(KGBError, match="architecture"):
        pnet.h.stage_weights(NeuralNet.loadModelFile(p1))
    pnet.free()


def test_error_paths_leave_the_handle_working(tmp_path, metarows):
    from katago_b200 import SelfPlay
    meta_path = modelgen.write_model(str(tmp_path / "m.bin"), "tiny_nbt", seed=5, meta_channels=64)
    plain_path = modelgen.write_model(str(tmp_path / "p.bin"), "tiny_nbt", seed=5)
    sp, gl = modelgen.synthetic_inputs(3, 19, 19, seed=13)
    meta = rows_for(metarows, 3, 13)
    net, plain = Net(meta_path, True), Net(plain_path, True)
    want, want_plain = net(sp, gl, meta), plain(sp, gl, None)
    with pytest.raises(KGBError, match="kgb_forward: the net has an SGF-metadata encoder.*kgb_forward_meta"):
        net(sp, gl, None)
    with pytest.raises(KGBError, match="metadata rows given for a net without an SGF-metadata encoder"):
        plain(sp, gl, meta)
    with pytest.raises(KGBError, match="SGF-metadata nets need a metadata row per evaluation; the self-play loop has none"):
        SelfPlay(net.h, 2, 8, komi=7.5, seed=1)
    assert _same(net(sp, gl, meta), want) and _same(plain(sp, gl, None), want_plain)
    net.free(); plain.free()


def test_kata_raw_human_nn_through_boundary_1(golden_dir, metarows, tmp_path):
    """The unmodified reference built against integration/b200backend.cpp answers kata-raw-human-nn under humanSLProfile = preaz_5k
    with a metadata net; its outputs agree with the oracle on the reference's own row for that position (preaz_5k, black to move on an
    empty 19x19 board)."""
    exe = os.path.join(ROOT, "oracle", "_ref", "katago_b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/katago_b200 was not built")
    model = os.path.join(golden_dir, "models", "torchref_b2c16_meta.bin.gz")
    cfg = tmp_path / "gtp.cfg"
    cfg.write_text("logDir = %s\nlogToStderr = false\nlogAllGTPCommunication = false\nlogSearchInfo = false\nnumSearchThreads = 1\n"
                   "maxVisits = 1\nnnMaxBatchSize = 8\nnnCacheSizePowerOfTwo = 10\nhumanSLProfile = preaz_5k\nuseFP16 = false\n"
                   "rules = tromp-taylor\n" % (tmp_path / "logs"))
    out = subprocess.run([exe, "gtp", "-config", str(cfg), "-model", model, "-human-model", model],
                         input="boardsize 19\nclear_board\nkata-raw-human-nn 0\nquit\n", capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-3000:]
    resp = out.stdout.split("= ")
    body = [r for r in resp if "policy" in r]
    assert body, out.stdout[-3000:]
    toks = body[0].split()
    vals = {}
    i = 0
    while i < len(toks):
        if toks[i] in ("whiteWin", "whiteLoss", "noResult"):
            vals[toks[i]] = float(toks[i + 1]); i += 2
        else:
            i += 1
    d = dict(zip(zip(metarows[1], metarows[2], metarows[3]), metarows[0]))
    row = d[("preaz_5k", "b", 361)][None].astype(np.float32)
    pos = np.load(os.path.join(golden_dir, "metarows.npz"))
    ref = mo.get_output(mo.load_meta_model(model), pos["position_spatial"][None], pos["position_global"][None], row)
    # NNEvaluator's post-processing (nneval.cpp:1133-1146): under positional superko and area scoring the no-result logit is dropped,
    # win / loss are a two-way softmax, and black to move swaps them into white's view (:1200-1215)
    v = ref["value"][0][:2].astype(np.float64)
    e = np.exp(v - v.max()); e /= e.sum()
    got = np.array([vals["whiteLoss"], vals["whiteWin"]])
    assert vals["noResult"] == 0.0 and np.abs(got - e).max() < 2e-3, (vals, e)
    # and the metadata row matters here: the same position under another profile's row gives other values
    other = mo.get_output(mo.load_meta_model(model), pos["position_spatial"][None], pos["position_global"][None], d[("rank_9d", "b", 361)][None])
    assert np.abs(other["value"] - ref["value"]).max() > 1e-2
