"""The fused nested-block boundary (kgb_conv_pair_kernel, kgb_conv_pair_epi_kernel) against float64, on caller data.

The boundary is a block's exit 1x1 (inner -> trunk channels, + the trunk stream S, the trunk BN and mish) and the next block's entry
1x1 (trunk -> inner channels, the inner BN and mish), with the activated trunk operand T between them kept inside the kernel.  The
error model is test_gpu_conv_fp64.py's, imported, with no new constant:

  exit:  a kind-2 1x1 layer (kind 4 with an fp32 trunk stream), cin = inner, cout = trunk, operand the inner operand A.  Its raw
         output is the trunk stream the kernel returns, checked against the same bounds as that module's layers.
  T:     never leaves the kernel, so it is not checked itself.  Its error is the exit's act bound, computation plus fp16 storage:
             e_T = act bound of the exit (computation) + half an fp16 ulp at |T| + e (storage)
  entry: a kind-3 1x1 layer, cin = trunk, cout = inner, whose reference takes the exact float64 T of the exit's reference.  The
         kernel's operand is off by at most e_T per channel, so its accumulator is off by at most conv(e_T, |w2h|) on top of its own
         accumulation term for K = trunk channels, and the activation by that times ACT_LIPSCHITZ |bn_scale|.  As everywhere in
         that module, a rounding to a stored dtype has no margin to give: conv(storage part of e_T, |w2h|) joins the storage term in
         full (s_operand in bounds()), and conv(computation part of e_T, |w2h|) the computation term (e_operand).  The total bound
         is the same; the split only decides what the reported ratio measures.  (Summed as a worst case, the storage part is tight
         only when every rounding of T leans the same way against the sign of its weight; over a million outputs the largest
         actual sum reaches 0.3-0.6 of it at K = 64-384, which would leave no room for the accumulation's margin.)

test_boundary_bounds_separate_correct_from_broken (no GPU) rehearses every case: the emulated kernel (accumulate() and the fp32
epilogue for the exit, fp16 T, then the same for the entry) must stay within a quarter of every bound, and each mutant must exceed a
bound at least 8x: one 32-column chunk of T missing from the entry; two chunks' T slots swapped; chunk 0 of each 128-row tile taken
from the previous tile's rows (the early hand-over of the next tile's chunk 0); the exit's residual read from the neighbouring
32-column slice; an off-board row left unmasked in both epilogues.  Cases of more than 24 images are rehearsed on 24 images.

Each GPU case asserts the kernel the launcher took, and the hook fails unless every masked row and padded channel of every output is
exactly zero (and, under a plan, nothing past the plan's end was written).
"""
import numpy as np
import pytest

import test_gpu_conv_fp64 as cf
import test_gpu_layout_fp64 as lf

F16, F32, F64 = np.float16, np.float32, np.float64
PAIR, PAIR_EPI, WG = "kgb_conv_pair_kernel", "kgb_conv_pair_epi_kernel", "kgb_conv_wg_kernel"


def _case(cid, inner, trunk, n, kernel, boards=None, trunk_fp32=False, inner_fp32=False, fused=True, env=None, check_images=None,
          plan=None):
    """plan: None for the frame layout, else a batch of test_gpu_layout_fp64.batch_boards ("widths": every width, all 8 symmetries)."""
    return pytest.param(dict(inner=inner, trunk=trunk, n=n, X=19, Y=19, kernel=kernel, boards=boards, trunk_fp32=trunk_fp32,
                             inner_fp32=inner_fp32, fused=fused, env=env or {}, check_images=check_images, plan=plan), id=cid)


MIXED = cf.MIXED
# a 19x19 image is 400 rows of the frame layout: 8 images are 25 tiles, 43 are 135 (the H100 has 132 SMs), 256 are 800, and at 1021
# the last tile is partial
CASES = [
    _case("b18-fp16-b8", 192, 384, 8, PAIR_EPI),
    _case("b18-fp16-b43-mixed", 192, 384, 43, PAIR_EPI, boards=MIXED),
    _case("b18-fp16-b256", 192, 384, 256, PAIR_EPI),
    _case("b18-fp16-b1021", 192, 384, 1021, PAIR_EPI, check_images=(0, 1, 330, 331, 660, 661, 1019, 1020)),
    _case("b18-fp16-ragged-widths", 192, 384, 0, PAIR_EPI, plan="widths"),
    _case("b18-fp16-b43-no-pair-epilogue-wg", 192, 384, 43, PAIR, boards=MIXED, env={"KGB_PAIR_EPILOGUE_WG": "0"}),
    _case("b18-fp32-trunk-b43", 192, 384, 43, PAIR, trunk_fp32=True),
    _case("b18-fp32-streams-b43-mixed", 192, 384, 43, PAIR, boards=MIXED, trunk_fp32=True, inner_fp32=True),
    _case("b18-fp16-b43-two-launches", 192, 384, 43, WG, fused=False),
    _case("mid-64-128-fp16-b43-mixed", 64, 128, 43, PAIR, boards=MIXED),
    # 32 inner channels padded to 64: the tile is (64, 64), and the inner outputs' channels 32-63 must stay zero
    _case("tiny-32-64-fp16-b43-mixed", 32, 64, 43, PAIR, boards=MIXED),
]


# ---- data ---------------------------------------------------------------------------------------------------------------------------

def case_batch(c):
    """(c with n set, boards [n][2], symmetries [n] or None, mask after the symmetry [n][Y][X])."""
    if c["plan"] is not None:
        boards, sym = lf.batch_boards(dict(ky=1, X=c["X"], Y=c["Y"], batch=c["plan"]))
        c = dict(c, n=len(boards))
        return c, boards, sym, lf.board_masks(boards, sym, c["X"], c["Y"])
    b = c["boards"] or ((c["X"], c["Y"]),)
    boards = np.array([b[i % len(b)] for i in range(c["n"])], np.int32)
    return c, boards, None, lf.board_masks(boards, np.zeros(c["n"], int), c["X"], c["Y"])


def make_data(c):
    """Seeded inputs, zero off the board (the hook reads board positions only).  The exit as a test_gpu_conv_fp64 layer (cin inner,
    cout trunk) and the entry's weights and BN constants."""
    c, boards, sym, mask = case_batch(c)
    n, X, Y, N2, N1 = c["n"], c["X"], c["Y"], c["inner"], c["trunk"]
    rng = np.random.default_rng([N2, N1, n, int(c["trunk_fp32"]), int(c["inner_fp32"])])
    m = mask[..., None].astype(F32)

    def bn(k):
        sc = (rng.uniform(0.25, 1.5, k) * rng.choice([-1.0, 1.0], k, p=[0.25, 0.75])).astype(F32)
        return sc, (rng.uniform(-1.0, 1.0, k) * rng.choice([0.5, 4.0, 12.0], k)).astype(F32)

    d = dict(w=(rng.standard_normal((1, 1, N2, N1)) / np.sqrt(N2)).astype(F32),
             x=rng.standard_normal((n, Y, X, N2), dtype=F32) * m,
             res=4.0 * rng.standard_normal((n, Y, X, N1), dtype=F32) * m, ncb=None, board_xy=boards, mask=mask)
    d["sc"], d["bi"] = bn(N1)
    d["w2"] = (rng.standard_normal((1, 1, N1, N2)) / np.sqrt(N1)).astype(F32)
    d["sc2"], d["bi2"] = bn(N2)
    return c, d, sym


def exit_case(c):
    return dict(ky=1, cin=c["inner"], cout=c["trunk"], n=c["n"], X=c["X"], Y=c["Y"], kind=4 if c["trunk_fp32"] else 2, fp16=True, act=2,
                boards=c["boards"], ncbias=False)


def entry_case(c):
    return dict(ky=1, cin=c["trunk"], cout=c["inner"], n=c["n"], X=c["X"], Y=c["Y"], kind=3, fp16=True, act=2, boards=c["boards"],
                ncbias=False, raw32=c["inner_fp32"])


def entry_data(d, T):
    return dict(d, w=d["w2"], x=T, res=None, sc=d["sc2"], bi=d["bi2"])


# ---- float64 reference and bounds ---------------------------------------------------------------------------------------------------

def reference(c, d):
    """The exit's and the entry's references and bounds: (c1, d1, ref1, bounds1, c2, d2, ref2, bounds2)."""
    c1, c2 = exit_case(c), entry_case(c)
    ref1 = cf.reference(c1, d)
    b1 = cf.bounds(c1, d, ref1)
    T = ref1["act"]   # the exact activated trunk operand
    (e_T, s_T) = b1[1]   # its computation and storage bounds
    d2 = entry_data(d, T)
    wh = cf._h(d["w2"])
    ideal = cf.conv64(T, wh)
    w64 = d["w2"].astype(F64)
    m = d["mask"][..., None]
    z = ideal * d["sc2"].astype(F64) + d["bi2"].astype(F64)
    act = m * cf.act64(z, 2)
    ref2 = dict(ideal=ideal, terms={}, sigma=np.sqrt(cf.conv64(T * T, w64 * w64)), sum_abs=np.abs(ideal), V=ideal, raw=m * ideal, z=z,
                act=act, lo=cf._h(act - cf._h(act)), mask=m, e_operand=cf.conv64(e_T, np.abs(wh)),
                s_operand=cf.conv64(s_T, np.abs(wh)))
    return c1, d, ref1, b1, c2, d2, ref2, cf.bounds(c2, d2, ref2)


def ratios(refs, trunk_s, inner_s, inner_a):
    """Worst error / bound of each output (> 1 fails)."""
    c1, d1, ref1, b1, c2, d2, ref2, b2 = refs
    return {"trunk.S": cf._ratio(trunk_s.astype(F64) - ref1["raw"], b1[0]),
            "inner.S": cf._ratio(inner_s.astype(F64) - ref2["raw"], b2[0]),
            "inner.A": cf._ratio(inner_a.astype(F64) - ref2["act"], b2[1])}


# ---- emulation (no GPU) and mutants ---------------------------------------------------------------------------------------------------

def frame_rows(a, X, Y):
    """NHWC -> the frame layout's rows (image i at row 400 i for 19x19: (Y + 1) x (X + 1) rows, the pad rows and columns zero)."""
    n = a.shape[0]
    r = np.zeros((n, Y + 1, X + 1) + a.shape[3:], a.dtype)
    r[:, 1:, :X] = a
    return r.reshape((-1,) + a.shape[3:])


def from_frame_rows(r, n, X, Y):
    return r.reshape((n, Y + 1, X + 1) + r.shape[1:])[:, 1:, :X]


def emulate(c, refs, mutant=None):
    """The kernel: the exit's accumulation and fp32 epilogue, T in fp16, then the entry's; `mutant` applied on the way."""
    c1, d1, ref1, b1, c2, d2, ref2, b2 = refs
    acc1 = cf.accumulate(c1, d1)
    s_out, T, _ = cf.emulate(c1, d1, ref1, acc1, drop={"exit-residual-neighbour-slice": "residual-neighbour-slice",
                                                       "unmasked": "unmasked"}.get(mutant))
    T = T.astype(F64)
    if mutant == "T-chunk-missing":
        T[..., 32:64] = 0.0
    elif mutant == "T-chunks-swapped":
        T[..., 0:64] = np.concatenate([T[..., 32:64], T[..., 0:32]], axis=-1)
    elif mutant == "chunk0-previous-tile":
        rows = frame_rows(T, c["X"], c["Y"])
        rows[:, :32] = np.roll(rows[:, :32], 128, axis=0)
        T = from_frame_rows(rows, T.shape[0], c["X"], c["Y"]).copy()
    de = dict(d2, x=T)
    acc2 = cf.accumulate(c2, de)
    i_s, i_a, _ = cf.emulate(c2, de, ref2, acc2, drop="unmasked" if mutant == "unmasked" else None)
    return s_out, i_s, i_a


MUTANTS = ("T-chunk-missing", "T-chunks-swapped", "chunk0-previous-tile", "exit-residual-neighbour-slice", "unmasked")


def _exempt(c, d, mutant):
    if mutant == "unmasked" and c["plan"] is not None:
        return "the mask is moved by the symmetry here"
    if mutant == "unmasked" and not any(b[0] < c["X"] or b[1] < c["Y"] for b in d["board_xy"]):
        return "every image covers the whole frame"
    return None


@pytest.mark.parametrize("c", CASES)
def test_boundary_bounds_separate_correct_from_broken(c):
    c, d, sym = make_data(dict(c, n=min(c["n"], cf.REHEARSAL_MAX_N)) if c["plan"] is None else c)
    if c["n"] > cf.REHEARSAL_MAX_N:
        d = cf.select_images(d, np.arange(cf.REHEARSAL_MAX_N))
        c = dict(c, n=cf.REHEARSAL_MAX_N)
    refs = reference(c, d)
    r = ratios(refs, *emulate(c, refs))
    print("correct emulation, worst error / bound:", {k: f"{v:.3g}" for k, v in r.items()})
    assert max(r.values()) <= 0.25, r
    tried = 0
    for mutant in MUTANTS:
        if _exempt(c, d, mutant):
            continue
        tried += 1
        rm = ratios(refs, *emulate(c, refs, mutant))
        print(f"mutant {mutant}: worst {max(rm.values()):.3g}x")
        assert max(rm.values()) >= 8.0, (mutant, rm)
    assert tried >= 4


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES)
def test_boundary_against_fp64(c, monkeypatch):
    from katago_b200 import nn_backend
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    c, d, sym = make_data(c)
    s_out, i_s, i_a, layout = nn_backend.test_conv_boundary_ex(
        c["inner"], c["trunk"], c["n"], c["X"], c["Y"], d["x"], d["w"][0, 0], d["res"], d["sc"], d["bi"], d["w2"][0, 0], d["sc2"], d["bi2"],
        board_xy=d["board_xy"], symmetry=sym, ragged=None if c["plan"] is None else True, trunk_fp32=c["trunk_fp32"],
        inner_fp32=c["inner_fp32"], fused=c["fused"])
    assert nn_backend.test_last_conv_kernel() == c["kernel"]
    if layout is not None:
        premask = lf.board_masks(d["board_xy"], np.zeros(c["n"], int), c["X"], c["Y"])
        assert layout == lf.rr.plan_stats(premask, sym, 1)
    if c["check_images"] is not None:
        idx = np.array(c["check_images"])
        d = cf.select_images(d, idx)
        s_out, i_s, i_a = s_out[idx], i_s[idx], i_a[idx]
        c = dict(c, n=len(idx))
    r = ratios(reference(c, d), s_out, i_s, i_a)
    print("worst error / bound:", {k: f"{v:.3g}" for k, v in r.items()})
    assert max(r.values()) <= 1.0, r
