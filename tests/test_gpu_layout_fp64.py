"""Ragged row plans layer by layer, and the evaluator's fp32 head kernels, against float64.

Convolution under a plan.  kgb_test_conv_plan runs the evaluator's own launchPlanRows and launchPackInput for boards given by size
and symmetry (ragged, or every image at the full frame), then one convolution launch.  The float64 reference and its bounds are the
ones of test_gpu_conv_fp64.py, imported: the reference does not depend on the layout, so its bounds carry over unchanged, applied to
the input moved by each image's symmetry.  The hook also fails unless every row below the plan's end that is not a board position
(pad rows and columns, gap rows, the tail up to 128 rows) is exactly zero in raw, hi and lo, and every output row past the plan's end
keeps the NaN bytes it was filled with; operand rows past the plan's end hold a finite sentinel that a board row's tap would pick up.
Each ragged launch is repeated with every image at the full frame: the board positions must hold the same bits.

Head kernels.  kgb_test_head_kernel runs one fp32 kernel on random tensors (row inputs NaN wherever they are not a board position).
Each has a numpy float64 reference of the semantics its comment cites (poolRowsGPool / poolRowsValueHead, addNCBiasInplace +
BatchNormLayer, MatMulLayer, PolicyHead::apply, getOutput) and bounds from an error model:
  sums and dot products in fp32 (the kernels use fmaf chains and tree reductions): C_SUM * K * 2^-24 * sum|terms| for K terms;
  each activation: ACT_LIPSCHITZ * (|scale| * e_x + Z_ROUND * |z|) + formula_error(z), as test_gpu_conv_fp64.py derives them;
  storage: half an fp16 ulp (hi) or the hi + lo split error, allowed in full and kept apart from the computation's bound;
  a value that is copied or counted must be exact.
test_head_bounds_separate_correct_from_broken (no GPU) rehearses every case: a numpy fp32 restatement of the kernel stays within a
quarter of every bound, and each mutant exceeds one at least 8x unless the case cannot show it (named, with the reason).
"""
import numpy as np
import pytest

import kg_nn_oracle as orc
import test_gpu_conv_fp64 as cf
import test_gpu_ragged_rows as rr

F16, F32, F64 = np.float16, np.float32, np.float64
C_SUM = 2.0   # fp32 sums: C_SUM * K * 2^-24 * sum|terms| (a chain of K roundings of at most 2^-24 each, with room for a tree's order)
U = 2.0 ** -24


# ---------------------------------------------------------------------------------------------------------------------------
# The plan, restated
# ---------------------------------------------------------------------------------------------------------------------------
def board_masks(board_xy, sym, X, Y):
    """[n][Y][X] float64: image i's mask, 1 on its top-left board before the symmetry, moved by sym[i] (the convolution's coordinates)."""
    out = np.zeros((len(board_xy), Y, X), F64)
    for i, (bx, by) in enumerate(board_xy):
        m = np.zeros((Y, X), F64)
        m[:by, :bx] = 1.0
        out[i] = orc.apply_symmetry_nhwc(m, int(sym[i]))
    return out


def restate_plan(mask, sym, pad, ragged=True):
    """The row plan of kgb_kernels.cuh for masks [n][Y][X] before symmetry: boxes (x0, y0, w, h) after it, each image's first row (-1
    without rows), each 128-row tile's pitch, and the stats.  Segments by increasing width, images of one width in image order."""
    n, Y, X = mask.shape
    bx = rr.boxes(mask, sym) if ragged else [(0, 0, X, Y)] * n
    base = [-1] * n
    tile_wp, start = [], 0
    for w in range(1, X + 1):
        imgs = [i for i in range(n) if bx[i] is not None and bx[i][2] == w]
        if not imgs:
            continue
        t = 0
        for i in imgs:
            base[i] = start + t
            t += (bx[i][3] + pad) * (w + pad)
        size = (t + pad * (w + pad) + pad + 127) // 128 * 128
        tile_wp += [w + pad] * (size // 128)
        start += size
    boxes_ = [b if b is not None else (0, 0, 0, 0) for b in bx]
    return dict(box=np.array(boxes_, np.int32).reshape(n, 4), base=np.array(base, np.int32), tile_wp=np.array(tile_wp, np.int32),
                stats=dict(rows=start, m_tiles=start // 128, segments=len({b[2] for b in bx if b is not None})))


def rows_conv(x_sym, w, plan, pad):
    """The convolution as the kernel computes it on a plan, in float64: every image's box copied to its rows, and every output row the
    sum over taps (dy, dx) of the row dy * pitch + dx away, with the pitch of the output row's 128-row tile.  Returns the outputs at
    the frame's positions (0 outside the boxes)."""
    n, Y, X, cin = x_sym.shape
    ky = w.shape[0]
    r = ky // 2
    M = plan["stats"]["rows"]
    A = np.zeros((M + 2 * (pad * (X + pad) + pad), cin), F64)   # zero beyond the rows, as the TMA fills it
    for i, (x0, y0, bw, bh) in enumerate(plan["box"]):
        for yy in range(bh):
            row = plan["base"][i] + (yy + pad) * (bw + pad)
            A[row:row + bw] = x_sym[i, y0 + yy, x0:x0 + bw]
    out = np.zeros((M, w.shape[3]), F64)
    for t, p in enumerate(plan["tile_wp"]):
        rows = np.arange(128 * t, 128 * t + 128)
        for dy in range(ky):
            for dx in range(ky):
                src = rows + (dy - r) * p + (dx - r)
                ok = src >= 0
                out[rows[ok]] += A[src[ok]] @ w[dy, dx]
    res = np.zeros((n, Y, X, w.shape[3]), F64)
    for i, (x0, y0, bw, bh) in enumerate(plan["box"]):
        for yy in range(bh):
            row = plan["base"][i] + (yy + pad) * (bw + pad)
            res[i, y0 + yy, x0:x0 + bw] = out[row:row + bw]
    return res


def segment_batch(X, Y, pad, residues):
    """Boards (w, h) of one width per residue, widths increasing, each width's images so many that its segment (rows + gap) ends
    `residue` rows past a multiple of 128: 0 ends exactly on a 128-row boundary, so the next segment's first tap at -pad reads the
    gap's last row; 1 leaves a 127-row tail."""
    boards, w0 = [], 1
    for res in residues:
        found = None
        for w in range(w0 + 1, X + 1):
            for h in range(2, Y + 1):
                for h2 in range(2, Y + 1):
                    for cnt in range(1, 60):
                        t = cnt * (h + pad) * (w + pad) + (h2 + pad) * (w + pad)
                        if (t + pad * (w + pad) + pad) % 128 == res:
                            found = (w, [(w, h)] * cnt + [(w, h2)])
                            break
                    if found:
                        break
                if found:
                    break
            if found:
                break
        assert found, (X, Y, pad, res)
        w0 = found[0]
        boards += found[1]
    return boards


def segment_symmetries(n, n_seg, seed):
    """Symmetries for a batch whose first n_seg images are segment_batch's: flips only there (a transposition would change the
    width of their boxes), all 8 on the others."""
    rng = np.random.default_rng(seed)
    sym = rng.integers(0, 8, n).astype(np.int32)
    sym[:n_seg] %= 4
    sym[n_seg:n_seg + 8] = np.arange(8)[:n - n_seg]
    return sym


def segment_ends(plan, pad):
    """Per segment width: (rows + gap) mod 128."""
    ends = {}
    for i, (x0, y0, w, h) in enumerate(plan["box"]):
        if w:
            ends[w] = ends.get(w, 0) + (h + pad) * (w + pad)
    return {w: (t + pad * (w + pad) + pad) % 128 for w, t in ends.items()}


def test_plan_restatement_on_hand_computed_boxes():
    """Boxes and first rows worked out by hand: a 9x9 board flipped in x sits at x0 = 10; a 13x7 board transposed is 7 wide; an
    empty mask has no rows; the 7-wide segment (one image, 14 x 8 rows + 9 gap rows = 121) rounds up to 128 and the 9-wide one follows."""
    X = Y = 19
    boards = [(9, 9), (9, 9), (13, 7), (0, 0), (9, 5)]
    sym = np.array([0, 2, 4, 0, 1])
    mask = board_masks(boards, np.zeros(5, int), X, Y)
    p = restate_plan(mask, sym, 1)
    assert p["box"].tolist() == [[0, 0, 9, 9], [10, 0, 9, 9], [0, 0, 7, 13], [0, 0, 0, 0], [0, 14, 9, 5]]
    assert p["base"].tolist() == [128, 228, 0, -1, 328]
    assert p["stats"] == dict(rows=512, m_tiles=4, segments=2) == rr.plan_stats(mask, sym, 1)
    assert p["tile_wp"].tolist() == [8, 10, 10, 10]
    frame = restate_plan(mask, sym, 2, ragged=False)
    assert frame["base"].tolist() == [0, 441, 882, 1323, 1764] and frame["stats"] == rr.plan_stats(mask, sym, 2, ragged=False)


@pytest.mark.parametrize("X,Y,pad,residues", [(19, 19, 1, (0, 1, 5)), (19, 19, 2, (0, 1)), (13, 9, 1, (1, 0))])
def test_plan_places_images_where_the_conv_reference_expects(X, Y, pad, residues):
    """The restated plan, convolved row by row as the kernel does (each tile at its own pitch, taps as row shifts), equals the float64
    convolution of the moved inputs at every board position: segments that end exactly on, or one row past, a 128-row boundary, all
    8 symmetries, empty masks and (on 19x19) every width from 2 to 19."""
    boards = segment_batch(X, Y, pad, residues)
    if X == Y == 19:   # every other width, in segments of their own
        used = {b[0] for b in boards}
        boards += [b for b in [(s, s) for s in range(2, 20)] + [(13, 7), (7, 13), (19, 5), (0, 0)] if b[0] not in used and b[1] not in used]
    n = len(boards)
    sym = segment_symmetries(n, len(segment_batch(X, Y, pad, residues)), n + pad)
    rng = np.random.default_rng(n)
    premask = board_masks(boards, np.zeros(n, int), X, Y)
    plan = restate_plan(premask, sym, pad)
    ends = segment_ends(plan, pad)
    for r in residues:
        assert r in ends.values()
    ky = 2 * pad + 1
    w = rng.standard_normal((ky, ky, 8, 4))
    x = rng.standard_normal((n, Y, X, 8)) * premask[..., None]
    xs = np.stack([orc.apply_symmetry_nhwc(x[i], int(sym[i])) for i in range(n)])
    m = board_masks(boards, sym, X, Y)[..., None]
    want = cf.conv64(xs, w) * m
    got = rows_conv(xs, w, plan, pad) * m
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    assert plan["stats"] == rr.plan_stats(premask, sym, pad)


# ---------------------------------------------------------------------------------------------------------------------------
# Convolution under ragged plans (GPU)
# ---------------------------------------------------------------------------------------------------------------------------
def conv_case(cid, ky, cin, cout, kind, fp16, act, batch, X=19, Y=19, ncbias=False, bias=1.0, check_images=None, kernel=None):
    """kernel: the kernel the launcher must take (None: not asserted)."""
    return pytest.param(dict(ky=ky, cin=cin, cout=cout, n=0, X=X, Y=Y, kind=kind, fp16=fp16, act=act, boards=None, ncbias=ncbias, bias=bias,
                             batch=batch, check_images=check_images, kernel=kernel), id=cid)


SIZES = [(s, s) for s in range(2, 20)] + [(13, 7), (7, 13), (19, 5)]


def batch_boards(c):
    """The boards (before symmetry) and symmetries of a case's batch."""
    X, Y, pad = c["X"], c["Y"], max(1, c["ky"] // 2)
    kind = c["batch"]
    if kind == "widths":        # every width 2-19, the three rectangles, empty masks between them; all 8 symmetries
        boards = []
        for k, s in enumerate(SIZES):
            boards.append(s)
            if k % 7 == 3:
                boards.append((0, 0))
    elif kind == "segments":    # one segment ending on a 128-row boundary, one a row past it, then other widths
        boards = segment_batch(X, Y, pad, (0, 1))
        used = {b[0] for b in boards}
        boards += [(s, s) for s in range(2, 20, 3) if s not in used] + [(0, 0)]
        return np.array(boards, np.int32), segment_symmetries(len(boards), len(segment_batch(X, Y, pad, (0, 1))), len(boards))
    elif kind == "rect":        # a 13x9 frame: no transposition
        boards = [(bx, by) for bx in (2, 5, 9, 13) for by in (2, 6, 9)] + [(0, 0), (13, 9)]
    elif kind == "chunks":      # past the planner's 2048-image chunk twice
        sizes = [(s, s) for s in range(2, X + 1)] + [(X, 3), (4, Y), (0, 0)]
        boards = [sizes[(i * 7) % len(sizes)] for i in range(4100)]
    else:
        raise ValueError(kind)
    boards = [(min(bx, X), min(by, Y)) for bx, by in boards]
    rng = np.random.default_rng(len(boards) + X)
    sym = rng.integers(0, 8, len(boards)).astype(np.int32)
    sym[:8] = np.arange(8)
    return np.array(boards, np.int32), sym


def plan_data(c):
    """Inputs of one plan case: test_gpu_conv_fp64's seeded data, with the input zero off the board (as fillRowV7 writes it)."""
    boards, sym = batch_boards(c)
    c = dict(c, n=len(boards))
    d = cf.make_data(c)
    d["board_xy"] = boards
    pre = board_masks(boards, np.zeros(len(boards), int), c["X"], c["Y"])
    d["x"] = (d["x"] * pre[..., None]).astype(F32)
    return c, d, sym


def moved(c, d, sym):
    """The case's inputs in the convolution's coordinates: the input and mask moved by each image's symmetry."""
    xs = np.stack([orc.apply_symmetry_nhwc(d["x"][i], int(sym[i])) for i in range(c["n"])])
    return dict(d, x=xs, mask=board_masks(d["board_xy"], sym, c["X"], c["Y"]))


PLAN_CASES = [
    conv_case("b18-3x3-192-k1-fp16-mish-widths", 3, 192, 192, 1, True, 2, "widths", bias=12.0),
    conv_case("b18-3x3-192-k2-split-identity-widths", 3, 192, 192, 2, False, 0, "widths"),
    conv_case("b18-3x3-192-k3-fp16-silu-segments", 3, 192, 192, 3, True, 3, "segments", bias=12.0),
    conv_case("b18-3x3-192-k4-split-mish-segments", 3, 192, 192, 4, False, 2, "segments", bias=12.0),
    conv_case("b28-3x3-256-k2-fp16-mish-widths", 3, 256, 256, 2, True, 2, "widths", bias=12.0),
    # b18's commonest 3x3 epilogue and its last-block form (kind 5: no raw output) on the epilogue-warpgroup kernel
    conv_case("b18-3x3-192-k2-fp16-mish-widths", 3, 192, 192, 2, True, 2, "widths", bias=12.0, kernel=cf.WG_EPI),
    conv_case("b18-3x3-192-k5-fp16-mish-widths", 3, 192, 192, 5, True, 2, "widths", bias=12.0, kernel=cf.WG_EPI),
    conv_case("1x1-cout64-k0-split-widths", 1, 128, 64, 0, False, 0, "widths"),
    conv_case("1x1-cout384-k3-fp16-relu-widths", 1, 192, 384, 3, True, 1, "widths"),
    conv_case("5x5-initial-k3-split-mish-ncbias-widths", 5, 22, 192, 3, False, 2, "widths", ncbias=True, bias=12.0),
    conv_case("5x5-initial-k3-fp16-mish-ncbias-segments", 5, 22, 192, 3, True, 2, "segments", ncbias=True, bias=12.0),
    conv_case("3x3-cout64-k1-split-silu-13x9", 3, 64, 64, 1, False, 3, "rect", X=13, Y=9, bias=12.0),
    conv_case("1x1-cout256-k2-fp16-mish-13x9", 1, 64, 256, 2, True, 2, "rect", X=13, Y=9, bias=12.0),
    conv_case("1x1-32-64-k2-fp16-mish-b4100", 1, 32, 64, 2, True, 2, "chunks", X=9, Y=9, bias=12.0,
              check_images=(0, 1, 2046, 2047, 2048, 2049, 4094, 4095, 4096, 4097, 4098, 4099)),
    conv_case("3x3-32-64-k1-split-mish-b4100", 3, 32, 64, 1, False, 2, "chunks", X=9, Y=9, bias=12.0,
              check_images=(0, 1, 2046, 2047, 2048, 2049, 4094, 4095, 4096, 4097, 4098, 4099)),
]


def _conv_plan(c, d, sym, ragged):
    from katago_b200 import nn_backend
    return nn_backend.test_conv_plan(c["ky"], c["ky"], c["cin"], c["cout"], d["w"], c["n"], c["X"], c["Y"], c["fp16"], c["kind"], d["x"],
                                     d["board_xy"], sym, ragged, ncbias=d["ncb"], residual=d["res"], bn_scale=d["sc"], bn_bias=d["bi"],
                                     activation=c["act"])


@pytest.mark.parametrize("c", PLAN_CASES)
def test_plan_cases_rehearse(c):
    """test_gpu_conv_fp64's rehearsal on the moved inputs of each plan case (its first 24 images): the emulated kernel within a quarter
    of every bound, and each mutant the case can show beyond 8x (the unmasked-position mutant is test_gpu_conv_fp64's own)."""
    c, d, sym = plan_data(c)
    n = min(c["n"], cf.REHEARSAL_MAX_N)
    d = cf.select_images(d, np.arange(n))
    c = dict(c, n=n)
    dm = moved(c, d, sym[:n])
    ref = cf.reference(c, dm)
    acc = cf.accumulate(c, dm)
    r = cf.check(c, dm, ref, *cf.emulate(c, dm, ref, acc))
    print("correct emulation, worst error / bound:", {k: f"{v:.3g}" for k, v in r.items()})
    assert r and max(r.values()) <= 0.25, r
    for mutant in cf.MUTANTS:
        why = "the mask is moved by the symmetry here" if mutant == "unmasked" else cf._exempt(c, mutant)
        if why:
            print(f"mutant {mutant}: exempt ({why})")
            continue
        rm = cf.check(c, dm, ref, *cf.emulate(c, dm, ref, acc, drop=mutant))
        print(f"mutant {mutant}: worst {max(rm.values()):.3g}x")
        assert max(rm.values()) >= 8.0, (mutant, rm)


@pytest.mark.gpu
@pytest.mark.parametrize("c", PLAN_CASES)
def test_conv_under_ragged_plans(c):
    from katago_b200 import nn_backend
    c, d, sym = plan_data(c)
    raw, hi, lo, stats, plan = _conv_plan(c, d, sym, True)
    if c["kernel"] is not None:
        assert nn_backend.test_last_conv_kernel() == c["kernel"]
    pad = max(1, c["ky"] // 2)
    premask = board_masks(d["board_xy"], np.zeros(c["n"], int), c["X"], c["Y"])
    want = restate_plan(premask, sym, pad)
    assert stats == want["stats"] == rr.plan_stats(premask, sym, pad)
    assert plan[:, :4].tolist() == want["box"].tolist() and plan[:, 4].tolist() == want["base"].tolist()
    if c["batch"] == "segments":
        assert {0, 1} <= set(segment_ends(want, pad).values())
    # every board position: the same bits with every image at the full frame (off the board the frame plan's raw output is v * 0,
    # which may be -0)
    fraw, fhi, flo, fstats, _ = _conv_plan(c, d, sym, False)
    assert fstats == rr.plan_stats(premask, sym, pad, ragged=False)
    dm = moved(c, d, sym)
    on = np.broadcast_to(dm["mask"][..., None] > 0, (c["n"], c["Y"], c["X"], c["cout"]))
    for a, b in ((raw, fraw), (hi, fhi), (lo, flo)):
        if a is not None:
            assert np.isfinite(a).all() and np.isfinite(b).all()
            assert np.array_equal(a[on].view(np.uint32), b[on].view(np.uint32))
    idx = np.array(c["check_images"]) if c["check_images"] else np.arange(c["n"])
    dm = cf.select_images(dm, idx)
    raw, hi, lo = (a[idx] if a is not None else None for a in (raw, hi, lo))
    r = cf.check(c, dm, cf.reference(c, dm), raw, hi, lo)
    print("worst error / bound:", {k: f"{v:.3g}" for k, v in r.items()}, stats)
    assert max(r.values()) <= 1.0, r


# ---------------------------------------------------------------------------------------------------------------------------
# The fused block boundary under ragged plans (GPU)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("inner_c,trunk_c,trunk_fp32,inner_fp32", [
    pytest.param(32, 64, False, False, id="tiny"),
    pytest.param(32, 64, True, True, id="tiny-fp32-all"),
    pytest.param(64, 128, False, False, id="mid"),
    pytest.param(192, 384, False, False, id="b18"),
    pytest.param(192, 384, True, False, id="b18-fp32-trunk"),
])
def test_boundary_under_ragged_plans(inner_c, trunk_c, trunk_fp32, inner_fp32):
    import ctypes as C
    from katago_b200 import load_library
    c = dict(ky=1, X=19, Y=19, batch="widths")
    boards, sym = batch_boards(c)
    boards = np.concatenate([boards, np.array(segment_batch(19, 19, 1, (0, 1)), np.int32)])
    sym = np.concatenate([sym, np.arange(len(boards) - len(sym)) % 4]).astype(np.int32)
    n = len(boards)
    lib = load_library()
    for ragged in (1, 0):
        out, stats = np.zeros(12, np.int64), np.zeros(3, np.int64)
        rc = lib.kgb_test_conv_boundary_plan(inner_c, trunk_c, n, 19, 19, boards.ctypes.data, sym.ctypes.data, ragged, int(trunk_fp32),
                                             int(inner_fp32), C.c_uint32(n + inner_c), out.ctypes.data, stats.ctypes.data)
        assert rc == 0, lib.kgb_last_error()
        premask = board_masks(boards, np.zeros(n, int), 19, 19)
        assert dict(rows=stats[0], m_tiles=stats[1], segments=stats[2]) == rr.plan_stats(premask, sym, 1, ragged=bool(ragged))
        assert out[:3].tolist() == [0, 0, 0], f"elements differing from the two launches (trunk.S, inner.S, inner.A): {out[:3]}"
        assert out[3:6].tolist() == [0, 0, 0], f"nonzero elements in rows that are not board positions / padded channels: {out[3:6]}"
        assert out[6:9].tolist() == [0, 0, 0], f"NaN outputs below the plan's end: {out[6:9]}"
        assert out[9:].tolist() == [0, 0, 0], f"bytes written past the plan's end: {out[9:]}"


# ---------------------------------------------------------------------------------------------------------------------------
# A whole net past the planner's chunk (GPU)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_whole_net_past_the_planner_chunk(tmp_path_factory):
    """tiny_reg at batch 4100 (the planner's 2048-image chunk loop runs three times): ragged rows give the same bits as every image at
    the full frame, and the layout the plan's definition gives."""
    path = rr.model("tiny_reg", tmp_path_factory)
    n = 4100
    sp, gl, sym, opt, mask = rr.mixed_batch(n, seed=41)
    results = {}
    for ragged in (True, False):
        eh = rr.EnvHandle(path, n, {"KGB_RAGGED_ROWS": None if ragged else "0"})
        results[ragged] = eh.forward(sp, gl, sym, opt)
        eh.free()
    (got, stats), (ref, ref_stats) = results[True], results[False]
    rr.assert_same_bits(got, ref, "tiny_reg b4100")
    assert stats == rr.plan_stats(mask, sym, 1)
    assert ref_stats == rr.plan_stats(mask, sym, 1, ragged=False)


# ---------------------------------------------------------------------------------------------------------------------------
# The fp32 head kernels against float64
# ---------------------------------------------------------------------------------------------------------------------------
def head_case(cid, kernel, **kw):
    return pytest.param(dict(kernel=kernel, **kw), id=cid)


HEAD_CASES = [
    head_case("pack-nhwc-split-widths", "pack", X=19, Y=19, pad=1, C=22, split=1, nhwc=1, batch="widths"),
    head_case("pack-nchw-fp16-13x9-pad2", "pack", X=13, Y=9, pad=2, C=22, split=0, nhwc=0, batch="rect"),
    head_case("gpool-mish-fp16raw-widths", "gpool", X=19, Y=19, C=40, act=2, value=0, raw32=0, batch="widths", vals="mixed"),
    head_case("gpool-identity-negative-widths", "gpool", X=19, Y=19, C=40, act=0, value=0, raw32=1, batch="widths", vals="neg"),
    head_case("gpool-identity-below-minus1-widths", "gpool", X=19, Y=19, C=40, act=0, value=0, raw32=1, batch="widths", vals="below"),
    head_case("gpool-full-and-2x2-boards", "gpool", X=19, Y=19, C=40, act=0, value=0, raw32=1, batch="full2", vals="below"),
    head_case("gpool-value-silu-frame", "gpool", X=19, Y=19, C=40, act=3, value=1, raw32=1, batch="widths", vals="mixed", ragged=False),
    head_case("gpool-value-mish-13x9", "gpool", X=13, Y=9, C=72, act=2, value=1, raw32=1, batch="rect", vals="mixed"),
    head_case("biasact-split-ncbias-widths", "bias_act", X=19, Y=19, C=48, act=2, split=1, raw32=1, ncbias=True, batch="widths"),
    head_case("biasact-fp16-relu-fp16raw-13x9", "bias_act", X=13, Y=9, C=100, act=1, split=0, raw32=0, ncbias=True, batch="rect"),
    head_case("matmul-cout160-ldo192-mish", "matmul", cin=120, cout=160, act=2, ldi=128, ldo=192, bias=True),
    head_case("matmul-cout3-ldo4-identity", "matmul", cin=96, cout=3, act=0, ldi=96, ldo=4, bias=False),
    head_case("policy-cp2-2-widths", "policy", X=19, Y=19, C=48, act=2, cp2=2, batch="widths"),
    head_case("policy-cp2-1-13x9", "policy", X=13, Y=9, C=32, act=1, cp2=1, batch="rect"),
    head_case("policy-cp2-2-frame", "policy", X=19, Y=19, C=24, act=3, cp2=2, batch="widths", ragged=False),
    head_case("ownership-widths", "ownership", X=19, Y=19, C=48, act=2, batch="widths"),
    head_case("ownership-13x9", "ownership", X=13, Y=9, C=32, act=0, batch="rect"),
] + [head_case(f"finalize-v{v}-cp2-{cp2}", "finalize", X=9, Y=9, version=v, cp2=cp2) for v, cp2 in ((3, 1), (5, 1), (8, 2), (9, 2), (15, 2))]


def head_boards(c):
    X, Y = c["X"], c["Y"]
    if c.get("batch") == "full2":
        boards = [(X, Y)] * 4 + [(2, 2)] * 4 + [(X, Y), (2, 2)]
    else:
        boards = batch_boards(dict(ky=1, X=X, Y=Y, batch=c["batch"]))[0].tolist()
    rng = np.random.default_rng(len(boards) + X + Y)
    sym = rng.integers(0, 8, len(boards)).astype(np.int32)
    sym[:8] = np.arange(8)
    sym[8:12] = (5, 6, 5, 6)[:len(sym[8:12])]
    return np.array(boards, np.int32), sym


def head_data(c):
    """Seeded tensors of a head case; row tensors [n][Y][X][C] are in the convolution's coordinates, zero off the board."""
    rng = np.random.default_rng(sum(map(ord, str(sorted(c.items())))))
    d = {}
    k = c["kernel"]
    if k in ("matmul", "finalize"):
        n = 24
        d["n"] = n
        if k == "matmul":
            d["in"] = rng.standard_normal((n, c["ldi"])).astype(F32)
            d["W"] = (rng.standard_normal((c["cin"], c["cout"])) / np.sqrt(c["cin"]) * 3).astype(F32)
            d["b"] = rng.standard_normal(c["cout"]).astype(F32) if c["bias"] else None
        else:
            d["pp"] = (4 * rng.standard_normal((n, 4))).astype(F32)
            d["opt"] = rng.uniform(0, 1, n).astype(F32) if c["cp2"] >= 2 else None
            d["value"] = rng.standard_normal((n, 3)).astype(F32)
            d["sv"] = (3 * rng.standard_normal((n, 6))).astype(F32)
        return d
    boards, sym = head_boards(c)
    n, X, Y = len(boards), c["X"], c["Y"]
    d.update(n=n, board_xy=boards, sym=sym)
    m = board_masks(boards, sym, X, Y)
    d["mask"] = m
    if k == "pack":
        pre = board_masks(boards, np.zeros(n, int), X, Y)
        sp = rng.standard_normal((n, Y, X, c["C"])).astype(F32) * pre[..., None].astype(F32)
        sp[..., 0] = pre
        d["sp_nhwc"] = sp
        d["sp"] = sp if c["nhwc"] else np.ascontiguousarray(sp.transpose(0, 3, 1, 2))
        return d
    C = c["C"]
    d["sc"] = (rng.uniform(0.25, 1.5, C) * rng.choice([-1.0, 1.0], C, p=[0.25, 0.75])).astype(F32)
    d["bi"] = (rng.uniform(-1, 1, C) * rng.choice([0.5, 4.0], C)).astype(F32)
    raw = 2.0 * rng.standard_normal((n, Y, X, C))
    vals = c.get("vals", "mixed")
    if vals in ("neg", "below"):   # identity activation: z = raw * 1 + 0 in (-1, -0.05) or in (-6, -1.5)
        d["sc"][:] = 1.0
        d["bi"][:] = 0.0
        raw = -rng.uniform(0.05, 0.95, raw.shape) if vals == "neg" else -rng.uniform(1.5, 6.0, raw.shape)
    d["raw"] = (raw * m[..., None]).astype(F32)
    if k == "bias_act":
        d["ncb"] = rng.standard_normal((n, C)).astype(F32) if c["ncbias"] else None
    if k == "policy":
        d["g1b"] = rng.standard_normal((n, C)).astype(F32)
        d["Wp2"] = (rng.standard_normal((C, c["cp2"])) / np.sqrt(C) * 2).astype(F32)
        d["opt"] = rng.uniform(0, 1, n).astype(F32)
    if k == "ownership":
        d["Wown"] = (rng.standard_normal(C) / np.sqrt(C) * 2).astype(F32)
    return d


def head_gpu(c, d):
    """The kernel's outputs from the hook, and the plan's stats."""
    from katago_b200 import nn_backend
    k, n = c["kernel"], d["n"]
    X, Y = c.get("X", 9), c.get("Y", 9)
    XY = X * Y
    kw = dict(board_xy=d.get("board_xy"), symmetry=d.get("sym"), ragged=c.get("ragged", True), pad=c.get("pad", 1))
    if k == "pack":
        C = c["C"]
        outs, stats, _ = nn_backend.test_head_kernel(k, n, X, Y, [C, c["split"], c["nhwc"]], [d["sp"]],
                                                     [(n, Y, X, C), (n, Y, X, C) if c["split"] else None, (n,), (n, Y, X)], **kw)
        return dict(hi=outs[0], lo=outs[1], mask_sum=outs[2], mask=outs[3]), stats
    if k == "matmul":
        outs, _, _ = nn_backend.test_head_kernel(k, n, X, Y, [c["cin"], c["cout"], c["act"], c["ldi"], c["ldo"]], [d["in"], d["W"], d["b"]],
                                                 [(n, c["ldo"])], **kw)
        return dict(out=outs[0]), None
    if k == "finalize":
        outs, _, _ = nn_backend.test_head_kernel(k, n, X, Y, [c["cp2"], 6, c["version"], 4], [d["pp"], d["opt"], d["value"], d["sv"]],
                                                 [(n, XY + 1), (n, 3), (n, 6)], **kw)
        return dict(policy=outs[0], value=outs[1], score=outs[2]), None
    C = c["C"]
    if k == "gpool":
        c0, ldr = 8, C + 24
        outs, stats, _ = nn_backend.test_head_kernel(k, n, X, Y, [C, c["act"], c["value"], c["raw32"], c0, ldr], [d["raw"], d["sc"], d["bi"]],
                                                     [(n, 3 * C)], **kw)
        return dict(pooled=outs[0]), stats
    if k == "bias_act":
        outs, stats, _ = nn_backend.test_head_kernel(k, n, X, Y, [C, c["act"], c["split"], c["raw32"]], [d["raw"], d["ncb"], d["sc"], d["bi"]],
                                                     [(n, Y, X, C), (n, Y, X, C) if c["split"] else None], **kw)
        return dict(hi=outs[0], lo=outs[1]), stats
    if k == "policy":
        outs, stats, _ = nn_backend.test_head_kernel(k, n, X, Y, [C, c["act"], c["cp2"], 4, C + 4],
                                                     [d["raw"], d["g1b"], d["sc"], d["bi"], d["Wp2"], d["opt"]], [(n, XY + 1)], **kw)
        return dict(policy=outs[0]), stats
    outs, stats, _ = nn_backend.test_head_kernel(k, n, X, Y, [C, c["act"], 0, C], [d["raw"], d["sc"], d["bi"], d["Wown"]], [(n, XY)], **kw)
    return dict(own=outs[0]), stats


# ---- float64 references and bounds -----------------------------------------------------------------------------------------
def _act_err(z, act, e_z):
    """Error of act(z) computed in fp32 from a z that is off by e_z (the fma's own rounding included by Z_ROUND)."""
    return cf.ACT_LIPSCHITZ[act] * (e_z + cf.Z_ROUND * np.abs(z)) + cf.formula_error(z, act)


def _scatter(p, sym, X, Y, inverse=True):
    """[n][Y*X] values at the convolution's positions -> the frame's order (the inverse symmetry; forward for the mutant)."""
    return np.stack([orc.apply_symmetry_nhwc(p[i].reshape(Y, X), int(sym[i]), reverse=inverse).reshape(-1) for i in range(len(p))])


def head_reference(c, d):
    """{output: (float64 value, computation bound, storage bound)}; a bound of 0 asks for the exact value."""
    k = c["kernel"]
    if k == "pack":
        sp = d["sp_nhwc"].astype(F64)
        xs = np.stack([orc.apply_symmetry_nhwc(sp[i], int(d["sym"][i])) for i in range(d["n"])])
        hi = cf._h(xs)
        z = np.zeros_like(hi)
        return dict(hi=(hi, z, z), lo=(cf._h(xs - hi), z, z) if c["split"] else None,
                    mask_sum=(d["mask"].sum(axis=(1, 2)), 0.0, 0.0), mask=(d["mask"], 0.0, 0.0))
    if k == "matmul":
        x, W = d["in"][:, :c["cin"]].astype(F64), d["W"].astype(F64)
        b = d["b"].astype(F64) if d["b"] is not None else 0.0
        v = x @ W + b
        e_v = C_SUM * (c["cin"] + 1) * U * (np.abs(x) @ np.abs(W) + np.abs(b))
        out = np.zeros((d["n"], c["ldo"]))
        pre = np.zeros_like(out)
        out[:, :c["cout"]] = cf.act64(v, c["act"])
        pre[:, :c["cout"]] = _act_err(v, c["act"], e_v)
        return dict(out=(out, pre, U * np.abs(out)))
    if k == "finalize":
        n, XY = d["n"], c["X"] * c["Y"]
        pp = d["pp"].astype(F64)
        opt = d["opt"].astype(F64) if d["opt"] is not None else np.zeros(n)
        pas = pp[:, 0] + (pp[:, 1] - pp[:, 0]) * opt if c["cp2"] >= 2 else pp[:, 0]
        pol = np.full((n, XY + 1), np.nan)
        pol[:, XY] = pas
        pe = np.zeros_like(pol)
        pe[:, XY] = 4 * U * (np.abs(pp[:, 0]) + 2 * np.abs(pp[:, 1] - pp[:, 0]) * opt)
        s = d["sv"].astype(F64)
        v = c["version"]
        score = np.zeros((n, 6))
        if v >= 9:
            score[:] = s
        elif v >= 8:
            score[:, :4] = s[:, :4]
        elif v >= 4:
            score[:, 0], score[:, 1], score[:, 2] = s[:, 0], s[:, 1], s[:, 0]
        else:
            score[:, 0], score[:, 1], score[:, 2] = s[:, 0], s[:, 0] ** 2, s[:, 0]
        se = np.zeros_like(score)
        se[:, 1] = 4 * U * np.abs(score[:, 1]) if v < 4 else 0.0
        return dict(policy=(pol, pe, 0.0), value=(d["value"].astype(F64), 0.0, 0.0), score=(score, se, 0.0))
    m = d["mask"][..., None]
    sc, bi = d["sc"].astype(F64), d["bi"].astype(F64)
    raw = d["raw"].astype(F64)
    if k in ("gpool", "bias_act") and not c["raw32"]:
        raw = cf._h(raw)
    if k in ("gpool", "ownership"):
        z = raw * sc + bi
        e_a = m * _act_err(z, c["act"], 0.0)
        a = m * cf.act64(z, c["act"])
    if k == "gpool":
        n, C = d["n"], c["C"]
        K = c["X"] * c["Y"]
        S = a.sum(axis=(1, 2))
        e_S = C_SUM * K * U * np.abs(a).sum(axis=(1, 2)) + e_a.sum(axis=(1, 2))
        div = d["mask"].sum(axis=(1, 2))[:, None]
        sq = np.sqrt(div)
        with np.errstate(invalid="ignore", divide="ignore"):
            mean = S / div
            e_mean = e_S / div + 2 * U * np.abs(mean)
        t1 = 0.1 * (sq - 14.0)
        out1 = mean * t1
        e1 = np.abs(t1) * e_mean + 0.1 * np.abs(mean) * sq * 2 * U + 4 * U * np.abs(out1)
        if c["value"]:
            t2 = (sq - 14.0) ** 2 * 0.01 - 0.1
            out2 = mean * t2
            # t2 cancels near sqrt(area) = 14 - sqrt(10) (a 13x9 board): its error is absolute, of the size of its terms
            e_t2 = 0.02 * np.abs(sq - 14.0) * sq * U + 4 * U * ((sq - 14.0) ** 2 * 0.01 + 0.1)
            e2 = np.abs(t2) * e_mean + np.abs(mean) * e_t2 + 2 * U * np.abs(out2)
        else:
            out2 = np.maximum(-1.0, (a + (m - 1.0)).max(axis=(1, 2)))
            e2 = np.where(out2 > -1.0, e_a.max(axis=(1, 2)), 0.0)
        val = np.concatenate([mean, out1, out2], axis=1)
        pre = np.concatenate([e_mean, e1, e2], axis=1)
        return dict(pooled=(val, pre, U * np.abs(val)))
    if k == "bias_act":
        nb = d["ncb"].astype(F64)[:, None, None, :] if d["ncb"] is not None else 0.0
        x = raw + nb
        z = x * sc + bi
        e_x = C_SUM * U * (np.abs(raw) + np.abs(nb))
        act = m * cf.act64(z, c["act"])
        e_a = m * _act_err(z, c["act"], np.abs(sc) * e_x)
        return dict(act=(act, e_a, m * cf.store_error((np.abs(act) + e_a) * (1 + 2.0 ** -9), not c["split"])), lo=cf._h(act - cf._h(act)))
    if k == "policy":
        g = d["g1b"].astype(F64)[:, None, None, :]
        z = (raw + g) * sc + bi
        h = m * cf.act64(z, c["act"])
        e_h = m * _act_err(z, c["act"], np.abs(sc) * U * (np.abs(raw) + np.abs(g)))
        W = d["Wp2"].astype(F64)
        L = h @ W
        e_L = np.abs(e_h) @ np.abs(W) + C_SUM * c["C"] * U * (np.abs(h) @ np.abs(W))
        opt = d["opt"].astype(F64)[:, None, None]
        if c["cp2"] >= 2:
            p = L[..., 0] + (L[..., 1] - L[..., 0]) * opt
            e_p = e_L[..., 0] * (1 + opt) + e_L[..., 1] * opt + 4 * U * (np.abs(L[..., 0]) + 2 * np.abs(L[..., 1] - L[..., 0]) * opt)
        else:
            p, e_p = L[..., 0], e_L[..., 0]
        n, X, Y = d["n"], c["X"], c["Y"]
        pol = np.full((n, X * Y + 1), np.nan)
        pre = np.zeros_like(pol)
        pol[:, :-1] = _scatter(p.reshape(n, -1), d["sym"], X, Y)
        pre[:, :-1] = _scatter(e_p.reshape(n, -1), d["sym"], X, Y)
        return dict(policy=(pol, pre, 0.0), _conv=p)
    # ownership
    W = d["Wown"].astype(F64)
    o = a @ W
    e_o = np.abs(e_a) @ np.abs(W) + C_SUM * c["C"] * U * (np.abs(a) @ np.abs(W))
    n, X, Y = d["n"], c["X"], c["Y"]
    return dict(own=(_scatter(o.reshape(n, -1), d["sym"], X, Y), _scatter(e_o.reshape(n, -1), d["sym"], X, Y), 0.0), _conv=o)


def head_ratios(c, d, ref, got):
    """Worst (|error| - storage) / computation bound per output; NaN where the kernel must not write is required, NaN elsewhere fails."""
    out = {}
    for name, g in got.items():
        if g is None or ref.get(name) is None:
            continue
        if c["kernel"] == "bias_act" and name in ("hi", "lo"):
            continue
        val, pre, store = ref[name]
        g = g.astype(F64)
        unwritten = np.isnan(val)
        if not np.array_equal(np.isnan(g), unwritten):
            out[name] = np.inf
            continue
        out[name] = cf._ratio(np.where(unwritten, 0.0, g - val), (np.broadcast_to(pre, val.shape), np.broadcast_to(store, val.shape)))
    if c["kernel"] == "bias_act":
        hi = got["hi"].astype(F64)
        lo = got["lo"].astype(F64) if got["lo"] is not None else 0.0
        val, pre, store = ref["act"]
        out["act"] = cf._ratio(hi + lo - val, (pre, store)) if np.isfinite(hi + lo).all() else np.inf
        if c["split"]:
            on = np.broadcast_to(d["mask"][..., None] > 0, val.shape)
            out["lo"] = cf._projection(hi + lo - val, ref["lo"], 1.0, on)
    return out


# ---- fp32 restatements of the kernels, and their mutants -------------------------------------------------------------------
def _act32(z, act):
    return cf.act64(z.astype(F64), act).astype(F32)


def head_emulate(c, d, mutant=None):
    """The kernel in numpy fp32 (sums pairwise or sequential, activations accurate, fp32 rounding after every operation)."""
    k = c["kernel"]
    if k == "pack":
        n = d["n"]
        xs = np.stack([orc.apply_symmetry_nhwc(d["sp_nhwc"][i], int(d["sym"][i])) for i in range(n)])
        hi = xs.astype(F16).astype(F32)
        lo = (xs - hi).astype(F16).astype(F32) if c["split"] else None
        ms = d["mask"].sum(axis=(1, 2)).astype(F32)
        if mutant == "mask-sum-frame":
            ms = np.full(n, c["X"] * c["Y"], F32)
        return dict(hi=hi, lo=lo, mask_sum=ms, mask=d["mask"].astype(F32))
    if k == "matmul":
        v = d["in"][:, :c["cin"]] @ d["W"]
        if d["b"] is not None:
            v = (v + d["b"]).astype(F32)
        out = np.zeros((d["n"], c["ldo"]), F32)
        out[:, :c["cout"]] = _act32(v, c["act"])
        if mutant == "matmul-padding-unwritten":
            out[:, c["cout"]:] = np.nan
        return dict(out=out)
    if k == "finalize":
        n, XY = d["n"], c["X"] * c["Y"]
        pp = d["pp"]
        opt = d["opt"] if d["opt"] is not None else np.zeros(n, F32)
        if mutant == "optimism-neighbour":
            opt = np.roll(opt, 1)
        pas = (pp[:, 0] + ((pp[:, 1] - pp[:, 0]).astype(F32) * opt).astype(F32)).astype(F32) if c["cp2"] >= 2 else pp[:, 0]
        pol = np.full((n, XY + 1), np.nan, F32)
        pol[:, XY] = pas
        v = 9 if mutant == "version-8-as-9" and c["version"] == 8 else c["version"]
        s = d["sv"]
        score = np.zeros((n, 6), F32)
        if v >= 9:
            score[:] = s
        elif v >= 8:
            score[:, :4] = s[:, :4]
        elif v >= 4:
            score[:, 0], score[:, 1], score[:, 2] = s[:, 0], s[:, 1], s[:, 0]
        else:
            score[:, 0], score[:, 1], score[:, 2] = s[:, 0], (s[:, 0] * s[:, 0]).astype(F32), s[:, 0]
        return dict(policy=pol, value=d["value"].copy(), score=score)
    m = d["mask"][..., None].astype(F32)
    raw = d["raw"] if k not in ("gpool", "bias_act") or c["raw32"] else d["raw"].astype(F16).astype(F32)
    n, X, Y = d["n"], c["X"], c["Y"]
    if k in ("gpool", "ownership"):
        a = m * _act32((raw * d["sc"] + d["bi"]).astype(F32), c["act"])
    if k == "gpool":
        S = a.sum(axis=(1, 2), dtype=F32)
        div = d["mask"].sum(axis=(1, 2)).astype(F32)[:, None]
        if mutant == "mask-sum-frame":
            div = np.full_like(div, X * Y)
        sq = np.sqrt(div)
        mean = (S / div).astype(F32)
        out1 = (mean * (sq - F32(14)) * F32(0.1)).astype(F32)
        if c["value"]:
            out2 = (mean * ((sq - F32(14)) * (sq - F32(14)) * F32(0.01) - F32(0.1))).astype(F32)
        elif mutant == "gpool-max-without-mask":
            out2 = np.maximum(F32(-1), a.max(axis=(1, 2)))
        else:
            out2 = np.maximum(F32(-1), (a + (m - 1)).max(axis=(1, 2)))
        return dict(pooled=np.concatenate([mean, out1, out2], axis=1))
    if k == "bias_act":
        ncb = d["ncb"]
        if ncb is not None and mutant == "ncbias-neighbour":
            ncb = np.roll(ncb, 1, axis=0)
        x = (raw + ncb[:, None, None, :]).astype(F32) if ncb is not None else raw
        a = m * _act32((x.astype(F64) * d["sc"] + d["bi"]).astype(F32), c["act"])
        hi = a.astype(F16).astype(F32)
        lo = (a.astype(F64) - hi).astype(F16).astype(F32) if c["split"] else None
        if lo is not None and mutant == "act-lo":
            lo = np.zeros_like(lo)
        return dict(hi=hi, lo=lo)
    if k == "policy":
        z = (((raw + d["g1b"][:, None, None, :]).astype(F32)).astype(F64) * d["sc"] + d["bi"]).astype(F32)
        h = m * _act32(z, c["act"])
        L = (h @ d["Wp2"]).astype(F32)
        opt = np.roll(d["opt"], 1) if mutant == "optimism-neighbour" else d["opt"]
        p = (L[..., 0] + (L[..., 1] - L[..., 0]) * opt[:, None, None]).astype(F32) if c["cp2"] >= 2 else L[..., 0]
        pol = np.full((n, X * Y + 1), np.nan, F32)
        pol[:, :-1] = _scatter(p.reshape(n, -1), d["sym"], X, Y, inverse=mutant != "forward-symmetry")
        return dict(policy=pol)
    o = (a @ d["Wown"]).astype(F32)
    return dict(own=_scatter(o.reshape(n, -1), d["sym"], X, Y, inverse=mutant != "forward-symmetry").astype(F32))


HEAD_MUTANTS = {"pack": ("mask-sum-frame",), "gpool": ("gpool-max-without-mask", "mask-sum-frame"), "bias_act": ("ncbias-neighbour", "act-lo"),
                "matmul": ("matmul-padding-unwritten",), "policy": ("forward-symmetry", "optimism-neighbour"), "ownership": ("forward-symmetry",),
                "finalize": ("version-8-as-9", "optimism-neighbour")}


def head_exempt(c, d, mutant):
    """Why this case cannot show `mutant`, or None."""
    k = c["kernel"]
    if k not in ("matmul", "finalize"):
        on = d["mask"].reshape(d["n"], -1) > 0
        full = bool(on[on.any(axis=1)].all())
    else:
        full = False
    if mutant == "mask-sum-frame" and full:
        return "every non-empty board fills the frame"
    if mutant == "gpool-max-without-mask":
        if c["value"]:
            return "the value head has no max term"
        if c.get("vals") not in ("neg",):
            return "the values are not all in (-1, 0): off-board 0 (mixed) or -1 (below -1) is not above the board's max"
    if mutant == "forward-symmetry" and c["X"] != c["Y"]:
        return "a rectangular frame has no transposition: every symmetry is its own inverse"
    if mutant == "act-lo" and not c["split"]:
        return "fp16 mode has no lo half"
    if mutant == "ncbias-neighbour" and d.get("ncb") is None:
        return "no ncbias"
    if mutant == "optimism-neighbour" and c["cp2"] < 2:
        return "one policy channel: no optimism blend"
    if mutant == "version-8-as-9" and c["version"] != 8:
        return "not a version 8 net"
    return None


@pytest.mark.parametrize("c", HEAD_CASES)
def test_head_bounds_separate_correct_from_broken(c):
    d = head_data(c)
    ref = head_reference(c, d)
    r = head_ratios(c, d, ref, head_emulate(c, d))
    print("correct emulation, worst error / bound:", {k: f"{v:.3g}" for k, v in r.items()})
    assert r and max(r.values()) <= 0.25, r
    for mutant in HEAD_MUTANTS[c["kernel"]]:
        why = head_exempt(c, d, mutant)
        if why:
            print(f"mutant {mutant}: exempt ({why})")
            continue
        rm = head_ratios(c, d, ref, head_emulate(c, d, mutant))
        print(f"mutant {mutant}: worst {max(rm.values()):.3g}x")
        assert max(rm.values()) >= 8.0, (mutant, rm)


@pytest.mark.gpu
@pytest.mark.parametrize("c", HEAD_CASES)
def test_head_kernel_against_fp64(c):
    d = head_data(c)
    got, stats = head_gpu(c, d)
    if stats is not None:
        pad = c.get("pad", 1)
        premask = board_masks(d["board_xy"], np.zeros(d["n"], int), c["X"], c["Y"])
        assert stats == rr.plan_stats(premask, d["sym"], pad, ragged=c.get("ragged", True))
    r = head_ratios(c, d, head_reference(c, d), got)
    print("worst error / bound:", {k: f"{v:.3g}" for k, v in r.items()})
    assert r and max(r.values()) <= 1.0, r
