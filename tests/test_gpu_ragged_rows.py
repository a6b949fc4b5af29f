"""Ragged rows: every image is laid out at the size of its own board (the bounding box of its mask after its symmetry), in segments
of one row pitch, instead of at the evaluator's full frame.  The outputs must be the same bits as with every image at the full frame
(KGB_RAGGED_ROWS=0, the reference plan), the layout must be the one the plan's definition gives for the inputs, nothing may carry over
from one forward's layout to the next, and the device self-play loop must play the same games move for move.
"""
import os

import numpy as np
import pytest

from katago_b200 import NeuralNet, SelfPlay, modelgen

FRAME = 19
OUTPUTS = ("policy", "value", "score_value", "ownership")
G170 = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "models", "g170-b6c96-s175395328-d26788732.bin.gz")


# ---------------------------------------------------------------------------------------------------------------------------
# The plan, restated: what layout_stats() must report for a batch
# ---------------------------------------------------------------------------------------------------------------------------
def sym_index(y, x, H, W, sym):
    """SymmetryHelpers' destination index of source (y, x) in a frame of pitch W (packInputKernel's symIndex, forward direction)."""
    transpose = (sym & 4) != 0 and H == W
    flip_x, flip_y = (sym & 2) != 0, (sym & 1) != 0
    if transpose:
        flip_x, flip_y = flip_y, flip_x
    hs, ws, hb, wb = W, 1, 0, 0
    if flip_y:
        hb, hs = (H - 1) * hs, -hs
    if flip_x:
        wb, ws = (W - 1) * ws, -ws
    if transpose:
        hs, ws = ws, hs
    return hb + y * hs + wb + x * ws


def boxes(mask, sym):
    """[n] (x0, y0, w, h) of the non-zero positions of mask[n][Y][X] once symmetry sym[n] has moved them; None for an empty mask."""
    n, Y, X = mask.shape
    out = []
    for i in range(n):
        ys, xs = np.nonzero(mask[i])
        if len(ys) == 0:
            out.append(None)
            continue
        d = sym_index(ys, xs, Y, X, int(sym[i]))
        yd, xd = d // X, d % X
        out.append((int(xd.min()), int(yd.min()), int(xd.max() - xd.min() + 1), int(yd.max() - yd.min() + 1)))
    return out


def plan_stats(mask, sym, pad, ragged=True):
    """Rows, 128-row tiles and segments: per box width one segment of its images' (h+pad)(w+pad) rows, the pad*(w+pad)+pad gap rows
    that end it, rounded up to 128 rows.  The reference plan puts every image at the full frame."""
    n, Y, X = mask.shape
    per_width = {}
    for b in (boxes(mask, sym) if ragged else [(0, 0, X, Y)] * n):
        if b is not None:
            per_width[b[2]] = per_width.get(b[2], 0) + (b[3] + pad) * (b[2] + pad)
    rows = sum((t + pad * (w + pad) + pad + 127) // 128 * 128 for w, t in per_width.items())
    return dict(rows=rows, m_tiles=rows // 128, segments=len(per_width))


def test_plan_restatement_on_known_boxes():
    """The restatement the GPU tests compare layout_stats() with: a flipped 9x9 board sits in the frame's right columns, a transposed 13x7
    board is 7 wide, an empty mask has no rows, and the reference plan is the frame layout plus one gap and one alignment tail."""
    m = np.zeros((4, FRAME, FRAME), np.float32)
    m[0, :9, :9] = 1
    m[1, :9, :9] = 1
    m[2, :7, :13] = 1
    sym = np.array([0, 2, 4, 0])
    assert boxes(m, sym) == [(0, 0, 9, 9), (10, 0, 9, 9), (0, 0, 7, 13), None]
    assert plan_stats(m, sym, 1) == dict(rows=256 + 128, m_tiles=3, segments=2)
    assert plan_stats(m, sym, 1, ragged=False) == dict(rows=(4 * 400 + 21 + 127) // 128 * 128, m_tiles=13, segments=1)


# ---------------------------------------------------------------------------------------------------------------------------
# Batches and forwards
# ---------------------------------------------------------------------------------------------------------------------------
SIZES = [(19, 19)] + [(s, s) for s in range(2, 19)] + [(13, 7), (7, 13), (19, 5), None]   # None: an empty mask


def mixed_batch(n, seed, nhwc=True, sizes=SIZES):
    """Boards of many sizes at the frame's top-left (as fillRowV7 places them), all 8 symmetries, some rows with an empty mask."""
    rng = np.random.default_rng(seed)
    pick = [sizes[(i + seed) % len(sizes)] for i in range(n)]
    rng.shuffle(pick)
    sp, gl = modelgen.synthetic_inputs(n, FRAME, FRAME, seed=seed, board_sizes=[b or (1, 1) for b in pick], nhwc=nhwc)
    for i, b in enumerate(pick):
        if b is None:
            sp[i] = 0.0
    sym = rng.integers(0, 8, n).astype(np.int32)
    sym[:min(n, 8)] = np.arange(min(n, 8))
    opt = rng.uniform(0, 1, n).astype(np.float32)
    mask = sp[..., 0] if nhwc else sp[:, 0]
    return sp, gl, sym, opt, mask


class EnvHandle:
    """A handle created with the given KGB_* variables set (None: unset), the process environment restored afterwards."""

    def __init__(self, path, max_batch, env, fp16=True, nhwc=True):
        old = {k: os.environ.get(k) for k in env}
        try:
            for k, v in env.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
            self.lm = NeuralNet.loadModelFile(path)
            self.ctx = NeuralNet.createComputeContext([0], FRAME, FRAME, fp16, self.lm)
            self.h = NeuralNet.createComputeHandle(self.ctx, self.lm, max_batch, False, nhwc, 0)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v

    def forward(self, sp, gl, sym, opt):
        got = NeuralNet.getOutput(self.h, sp.reshape(sp.shape[0], -1), gl, sym, opt)
        return got, self.h.layout_stats()

    def free(self):
        self.h.free(); self.ctx.free(); self.lm.free()


def assert_same_bits(a, b, what=""):
    for k in OUTPUTS:
        assert a[k].shape == b[k].shape
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), (what, k)


_models = {}


def model(cfg, tmp_path_factory):
    if cfg == "g170":
        return G170
    if cfg not in _models:
        d = tmp_path_factory.mktemp("ragged_models")
        if cfg == "tiny_relu_v8":
            _models[cfg] = modelgen.write_model(str(d / "tiny_v8.bin"), "tiny_reg", seed=6, version=8, activation="ACTIVATION_RELU")
        else:
            _models[cfg] = modelgen.write_model(str(d / f"{cfg}.bin"), cfg, seed=3)
    return _models[cfg]


# ---------------------------------------------------------------------------------------------------------------------------
# 1 + 2: whole-net bit identity against the reference plan, and the layout the plan reports
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg,n,fp16,streams,fuse,nhwc", [
    ("tiny_reg", 1, True, None, True, True),
    ("tiny_reg", 7, True, None, True, False),
    ("tiny_reg", 1021, False, None, True, True),
    ("tiny_nbt", 7, True, None, False, True),
    ("tiny_nbt", 256, True, None, True, False),
    ("tiny_nbt", 7, False, None, True, True),
    ("mid_nbt", 256, True, "trunk", True, True),
    ("mid_nbt", 256, True, "all", False, False),
    ("tiny_relu_v8", 256, True, None, True, True),
    ("tiny_relu_v8", 7, False, None, True, False),
    ("b18c384nbt", 256, True, None, True, True),
    ("b18c384nbt", 256, True, None, False, False),
    ("b18c384nbt", 256, True, "trunk", True, True),
    ("b18c384nbt", 256, True, "all", True, True),
    ("b18c384nbt", 256, False, None, True, True),
    ("b18c384nbt", 1021, True, None, True, True),
    ("g170", 256, True, None, True, True),
    ("g170", 7, False, None, True, False),
    ("b28c512nbt", 1024, True, None, True, True),
])
def test_outputs_match_the_reference_plan(tmp_path_factory, cfg, n, fp16, streams, fuse, nhwc):
    path = model(cfg, tmp_path_factory)
    pad = 2 if cfg == "g170" else 1              # g170-b6c96 has a 5x5 first convolution
    sp, gl, sym, opt, mask = mixed_batch(n, seed=n + len(cfg), nhwc=nhwc)
    env = {"KGB_STREAM_FP32": streams, "KGB_FUSE_BOUNDARY": None if fuse else "0"}
    results = {}
    for ragged in (True, False):
        eh = EnvHandle(path, n, dict(env, KGB_RAGGED_ROWS=None if ragged else "0"), fp16=fp16, nhwc=nhwc)
        results[ragged] = eh.forward(sp, gl, sym, opt)
        eh.free()
    (got, stats), (ref, ref_stats) = results[True], results[False]
    assert_same_bits(got, ref, cfg)
    on = np.array([mask[i].any() for i in range(n)])
    for k in OUTPUTS:
        assert np.isfinite(got[k][on]).all(), k
    assert stats == plan_stats(mask, sym, pad)
    assert ref_stats == plan_stats(mask, sym, pad, ragged=False)
    P = (FRAME + pad) ** 2
    assert ref_stats["rows"] == (n * P + pad * (FRAME + pad) + pad + 127) // 128 * 128
    if n >= 256:
        assert stats["rows"] < n * P


@pytest.mark.gpu
def test_layout_of_uniform_and_small_batches(tmp_path_factory):
    """An all-19x19 batch takes the frame layout's rows (plus one gap and alignment tail) in one segment; an all-9x9 batch a quarter of
    them; the reference plan the full frame whatever the boards."""
    path = model("tiny_reg", tmp_path_factory)
    n = 64
    eh = EnvHandle(path, n, {"KGB_RAGGED_ROWS": None})
    ref = EnvHandle(path, n, {"KGB_RAGGED_ROWS": "0"})
    full = (n * 400 + 21 + 127) // 128 * 128
    for sizes, rows in (([(19, 19)], full), ([(9, 9)], (n * 100 + 11 + 127) // 128 * 128)):
        sp, gl, sym, opt, mask = mixed_batch(n, seed=1, sizes=sizes)
        sym[:] = 0
        got, stats = eh.forward(sp, gl, sym, opt)
        want, ref_stats = ref.forward(sp, gl, sym, opt)
        assert_same_bits(got, want)
        assert stats == dict(rows=rows, m_tiles=rows // 128, segments=1)
        assert ref_stats == dict(rows=full, m_tiles=full // 128, segments=1)
    eh.free(); ref.free()


# ---------------------------------------------------------------------------------------------------------------------------
# 3: no state carried from one forward's layout to the next
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["mid_nbt", "g170"])
def test_no_state_carried_between_forwards(tmp_path_factory, cfg):
    """One handle runs batches whose layouts overlap differently - all 19x19, all 5x5, mixed, all 19x19 - and each result is the same
    bits as that batch on a fresh handle: gap rows and the taps of the last tile never see rows an earlier forward left behind."""
    path = model(cfg, tmp_path_factory)
    n = 64
    batches = [mixed_batch(n, seed=2, sizes=[(19, 19)]), mixed_batch(n, seed=3, sizes=[(5, 5)]), mixed_batch(n, seed=4),
               mixed_batch(n, seed=5, sizes=[(19, 19)])]
    eh = EnvHandle(path, n, {"KGB_RAGGED_ROWS": None})
    seq = [eh.forward(*b[:4]) for b in batches]
    eh.free()
    for (sp, gl, sym, opt, _), (got, stats) in zip(batches, seq):
        fresh = EnvHandle(path, n, {"KGB_RAGGED_ROWS": None})
        want, want_stats = fresh.forward(sp, gl, sym, opt)
        fresh.free()
        assert_same_bits(got, want)
        assert stats == want_stats


# ---------------------------------------------------------------------------------------------------------------------------
# 4: the self-play loop, move for move
# ---------------------------------------------------------------------------------------------------------------------------
def game_setups(n, rng):
    """What GameInitializer draws with selfplay8mainb18.cfg's board sizes: bSizes 7..19, 10% rectangles, every ko rule."""
    sizes = np.array([7, 9, 11, 13, 15, 17, 19, 8, 10, 12, 14, 16, 18])
    probs = np.array([1, 4, 3, 10, 7, 9, 75, 1, 2, 4, 6, 8, 10], float)   # bSizeRelProbs: 19x19 gets 75 of 140
    probs /= probs.sum()
    x = rng.choice(sizes, n, p=probs)
    y = np.where(rng.uniform(size=n) < 0.10, rng.choice(sizes, n, p=probs), x)
    return np.stack([x, y, rng.integers(0, 4, n), rng.integers(0, 2, n)], 1).astype(np.int32)


def run_loops(path, n, visits, iterations, max_moves, layouts=(True, False), cache=0):
    """Two loops with the same seed and setups, one per layout (True: ragged, False: the reference plan), compared after every few
    waves and at the end.  The evaluation cache is off by default: two games that store the same position in one wave race for its
    entry (the loser skips the store), so its contents and counters vary from run to run whatever the layout."""
    rng = np.random.default_rng(n)
    first, nxt = game_setups(n, rng), game_setups(n, rng)
    loops, handles = [], []
    for ragged in layouts:
        eh = EnvHandle(path, n, {"KGB_RAGGED_ROWS": None if ragged else "0"})
        sp = SelfPlay(eh.h, n, visits, komi=7.5, max_moves=max_moves, seed=21, use_graph_search=True, nn_cache_size_power_of_two=cache,
                      root_num_symmetries_to_sample=4, root_noise_enabled=True, use_play_selection=True, chosen_move_temperature_early=0.75,
                      chosen_move_temperature=0.15, debug_hold_at_max_visits=True)
        sp.set_game_setup(first, also_current_games=True)
        sp.set_game_setup(nxt)
        loops.append(sp); handles.append(eh)
    for _ in range(iterations):
        held = []
        for sp in loops:
            sp.run(4)
            held.append(np.asarray(sp.root_visits()))
        assert np.array_equal(held[0], held[1])
        release = (held[0] >= visits).astype(np.uint8)
        for sp in loops:
            sp.release(release)
            sp.run(1)
    a, b = loops
    st = a.stats()
    assert st == b.stats()
    assert np.array_equal(a.root_visits(), b.root_visits())
    for g in range(n):
        ca, ia = a.game(g)
        cb, ib = b.game(g)
        assert np.array_equal(ca, cb) and ia == ib, g
        for x, y in zip(a.root_children(g), b.root_children(g)):
            assert np.array_equal(x, y), g
    stats = [eh.h.layout_stats() for eh in handles]
    for sp in loops:
        sp.free()
    for eh in handles:
        eh.free()
    return st, stats


@pytest.mark.gpu
def test_self_play_loop_move_for_move_tiny(tmp_path_factory):
    st, (ragged, ref) = run_loops(model("tiny_reg", tmp_path_factory), 64, 16, 250, 24)
    assert st["total_moves"] >= 64 * 20 and st["games_finished"] >= 64
    assert ragged["rows"] < ref["rows"]


@pytest.mark.gpu
def test_self_play_loop_move_for_move_b18(tmp_path_factory):
    st, (ragged, ref) = run_loops(model("b18c384nbt", tmp_path_factory), 256, 8, 30, 0)
    assert st["total_moves"] >= 256 * 3
    assert ragged["rows"] < ref["rows"]
