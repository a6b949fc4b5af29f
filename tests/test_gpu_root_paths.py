"""GPU tests of the ways a game's root position moves outside the search: random openings against the same moves played as a list,
and a game started by a list against a fresh game."""
import numpy as np
import pytest

from katago_b200 import NeuralNet, SelfPlay, board_replay, modelgen
from katago_b200.nn_backend import history_replay, rand_uint32_stream

pytestmark = pytest.mark.gpu

SEED = 7
KO_POSITIONAL = 1


@pytest.fixture(scope="module")
def handles(tmp_path_factory):
    path = modelgen.write_model(str(tmp_path_factory.mktemp("roots") / "tiny_nbt.bin"), "tiny_nbt", seed=11)
    lm = NeuralNet.loadModelFile(path)
    out, owned = {}, []
    for n in (9, 19):
        ctx = NeuralNet.createComputeContext([0], n, n, True, lm)
        h = NeuralNet.createComputeHandle(ctx, lm, 16, False, True, 0)
        out[n] = h
        owned.append((h, ctx))
    yield out
    for h, ctx in owned:
        h.free(); ctx.free()


def _legal_after(n, prefixes, superko):
    """Legal points (row-major flat index) for the player to move after each move list, from the reference-pinned replay hooks."""
    if len(prefixes[0]) == 0:
        return [np.ones(n * n, bool) for _ in prefixes]
    if superko:
        mv = np.array([[(-1, -1) if m is None else m for m in p] for p in prefixes], np.int8)
        _, legal, _ = history_replay(n, n, KO_POSITIONAL, True, mv)
        return [legal[i, -1].astype(bool) for i in range(len(prefixes))]
    mv = np.array([[(-1, -1, 0) if m is None else (m[0], m[1], 0) for m in p] for p in prefixes], np.int8)
    mv[:, :, 2] = np.where(np.arange(mv.shape[1]) % 2 == 0, 1, 2)   # black first, colours alternate
    legal = board_replay(n, n, mv, True)["legal_next"]
    return [legal[i, -1].reshape(-1).astype(bool) for i in range(len(prefixes))]


def _random_opening_lists(n, games, max_len, superko):
    """The moves spRandomOpeningsKernel plays, rebuilt on the host: each game's non-search generator draws the length, then the r-th legal
    point in row-major order for every move."""
    streams = [rand_uint32_stream(f"kgb200$seed{SEED}$game{g}$nonSearchRand", max_len + 2) for g in range(games)]
    lens = [int(s[0] % (max_len + 1)) for s in streams]
    lists = [[] for _ in range(games)]
    for m in range(max(lens)):
        active = [g for g in range(games) if len(lists[g]) == m and m < lens[g]]
        if not active:
            break
        for g, legal in zip(active, _legal_after(n, [lists[g] for g in active], superko)):
            pts = np.nonzero(legal)[0]
            if len(pts) == 0:
                continue
            p = int(pts[int(streams[g][1 + m]) % len(pts)])
            lists[g].append((p % n, p // n))
    return lists


def _loop(h, games, superko):
    kw = dict(ko_rule=KO_POSITIONAL) if superko else {}
    return SelfPlay(h, games, 8, komi=7.5, seed=SEED, debug_fake_nn=True, **kw)


def _assert_same_root(a, ga, b, gb, what):
    ca, ia = a.game(ga)
    cb, ib = b.game(gb)
    assert np.array_equal(ca, cb) and ia == ib, (what, ia, ib)
    sa, la = a.nn_row(ga)
    sb, lb = b.nn_row(gb)
    bad = sorted({int(c) for c in np.nonzero((sa != sb).any(axis=0))[0]})
    assert np.array_equal(sa, sb) and np.array_equal(la, lb), (what, "spatial planes differ:", bad)


@pytest.mark.parametrize("n,max_len,superko", [(9, 60, False), (9, 60, True), (19, 150, False), (19, 150, True)])
def test_random_openings_equal_the_same_moves_played_as_a_list(handles, n, max_len, superko):
    """Board, history planes 9-13 and ladder planes 15/16 after random openings are bit for bit those of the same moves given to play_moves."""
    games = 12
    lists = _random_opening_lists(n, games, max_len, superko)
    assert len({len(l) for l in lists}) > 3 and max(len(l) for l in lists) > 10
    a = _loop(handles[n], games, superko)
    a.random_openings(max_len)
    b = _loop(handles[n], games, superko)
    for g in range(games):
        b.play_moves_game(g, lists[g])
    for g in range(games):
        assert a.game(g)[1]["move_num"] == len(lists[g]), g
    a.run(1); b.run(1)
    for g in range(games):
        _assert_same_root(a, g, b, g, (n, superko, g, len(lists[g])))
    a.free(); b.free()


@pytest.mark.parametrize("superko", [False, True])
@pytest.mark.parametrize("tail_len", [0, 1, 2, 30])
def test_game_started_by_a_list_is_like_a_fresh_game(handles, superko, tail_len):
    """A move list that ends a game with two passes and goes on: the new game equals a fresh slot that plays only the tail, and the ended
    game's move record shows the end."""
    n = 9
    prefix, tail = sorted(_random_opening_lists(n, 8, 60, superko), key=len, reverse=True)[:2]
    tail = tail[:tail_len]
    assert len(tail) == tail_len and len(prefix) > 10
    sp = _loop(handles[n], 2, superko)
    sp.play_moves_game(0, prefix + [None, None] + tail)
    sp.play_moves_game(1, tail)
    lm = sp.last_move(0)
    assert lm["game_over"] and not lm["no_result"] and not lm["hit_move_limit"], lm
    assert lm["xy"] == (-1, -1) and lm["move_num"] == len(prefix) + 1 and lm["game_index"] == 0, lm
    sp.run(1)
    _assert_same_root(sp, 0, sp, 1, (superko, tail_len))
    sp.free()
