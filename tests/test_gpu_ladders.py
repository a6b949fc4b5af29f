"""The ladder reader (katago_b200/csrc/kgb_ladder.cuh: feature planes 14-17 of every row the loop evaluates) against the reference's
iterLadders / searchIsLadderCaptured, through NNInputs::fillRowV7 rows dumped by tests/golden/make_ladder_fixtures.py:

  tiny         every legal position of 2x2, 3x2 and 3x3 (57 / 489 / 12 675), both sides to move, in a 3x3 frame - every point is an
               edge and the search stack limit is smallest there
  small        random legal 4x3, 4x4 and 5x5 positions with many 1-2 liberty chains, all three ko rules
  constructed  ladders built on purpose (working chases of up to 34 moves, breakers, an attacker stone on the path, escapes by capture,
               two working moves, both liberties open, a first attacker move that is suicide) under every symmetry of 19x19, 13x7,
               7x13, 10x10 boards and 9x9 / 13x7 / 5x5 boards inside a 19x19 frame, also played into the chase (planes 15/16);
               each carries the outcome it was designed for
  heavy        dense random 19x19 and 13x13 positions with the most 1-2 liberty chains (40 or more: every warp takes several searches)
  ko           random 4x4 to 19x19 positions (some inside a 19x19 frame) whose last move took a ko, mostly with a 2-liberty chain
               whose liberty is the ko point: the attacker's first move there is illegal

The CPU part checks the designed outcomes and the coverage against the reference rows; the GPU part loads every position into a slot of
one SelfPlay (debug_fake_nn) and compares the row of its root leaf with the reference bit for bit - planes 14-17 first, then every plane
and every global - unbudgeted and with ladder_nodes_per_wave 1, 7 and 256 (the suspended-and-resumed searches must give the same rows)."""
import os

import numpy as np
import pytest

FAMILIES = ("tiny", "small", "constructed", "heavy", "ko")
PAD = -128
SLOTS = 512                 # ladder scratch is about 2.2 MB per slot
BUDGETS = (1, 7, 256)
BUDGET_SAMPLE = 1024        # positions per frame that also run with each ladder_nodes_per_wave budget
MAX_BUDGET_WAVES = 60000    # no fixture search comes near 25 000 moves, so even one move per wave finishes well within this
# Positions where the device's row differs from the reference's by design, with the device's result asserted instead: the reference's
# "lower bound of liberties >= 3" shortcut at a defender node (game/board.cpp:1716-1722) is applied to the LAST move of its list.  When
# the defender's lone liberty is itself a capturing move and other captures exist, findLiberties does not append the liberty again, so
# that last move is whichever capture the chain's linked list reaches last - an order the bitboard reader does not have (DESIGN.md,
# "Known deviations").  Here, after the attacker's move on (7, 18), the lone liberty (5, 17) captures one stone and (2, 17) captures
# two; the reference calls the chain escaped by the bound, the device's full search finds it captured.  (family, name): [(x, y, plane, device value)]
KNOWN_ORDER_DEPENDENT = {
    # the two previous boards (a pass and a move elsewhere back) hold the same chain in the same surroundings: planes 15 and 16 too
    ("ko", "ko19x19in19x19:3996:kolib"): [(x, 18, pl, 1) for pl in (14, 15, 16) for x in (4, 5, 6)],
}


def _load(golden_dir, tag):
    d = np.load(os.path.join(golden_dir, f"ladders_{tag}.npz"))
    return {k: d[k] for k in d.files}


@pytest.fixture(scope="module")
def fixtures(golden_dir):
    return {tag: _load(golden_dir, tag) for tag in FAMILIES}


def _row(d, i):
    NX, NY = int(d["NX"][i]), int(d["NY"][i])
    return np.unpackbits(d["rows"][i])[:NX * NY * 22].reshape(NY * NX, 22)


def _moves(d, i):
    m = d["moves"][i]
    m = m[m[:, 0] != PAD]
    return [None if x < 0 else (int(x), int(y)) for x, y in m]


def _diagram(d, i, row=None):
    """The position as text ('X' black, 'O' white, '.' empty; the side to move in the header)."""
    X, Y, NX = int(d["X"][i]), int(d["Y"][i]), int(d["NX"][i])
    row = _row(d, i) if row is None else row
    lines = []
    for y in range(Y):
        s = ""
        for x in range(X):
            p = row[y * NX + x]
            s += "M" if p[1] else "T" if p[2] else "."
        lines.append(s)
    return "(M = side to move, T = opponent)\n" + "\n".join(lines)


def _chain_count(row, NX, X, Y, plane):
    """Number of 4-connected groups of set points of `plane` (laddered chains for plane 14)."""
    on = row[:, plane].reshape(-1, NX)[:Y, :X].astype(bool)
    seen = np.zeros_like(on)
    n = 0
    for y in range(Y):
        for x in range(X):
            if on[y, x] and not seen[y, x]:
                n += 1
                stack = [(x, y)]
                seen[y, x] = True
                while stack:
                    px, py = stack.pop()
                    for qx, qy in ((px - 1, py), (px + 1, py), (px, py - 1), (px, py + 1)):
                        if 0 <= qx < X and 0 <= qy < Y and on[qy, qx] and not seen[qy, qx]:
                            seen[qy, qx] = True
                            stack.append((qx, qy))
    return n


# ------------------------------------------------------------------------------------------------------------------ CPU part
def test_ladder_fixtures_hold_their_designed_outcomes(fixtures):
    """Every constructed position decides what it was built for, by the reference's own rows: the hunted chain is (or is not) laddered
    and plane 17 holds exactly the designed working moves.  Without this a family could quietly degrade into "nothing is laddered"."""
    checked = 0
    for tag, d in fixtures.items():
        for i, x, y, pl, val in d["exp"]:
            row = _row(d, i)
            assert row[y * int(d["NX"][i]) + x, pl] == val, (tag, str(d["name"][i]), (x, y), pl, _diagram(d, i, row))
            checked += 1
        for i in np.flatnonzero(d["exact17"] >= 0):
            row = _row(d, i)
            assert int(row[:, 17].sum()) == int(d["exact17"][i]), (tag, str(d["name"][i]), _diagram(d, i, row))
    assert checked > 0


def test_ladder_fixture_coverage(fixtures):
    """Coverage of each family, printed, with minimums: positions, laddered chains, plane-17 bits, positions with a simple-ko point
    (the only ko the ladder reader sees) and with a 2-liberty chain on it; the exhaustive tiny boards are complete (57 / 489 / 12 675
    legal positions, each with both sides to move); the designed escapes by capture and chases of 15 moves or more are there."""
    print()
    print(f"{'family':12s} {'positions':>9s} {'laddered':>9s} {'plane17':>8s} {'simple ko':>9s} {'2-lib on ko':>11s}")
    totals = {}
    for tag, d in fixtures.items():
        n = len(d["name"])
        lad = p17 = ko = 0
        for i in range(n):
            row = _row(d, i)
            lad += _chain_count(row, int(d["NX"][i]), int(d["X"][i]), int(d["Y"][i]), 14)
            p17 += int(row[:, 17].sum())
        ko = int(d["simple_ko"].sum())
        kolib = sum(1 for s in d["name"] if str(s).endswith(":kolib"))
        totals[tag] = (n, lad, p17, ko, kolib)
        print(f"{tag:12s} {n:9d} {lad:9d} {p17:8d} {ko:9d} {kolib:11d}")
    names = [str(s) for s in fixtures["tiny"]["name"]]
    for size, count in (("2x2", 57), ("3x2", 489), ("3x3", 12675)):
        got = sum(1 for s in names if s.startswith(f"tiny{size}:"))
        print(f"exhaustive {size}: {got // 2} positions x 2 sides to move")
        assert got == 2 * count, (size, got)
    for tag in FAMILIES:
        n, lad, p17, ko, kolib = totals[tag]
        assert lad >= n // 20 and p17 > 0, (tag, totals[tag])
    assert totals["ko"][3] == totals["ko"][0] and totals["ko"][4] >= 1000, totals["ko"]
    # plane 6 marks the simple-ko point under the simple ko rule: the reference saw the ko the generator built
    ko = fixtures["ko"]
    assert all(_row(ko, i)[:, 6].any() for i in np.flatnonzero(ko["ko"] == 0))
    names = [str(s) for s in fixtures["constructed"]["name"]]
    escapes = sum(1 for s in names if s.startswith("escape_capture_") and "control" not in s)
    long_chases = sum(1 for s in names if s.startswith("working_long:"))      # a 34-move chase along the 19x19 diagonal
    print(f"designed escapes by capture: {escapes}; chases of 15+ moves: {long_chases}")
    assert escapes >= 16 and long_chases >= 8


# ------------------------------------------------------------------------------------------------------------------ GPU part
def _groups(fixtures):
    """(NX, NY) frame -> [(tag, index)]"""
    out = {}
    for tag, d in fixtures.items():
        for i in range(len(d["name"])):
            out.setdefault((int(d["NX"][i]), int(d["NY"][i])), []).append((tag, i))
    return out


def _device_rows(h, fixtures, entries, budget, kind):
    """Rows of the root leaf of every position in `entries`, SLOTS positions per SelfPlay.  budget 0: the first wave delivers every
    root leaf (nn_row); otherwise waves run until every root was evaluated, and the row kept for the root is read (root_row)."""
    from katago_b200 import SelfPlay
    rows, stats = [], dict(ladder_searches=0, ladder_nodes=0, stalled_waves=0, waves=0)
    for c0 in range(0, len(entries), SLOTS):
        chunk = entries[c0:c0 + SLOTS]
        n = len(chunk)
        sp = SelfPlay(h, n, 8, komi=7.5, seed=1, debug_fake_nn=True, debug_hold_at_max_visits=True, ladder_nodes_per_wave=budget)
        setup = np.array([[int(fixtures[t]["X"][i]), int(fixtures[t]["Y"][i]), int(fixtures[t]["ko"][i]), int(fixtures[t]["multi"][i])]
                          for t, i in chunk], np.int32)
        sp.set_game_setup(setup, also_current_games=True)
        for g, (t, i) in enumerate(chunk):
            sp.play_moves_game(g, _moves(fixtures[t], i))
        if budget == 0:
            sp.run(1)
            stats["waves"] += 1
            for g in range(n):
                path, valid = sp.leaf_path(g)
                assert valid and path == [], (kind, chunk[g], path, valid)
                rows.append(sp.nn_row(g))
        else:
            for _ in range(MAX_BUDGET_WAVES // 8):
                if (sp.root_visits() >= 1).all():
                    break
                sp.run(8)
                stats["waves"] += 8
            else:
                raise AssertionError(f"{kind}: ladder searches with budget {budget} never finished")
            rows += [sp.root_row(g) for g in range(n)]
        st = sp.stats()
        for k in ("ladder_searches", "ladder_nodes", "stalled_waves"):
            stats[k] += st[k]
        sp.free()
    return rows, stats


def _compare(fixtures, entries, rows, kind):
    """Mismatches, ladder planes first: (family, name, what, diagram)."""
    bad = []
    for (t, i), (row, gl) in zip(entries, rows):
        d = fixtures[t]
        ref = _row(d, i).astype(np.float32)
        NX = int(d["NX"][i])
        for x, y, pl, val in KNOWN_ORDER_DEPENDENT.get((t, str(d["name"][i])), []):
            assert ref[y * NX + x, pl] != val, ("the reference now agrees with the device", t, str(d["name"][i]))
            ref[y * NX + x, pl] = val
        for pl in (14, 15, 16, 17) + tuple(p for p in range(22) if p not in (14, 15, 16, 17)):
            if not np.array_equal(row[:, pl], ref[:, pl]):
                pts = [(int(p) % NX, int(p) // NX, "dev" if row[p, pl] else "ref") for p in np.flatnonzero(row[:, pl] != ref[:, pl])]
                bad.append((t, str(d["name"][i]), f"plane {pl} at (x, y, set by): {pts[:12]}", _diagram(d, i, ref.astype(np.uint8))))
                break
        else:
            if not np.array_equal(gl, d["glob"][i]):
                bad.append((t, str(d["name"][i]), f"globals {gl} vs {d['glob'][i]}", _diagram(d, i)))
    return bad


def _report(bad, kind):
    for t, name, what, diagram in bad[:8]:
        print(f"{kind}: {t} {name}: {what}\n{diagram}")
    return f"{kind}: {len(bad)} positions differ from the reference, first: {[b[:3] for b in bad[:4]]}"


@pytest.mark.gpu
def test_ladder_rows_match_reference_bit_for_bit(fixtures, tmp_models):
    """Every fixture position's root row equals the reference's fillRowV7 row on every plane and global; then the same rows again with the
    searches cut into slices of 1, 7 and 256 moves per wave (suspended in one wave, resumed in a later one)."""
    from katago_b200 import NeuralNet
    lm = NeuralNet.loadModelFile(tmp_models["tiny_reg"])
    failures, stalled = [], {b: 0 for b in BUDGETS}
    for (NX, NY), entries in sorted(_groups(fixtures).items()):
        ctx = NeuralNet.createComputeContext([0], NX, NY, True, lm)
        h = NeuralNet.createComputeHandle(ctx, lm, min(SLOTS, len(entries)), False, True, 0)
        kind = f"frame {NX}x{NY}"
        rows, st = _device_rows(h, fixtures, entries, 0, kind)
        bad = _compare(fixtures, entries, rows, kind)
        print(f"{kind}: {len(entries)} positions, {st['ladder_searches']} ladder searches, {st['ladder_nodes']} nodes, {len(bad)} differ")
        if bad:
            failures.append(_report(bad, kind))
        # budgeted: a stride sample of each frame's positions, with every heavy one
        heavy = [k for k, (t, i) in enumerate(entries) if t == "heavy"]
        step = max(1, len(entries) // BUDGET_SAMPLE)
        pick = sorted(set(range(0, len(entries), step)) | set(heavy))
        sub = [entries[k] for k in pick]
        for budget in BUDGETS:
            brows, bst = _device_rows(h, fixtures, sub, budget, f"{kind} budget {budget}")
            diff = [entries[k] for k, r in zip(pick, brows) if not (np.array_equal(r[0], rows[k][0]) and np.array_equal(r[1], rows[k][1]))]
            print(f"{kind} ladder_nodes_per_wave {budget}: {len(sub)} positions, {bst['waves']} waves, {bst['stalled_waves']} stalled game-waves, "
                  f"{bst['ladder_searches']} searches, {bst['ladder_nodes']} nodes, {len(diff)} rows differ from the unbudgeted run")
            if diff:
                failures.append(f"{kind} budget {budget}: rows differ from the unbudgeted run at {[(t, str(fixtures[t]['name'][i])) for t, i in diff[:6]]}")
            stalled[budget] += bst["stalled_waves"]
        h.free(); ctx.free()
    lm.free()
    assert not failures, "\n".join(failures)
    assert stalled[1] > 0 and stalled[7] > 0, stalled      # the small budgets did suspend searches
