"""Generates tests/golden/searchfake_1600.npz: BASELINE config 3's search size (19x19, maxVisits 1600) from the REFERENCE Search.

The reference's Search runs with the deterministic fake net (oracle/_ref/kgref_driver searchfake, see make_search_fixtures.py) on 8
positions of boardstream_19x19_multisuicide, from the empty board to past move 130, with the search block bench.py runs as far as
the driver implements it: selfplay8mainb18.cfg, graph search, subtree value bias, LCB, both root options and the root policy
temperature.  The root's evaluation is not averaged over symmetries (rootNumSymmetriesToSample 1), so no search draws from the
thread's Rand and one device loop can hold all 8 positions at once.

The stored game streams are the two 19x19 board streams with every pair of passes that would end the game removed (a pass pair
changes neither the stones nor the player to move), up to FILL_MOVES moves.  Every prefix of them is a game in progress, and the
driver checks that each move is legal under the stream's suicide rule.  The device test fills the loop's other slots with them."""
import json, os, sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_search_fixtures as F

VISITS = 1600
PARAMS = dict(F.SELFPLAY8B18, useGraphSearch=1, rootEndingBonusPoints=0.5, rootPruneUselessMoves=1, rootPolicyTemperature=1.1,
              rootPolicyTemperatureEarly=1.5, chosenMoveTemperatureHalflife=19, **F.BIAS, **F.LCB)
PREFIXES = (0, 7, 24, 41, 66, 93, 118, 136)     # moves of the multisuicide stream played before each search
FILL_MOVES = 150
STREAMS = ("boardstream_19x19_multisuicide.npz", "boardstream_19x19_nosuicide.npz")


def game_stream(name, n):
    """The first n moves of a board stream, with every pass that follows a pass dropped together with that pass."""
    out = []
    for x, y, _ in np.load(os.path.join(HERE, name))["moves"]:
        m = None if x < 0 else (int(x), int(y))
        if m is None and out and out[-1] is None:
            out.pop()
        else:
            out.append(m)
        if len(out) == n:
            break
    assert len(out) == n
    return out


def as_array(moves):
    return np.array([(-1, -1) if m is None else m for m in moves], np.int8).reshape(-1, 2)


if __name__ == "__main__":
    store = {"num_cases": len(PREFIXES), "visits": VISITS, "params": np.array(json.dumps(PARAMS))}
    for name in STREAMS:
        moves = game_stream(name, FILL_MOVES)
        # the driver plays every move through BoardHistory::isLegal and refuses an illegal one (it allows multi-stone suicide, which
        # the nosuicide stream never plays: dropping passes moves no stone)
        F.run(19, 19, 2, moves)
        store["fill_" + name.split("_")[-1].split(".")[0]] = as_array(moves)
    main = game_stream(STREAMS[0], max(PREFIXES))
    for i, k in enumerate(PREFIXES):
        moves = main[:k]
        root, v, u, pol, center, psv, threadseed, cstats, rstats = F.run(19, 19, VISITS, moves, PARAMS)
        assert root[0] == VISITS and v.sum() == VISITS - 1, (root, v.sum())
        store[f"c{i}_moves"] = as_array(moves)
        store[f"c{i}_visits"] = v; store[f"c{i}_util"] = u; store[f"c{i}_policy"] = pol; store[f"c{i}_play_selection"] = psv
        store[f"c{i}_child_stats"] = cstats; store[f"c{i}_root_stats"] = rstats
        print(i, len(moves), "moves; children", int((v > 0).sum()), "max visits", int(v.max()), "root util", root[1])
    np.savez_compressed(os.path.join(HERE, "searchfake_1600.npz"), **store)
