"""Generates tests/golden/searchfake_wide.npz: whole REFERENCE searches on the wide hash net (oracle/_ref/kgref_driver searchfake with
KGREF_FAKE_WIDE=1; the device loop's debug_fake_nn = 4).

The narrow hash net of searchfake.npz returns a no-result logit of -30, stdev logits in [-2, 2) and policy logits in [-4, 4), so
P(no result) stays near 1e-13 in every search.  The wide net draws the no-result logit like win and loss from [-6, 6), the stdev logit
from [-8, 56), policy logits from [-24, 24) with one point in 16 a further 96 below, mean and lead from [-3, 3): the no-result moment,
superko's removal of it, noResultUtilityForWhite, the linear softplus branch and underflowing policy tails then act in every search and
are backed up through the tree.  Stored per case like searchfake.npz (same keys), plus `c{i}_device` (device-only switches: the
evaluation cache, whose hits run utilityFromEval in the select kernel) and `c{i}_branches`: how many of the reference's evaluations had
P(no result) > 0.05, had that removed by superko, took the linear softplus branch, had a policy term underflow to 0 in float.

Needs oracle/_ref/kgref_driver (run `python __graft_entry__.py` first)."""
import json, os, subprocess, sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_search_fixtures as F  # noqa: E402

WIDE = {"KGREF_FAKE_WIDE": "1"}


def cases():
    p9 = F.prefix_from_stream("boardstream_9x9_multisuicide.npz", 12)
    p19 = F.prefix_from_stream("boardstream_19x19_multisuicide.npz", 40)
    p5 = F.prefix_from_stream("boardstream_5x5_multisuicide.npz", 9)
    p13 = F.prefix_from_stream("boardstream_13x7_nosuicide.npz", 20)
    SP, GRAPH = dict(F.SELFPLAY8B18), dict(F.SELFPLAY8B18, useGraphSearch=1, **F.BIAS)
    # (X, Y, visits, moves, SearchParams overrides, frame or None, device-only switches)
    return [
        (9, 9, 400, p9, {"noResultUtilityForWhite": -0.5}, None, {}),                                    # simple ko, no-result utility
        (9, 9, 400, p9, dict(SP, noResultUtilityForWhite=0.3), None, {}),
        (9, 9, 400, p9, {"koRule": 1}, None, {}),                                                         # positional superko
        (9, 9, 400, p9, dict(SP, koRule=2, noResultUtilityForWhite=-0.5), None, {}),                    # situational superko
        (19, 19, 300, p19, dict(SP), None, {}),                                                           # selfplay8mainb18 block
        (9, 9, 500, p9, dict(GRAPH, noResultUtilityForWhite=0.2), None, {}),                            # graph search + bias
        (9, 9, 300, p9, dict(SP, rootNumSymmetriesToSample=4, noResultUtilityForWhite=-0.3), None, {}),  # 4 root symmetries
        (9, 9, 400, p9, dict(SP, noResultUtilityForWhite=-0.5), None, {"nn_cache_size_power_of_two": 12}),  # evaluation cache on
        (9, 9, 400, p9, dict(SP, noResultUtilityForWhite=0.3), 19, {}),                                  # 9x9 in a 19x19 frame
        (7, 7, 300, F.PRUNE_7X7, dict(SP, rootEndingBonusPoints=0.5, rootPruneUselessMoves=1, noResultUtilityForWhite=-0.4), None, {}),
        (5, 5, 600, p5, {"noResultUtilityForWhite": -0.5}, None, {}),                                   # reaches terminal positions
        (5, 5, 600, p5, dict(SP, koRule=1), None, {}),
        (19, 19, 300, p19, dict(GRAPH, noResultUtilityForWhite=0.3), None, {"nn_cache_size_power_of_two": 12}),
        (9, 9, 400, p9, dict(SP, winLossUtilityFactor=0.7, noResultUtilityForWhite=-0.3, drawEquivalentWinsForWhite=0.3), None, {}),
        (13, 7, 300, p13, dict(SP, koRule=2), None, {}),
        (9, 9, 600, p9, dict(SP, **F.LCB, noResultUtilityForWhite=0.2), None, {}),                        # play selection with LCB
    ]


def branches(X, Y, visits, moves, params, frame):
    s = " ".join("pass" if m is None else f"{m[0]},{m[1]}" for m in moves)
    env = dict(os.environ, **WIDE, **({"KGREF_NN_LEN": str(frame)} if frame else {}))
    out = subprocess.run([F.DRIVER, "searchfake", F.MODEL, str(X), str(Y), str(visits), s] + [f"{k}={float(v)!r}" for k, v in params.items()],
                         capture_output=True, text=True, check=True, env=env).stdout
    return np.array([int(t) for t in next(ln for ln in out.splitlines() if ln.startswith("widebranches")).split()[1:]], np.int64)


if __name__ == "__main__":
    cs = cases()
    store = {"num_cases": np.int32(len(cs))}
    for i, (X, Y, visits, moves, params, frame, dev) in enumerate(cs):
        root, v, u, pol, center, psv, threadseed, cstats, rstats = F.run(X, Y, visits, moves, params, env=WIDE, frame=frame)
        store[f"c{i}_child_stats"] = cstats; store[f"c{i}_root_stats"] = rstats
        store[f"c{i}_thread_seed"] = np.array(threadseed)
        store[f"c{i}_play_selection"] = psv
        store[f"c{i}_params"] = np.array(json.dumps(params))
        store[f"c{i}_device"] = np.array(json.dumps(dev))
        store[f"c{i}_shape"] = np.array([X, Y, visits, frame or 0], np.int32)
        store[f"c{i}_moves"] = np.array([(-1, -1) if m is None else m for m in moves], np.int8).reshape(-1, 2)
        store[f"c{i}_visits"] = v; store[f"c{i}_util"] = u; store[f"c{i}_policy"] = pol
        store[f"c{i}_root_util"] = np.float64(root[1])
        store[f"c{i}_branches"] = branches(X, Y, visits, moves, params, frame)
        print(i, X, Y, visits, "root visits", root[0], "branches", store[f"c{i}_branches"])
    np.savez_compressed(os.path.join(HERE, "searchfake_wide.npz"), **store)
