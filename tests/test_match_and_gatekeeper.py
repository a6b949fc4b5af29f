"""SURVEY §8f row 4: games between two nets (katago_b200/match_play.py) and the gatekeeper / match commands on top of them.
CPU tests drive the host logic with scripted loops; the GPU tests play real games on the device."""
import os
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from katago_b200 import gatekeeper_cli as G
from katago_b200.match_play import MatchPlay


class ScriptedLoop:
    """What MatchPlay uses of a SelfPlay: every search is finished at once, move t of a game is point t of a 5x5 board, game k of slot g
    ends after lengths[g][k] moves with score scores[g][k] (white minus black)."""

    def __init__(self, n, lengths, scores):
        self.num_games, self.x, self.y, self.max_visits = n, 5, 5, 4
        self.lengths, self.scores = lengths, scores
        self.t = [0] * n; self.k = [0] * n
        self.released = np.zeros(n, bool)
        self.last = [None] * n
        self.mirrored = [[] for _ in range(n)]
        self.last_setup = np.tile(np.array([5, 5, 0, 1], np.int32), (n, 1)); self.last_komi = np.full(n, 7.5, np.float32)

    def run(self, waves):
        for g in np.flatnonzero(self.released):
            self._advance(int(g), None)
        self.released[:] = False

    def _advance(self, g, move):
        t = self.t[g]
        mv = (t % 5, t // 5) if move is None else move
        assert mv == (t % 5, t // 5), "the loops are out of step"
        self.t[g] += 1
        over = self.t[g] >= self.lengths[g][self.k[g]]
        self.last[g] = dict(xy=mv, game_over=over, no_result=False, hit_move_limit=False, game_index=self.k[g],
                            final_white_minus_black_score=self.scores[g][self.k[g]] if over else 0.0)
        if over:
            self.t[g] = 0; self.k[g] += 1

    def root_visits(self):
        return np.full(self.num_games, self.max_visits, np.int32)

    def release(self, mask):
        self.released |= np.asarray(mask, bool)

    def last_move(self, g):
        return self.last[g]

    def play_moves_game(self, g, moves):
        for m in moves:
            self.mirrored[g].append(m)
            self._advance(g, m)

    def game_setups(self):
        return self.last_setup.copy(), self.last_setup.copy()

    def komi_values(self):
        return self.last_komi.copy(), self.last_komi.copy()


def test_match_play_mirrors_moves_alternates_colours_and_tallies():
    n = 3
    lengths = [[4, 3, 5, 2], [2, 6, 3, 3], [5, 5, 5, 5]]
    scores = [[2.5, -1.5, 0.0, 3.5], [-0.5, 4.5, -2.5, 1.5], [1.5, 1.5, -3.5, 0.5]]
    a, b = ScriptedLoop(n, lengths, scores), ScriptedLoop(n, lengths, scores)
    seen = []
    mp = MatchPlay([a, b], ["base", "cand"], 7, on_game=lambda slot, game, bn, wn, res: seen.append((slot, bn, wn, res, list(game.moves), game.x_size)))
    mp.run(waves=1, max_pumps=200)
    assert mp.games_tallied == 7 and len(seen) == 7 and mp.done()
    # every game was played out move for move in BOTH loops: each move was made by one and mirrored into the other
    for g in range(n):
        assert a.k[g] == b.k[g] and a.t[g] == b.t[g]
        assert len(a.mirrored[g]) + len(b.mirrored[g]) >= sum(lengths[g][:a.k[g]])
    # colours alternate per slot, starting with bot g % 2 as black
    per_slot = {}
    for slot, bn, wn, res, moves, xs in seen:
        per_slot.setdefault(slot, []).append(bn)
        assert {bn, wn} == {"base", "cand"} and xs == 5 and moves == [(t % 5, t // 5) for t in range(len(moves))]
    for slot, blacks in per_slot.items():
        assert blacks[0] == ["base", "cand"][slot % 2]
        assert all(x != y for x, y in zip(blacks, blacks[1:]))
    # points: a win is 1, a drawn score 0.5 each (noResultUtilityForWhite 0), and they add up to the games
    assert abs(sum(mp.win_points) - 7) < 1e-12
    pts = {"base": 0.0, "cand": 0.0}
    for slot, bn, wn, res, moves, xs in seen:
        if res.startswith("B+"):
            pts[bn] += 1
        elif res.startswith("W+"):
            pts[wn] += 1
        else:
            pts[bn] += 0.5; pts[wn] += 0.5
    assert abs(pts["base"] - mp.win_points[0]) < 1e-12 and abs(pts["cand"] - mp.win_points[1]) < 1e-12


class ResigningLoop(ScriptedLoop):
    """ScriptedLoop whose searches always say white is lost (root win/loss -0.95) and which understands the passes that end a resigned game."""

    def root_value_stats(self, g):
        return None, np.array([-0.95, 0.0, -20.0, 400.0, -20.0])

    def game(self, g):
        return None, dict(move_num=self.t[g])

    def play_moves_game(self, g, moves):
        if moves == [None]:
            self.passes = getattr(self, "passes", {})
            self.passes[g] = self.passes.get(g, 0) + 1
            self.t[g] += 1
            if self.passes[g] == 2:                # two passes: the slot's next game begins
                self.passes[g] = 0; self.t[g] = 0; self.k[g] += 1
            return
        super().play_moves_game(g, moves)


def test_match_play_resignation():
    """allowResignation (play.cpp:1903-1929): after its move, a player whose last resignConsecTurns root values were all beyond the threshold
    resigns - not before turn 1 + area / 5 - the game counts for the opponent ("B+R"), both loops start the slot's next game."""
    n = 2
    lengths = [[30] * 6, [30] * 6]
    scores = [[5.5] * 6, [5.5] * 6]                # never reached: white resigns long before move 30
    a, b = ResigningLoop(n, lengths, scores), ResigningLoop(n, lengths, scores)
    seen = []
    mp = MatchPlay([a, b], ["base", "cand"], 4, on_game=lambda slot, game, bn, wn, res: seen.append((slot, bn, wn, res, len(game.moves), getattr(game, "resigned", False))),
                   allow_resignation=True, resign_threshold=-0.9, resign_consec_turns=3)
    mp.run(waves=1, max_pumps=400)
    assert mp.games_tallied == 4 and all(res == "B+R" and resigned for _, _, _, res, _, resigned in seen)
    # 5x5 board: no resignation before turn index 1 + 25 // 5 = 6; white moves on odd indices, so its first chance is its move with index 7 (8 moves made)
    assert all(nm == 8 for _, _, _, _, nm, _ in seen), [s[4] for s in seen]
    pts = {"base": 0.0, "cand": 0.0}
    for slot, bn, wn, res, nm, _ in seen:
        pts[bn] += 1.0
    assert pts["base"] == mp.win_points[0] and pts["cand"] == mp.win_points[1]
    assert a.k == b.k and a.t == b.t


def test_gatekeeper_protocol_with_a_scripted_match(tmp_path):
    """The directory protocol of command/gatekeeper.cpp: candidate = newest test net, baseline = newest accepted net, auto-rejection of
    older candidates, acceptance with ties going to the candidate, files or model directories moved, self-play directories prepared."""
    test, acc, rej, sgf, sp = (tmp_path / d for d in ("test", "accepted", "rejected", "sgf", "selfplay"))
    for d in (test, acc, rej):
        d.mkdir()
    (acc / "net-a.bin.gz").write_bytes(b"a")
    old = test / "net-old.bin.gz"; old.write_bytes(b"o")
    os.utime(old, (time.time() - 1000, time.time() - 1000))
    assert G.find_latest_model(str(tmp_path / "rejected")) is None
    log = []

    class A:
        test_models_dir, accepted_models_dir, rejected_models_dir, sgf_output_dir, selfplay_dir = str(test), str(acc), str(rej), str(sgf), str(sp)
        required_candidate_win_prop, no_autoreject_old_models, games_per_gpu, seed = 0.5, False, 8, 0
    calls = []

    def play(cfg, base_file, cand_file, names, sgf_dir, games, prop, lg, seed=0):
        calls.append((os.path.basename(base_file), os.path.basename(cand_file), names))
        return play.result
    # 1. a candidate older than the accepted net is rejected without a game
    assert G.gate_once(A, {}, log.append, play) == "autorejected" and calls == [] and (rej / "net-old.bin.gz").exists() and not old.exists()
    # 2. a model directory as candidate, exact tie: accepted (the candidate wins ties), directory moved, self-play directories made
    (test / "net-b").mkdir(); (test / "net-b" / "model.bin.gz").write_bytes(b"b")
    os.utime(test / "net-b", (time.time() + 10, time.time() + 10))
    play.result = (4.0, 4.0, 8)
    assert G.gate_once(A, {}, log.append, play) == "accepted"
    assert calls[-1] == ("net-a.bin.gz", "model.bin.gz", ("net-a", "net-b")) and (acc / "net-b" / "model.bin.gz").exists() and not (test / "net-b").exists()
    assert all((sp / "net-b" / s).is_dir() for s in ("sgfs", "tdata", "vadata"))
    assert any("Candidate won match, score 4.000 to 4.000 in 8 games, accepting candidate net-b" in l for l in log)
    # 3. the next candidate plays the newly accepted net and loses
    (test / "net-c.bin.gz").write_bytes(b"c")
    os.utime(test / "net-c.bin.gz", (time.time() + 20, time.time() + 20))
    play.result = (4.5, 3.5, 8)
    assert G.gate_once(A, {}, log.append, play) == "rejected" and calls[-1][2] == ("net-b", "net-c") and (rej / "net-c.bin.gz").exists()
    assert G.gate_once(A, {}, log.append, play) == "none"
    # early termination rule (gatekeeper.cpp:181-192) and the final verdict (:581)
    assert G.early_verdict(100.0, 150, 200, 0.5) == 1 and G.early_verdict(20.0, 121, 200, 0.5) == -1 and G.early_verdict(50.0, 100, 200, 0.5) == 0
    assert G.early_verdict(120.0, 200, 200, 0.5) == 0
    assert G.candidate_is_accepted(100.0, 200, 0.5) and not G.candidate_is_accepted(99.5, 200, 0.5) and G.candidate_is_accepted(110.0, 200, 0.55)


def test_match_configuration_per_bot_keys():
    from katago_b200.match_cli import bot_cfg
    cfg = {"maxVisits": "100", "maxVisits0": "50", "cpuctExploration1": "2.0", "botName0": "a", "botName1": "b", "nnModelFile0": "x", "numBots": "2",
           "koRules": "SIMPLE", "cudaDeviceToUseModel0Thread0": "0"}
    assert bot_cfg(cfg, 0) == {"maxVisits": "50", "numBots": "2", "koRules": "SIMPLE", "cudaDeviceToUseModel0Thread0": "0"}
    assert bot_cfg(cfg, 1) == {"maxVisits": "100", "numBots": "2", "koRules": "SIMPLE", "cudaDeviceToUseModel0Thread0": "0", "cpuctExploration": "2.0"}


GATE_CFG = """numGameThreads = 8
maxMovesPerGame = 70
numGamesPerGating = {games}
koRules = SIMPLE,POSITIONAL
scoringRules = AREA
taxRules = NONE
multiStoneSuicideLegals = false,true
hasButtons = false
bSizes = 7,9
bSizeRelProbs = 1,2
komiMean = 6.5
komiStdev = 0.5
maxVisits = {visits}
nnCacheSizePowerOfTwo = 12
chosenMoveTemperatureEarly = 0.5
chosenMoveTemperatureHalflife = 19
chosenMoveTemperature = 0.2
useLcbForSelection = true
lcbStdevs = 5.0
minVisitPropForLCB = 0.15
staticScoreUtilityFactor = 0.00
dynamicScoreUtilityFactor = 0.25
dynamicScoreCenterZeroWeight = 0.25
dynamicScoreCenterScale = 0.50
cpuctExploration = 1.1
cpuctExplorationLog = 0.0
valueWeightExponent = 0.5
subtreeValueBiasFactor = 0.35
subtreeValueBiasWeightExponent = 0.8
useNonBuggyLcb = true
useGraphSearch = true
"""


@pytest.mark.gpu
def test_two_loops_play_the_same_games_move_for_move(tmp_models):
    """Both loops hold every game: after each pump the boards, players to move and move numbers of slot g agree in the two loops, on
    boards of different sizes, across game ends (the mirror loop restarts the slot with the same next setup)."""
    from katago_b200 import NeuralNet, SelfPlay
    from katago_b200.game_initializer import GameInitializer
    loops, owned = [], []
    for i, name in enumerate(("tiny_reg", "tiny_nbt")):
        lm = NeuralNet.loadModelFile(tmp_models[name])
        ctx = NeuralNet.createComputeContext([0], 9, 9, True, lm)
        h = NeuralNet.createComputeHandle(ctx, lm, 8, False, True, 0)
        owned += [h, ctx]
        loops.append(SelfPlay(h, 6, 12 + 4 * i, komi=7.5, max_moves=40, seed=3 + i, use_graph_search=True, value_weight_exponent=0.5,
                              debug_hold_at_max_visits=True, use_play_selection=True, chosen_move_temperature=0.2, chosen_move_temperature_early=0.5))
    init = GameInitializer([(5, 5), (7, 7), (9, 9), (9, 7)], [1, 1, 1, 1], ko_rules=(0, 1), multi_stone_suicide_legals=(False, True), komi_mean=6.5, komi_stdev=1.0, seed=4)
    games = []
    mp = MatchPlay(loops, ["reg", "nbt"], 14, init, on_game=lambda slot, game, bn, wn, res: games.append((slot, bn, wn, res, game)))
    for _ in range(3000):
        mp.pump(4)
        for g in range(6):
            (ca, ia), (cb, ib) = loops[0].game(g), loops[1].game(g)
            assert np.array_equal(ca, cb) and ia["move_num"] == ib["move_num"] and ia["black_to_move"] == ib["black_to_move"], (g, ia, ib)
        assert np.array_equal(loops[0].game_setups()[0], loops[1].game_setups()[0]) and np.array_equal(loops[0].komi_values()[0], loops[1].komi_values()[0])
        if mp.done():
            break
    assert mp.games_tallied == 14 and abs(sum(mp.win_points) - 14) < 1e-9
    sizes = {(gm.x_size, gm.y_size) for _, _, _, _, gm in games}
    assert len(sizes) >= 2 and all(len(gm.moves) >= 2 for _, _, _, _, gm in games)
    for sp in loops:
        sp.free()
    for o in owned:
        o.free()


@pytest.mark.gpu
def test_gatekeeper_accepts_a_trained_net_over_a_random_one_and_rejects_the_reverse(tmp_path, golden_dir):
    """The whole command on the device: candidate = the trained g170-b6c96 net of the reference's test suite, baseline = a random-weight
    net: accepted (it wins nearly every game at 7x7 / 9x9 with 24 visits); then a random candidate against the trained net: rejected."""
    import shutil
    from katago_b200 import modelgen
    trained = os.path.join(golden_dir, "models", "g170-b6c96-s175395328-d26788732.bin.gz")
    test, acc, rej, sgf = (tmp_path / d for d in ("test", "accepted", "rejected", "sgf"))
    for d in (test, acc, rej):
        d.mkdir()
    modelgen.write_model(str(acc / "random0.bin"), "tiny_reg", seed=3)
    shutil.copy(trained, test / "trained1.bin.gz")
    os.utime(test / "trained1.bin.gz", (time.time() + 5, time.time() + 5))
    cfg = tmp_path / "gate.cfg"
    cfg.write_text(GATE_CFG.format(games=10, visits=24))
    args = ["-config", str(cfg), "-test-models-dir", str(test), "-sgf-output-dir", str(sgf), "-accepted-models-dir", str(acc), "-rejected-models-dir", str(rej),
            "-selfplay-dir", str(tmp_path / "selfplay"), "-quit-if-no-nets-to-test", "-games-per-gpu", "8", "-required-candidate-win-prop", "0.6"]
    assert G.main(args) == 0
    assert (acc / "trained1.bin.gz").exists() and not os.listdir(test) and (tmp_path / "selfplay" / "trained1" / "tdata").is_dir()
    records = [l for f in os.listdir(sgf / "trained1") for l in open(sgf / "trained1" / f)]
    assert 6 <= len(records) <= 10 and all(("PB[trained1]" in r) != ("PW[trained1]" in r) for r in records)      # early stop once the verdict is fixed
    wins = sum(1 for r in records if ("PB[trained1]" in r and "RE[B+" in r) or ("PW[trained1]" in r and "RE[W+" in r))
    assert wins >= 6, (wins, len(records))
    # a random net newer than the accepted trained net: plays and loses
    modelgen.write_model(str(test / "random2.bin"), "tiny_nbt", seed=9)
    os.utime(test / "random2.bin", (time.time() + 50, time.time() + 50))
    assert G.main(args) == 0
    assert (rej / "random2.bin").exists() and not (acc / "random2.bin").exists()


@pytest.mark.gpu
def test_match_command_plays_two_named_bots(tmp_path, tmp_models):
    from katago_b200 import match_cli
    cfg = tmp_path / "match.cfg"
    cfg.write_text(GATE_CFG.format(games=6, visits=16).replace("numGamesPerGating", "numGamesTotal") +
                   f"numBots = 2\nbotName0 = reg\nbotName1 = nbt\nnnModelFile0 = {tmp_models['tiny_reg']}\nnnModelFile1 = {tmp_models['tiny_nbt']}\nmaxVisits1 = 24\n")
    out = tmp_path / "sgfs"
    assert match_cli.main(["-config", str(cfg), "-sgf-output-dir", str(out), "-log-file", str(tmp_path / "match.log"), "-games-per-gpu", "4"]) == 0
    records = [l for f in os.listdir(out) for l in open(out / f)]
    assert len(records) == 6 and all(("PB[reg]PW[nbt]" in r) or ("PB[nbt]PW[reg]" in r) for r in records)
    assert 2 <= sum("PB[reg]" in r for r in records) <= 4          # a slot's bots swap colours from game to game
    log = open(tmp_path / "match.log").read()
    assert "Match finished" in log and "maxVisits 24" in log and "maxVisits 16" in log


@pytest.mark.gpu
def test_match_with_resignation_between_a_deep_and_a_shallow_search(tmp_path, golden_dir):
    """Two bots on the same trained net, 48 visits against 4, allowResignation: games may end by resignation - then the loser is the player
    who made the last move (a player resigns after its own move), the record says "+R", and both loops carry on with the slot's next game."""
    import re
    from katago_b200 import match_cli
    model = os.path.join(golden_dir, "models", "g170-b6c96-s175395328-d26788732.bin.gz")
    cfg = tmp_path / "match.cfg"
    cfg.write_text(GATE_CFG.format(games=10, visits=48).replace("numGamesPerGating", "numGamesTotal").replace("bSizes = 7,9", "bSizes = 9").replace("bSizeRelProbs = 1,2", "bSizeRelProbs = 1") +
                   f"numBots = 2\nbotName0 = deep\nbotName1 = shallow\nnnModelFile = {model}\nmaxVisits1 = 4\nallowResignation = true\nresignThreshold = -0.80\nresignConsecTurns = 3\n")
    out = tmp_path / "sgfs"
    assert match_cli.main(["-config", str(cfg), "-sgf-output-dir", str(out), "-log-file", str(tmp_path / "match.log"), "-games-per-gpu", "6"]) == 0
    records = [l for f in os.listdir(out) for l in open(out / f)]
    assert len(records) == 10
    resigned = 0
    for r in records:
        res = re.search(r"RE\[([^\]]*)\]", r).group(1)
        moves = re.findall(r";([BW])\[", r)
        if res.endswith("+R"):
            resigned += 1
            assert moves and moves[-1] != res[0] and len(moves) >= 1 + 81 // 5        # the last mover lost; not before turn 1 + area / 5
    log = open(tmp_path / "match.log").read()
    print(f"{resigned} of 10 games ended by resignation")
    assert "Match finished" in log


def test_resignation_rule_equals_the_reference_games(golden_dir):
    """Seven games of the reference's Play::runGame with allowResignation (tests/golden/make_resign_fixture.py: thresholds -0.02 .. -0.6, 1-4 consecutive
    turns, 5x5 .. 13x13): replaying the root win/loss values through `should_resign`, the rule fires exactly at the move after which the
    reference's game was resigned - by the player who made that move, won by the other - and never in the game that ended otherwise."""
    import gzip, json
    from katago_b200.match_play import should_resign
    games = json.loads(gzip.open(os.path.join(golden_dir, "resign.json.gz")).read())
    assert sum(g["resigned"] for g in games) >= 5 and any(not g["resigned"] for g in games)
    for g in games:
        thr, consec = g["resign"].split(",")
        thr, consec, area = float(thr), int(consec), g["size"] ** 2
        fired = [i for i in range(g["turns"]) if should_resign(g["rootWinLoss"][:i + 1], i, area, i % 2 == 0, thr, consec)]
        if g["resigned"]:
            last = g["turns"] - 1
            assert fired and fired[0] == last, (g["size"], g["resign"], fired, last)
            assert g["winner"] == (2 if last % 2 == 0 else 1)          # the mover of the last move (black on even indices) lost: P_WHITE = 2, P_BLACK = 1
        else:
            assert fired == [], (g["size"], g["resign"], fired)
