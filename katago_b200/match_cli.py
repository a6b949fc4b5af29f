"""`python -m katago_b200.match_cli` - the reference's `katago match` command (command/match.cpp) for two bots on the device loops
(SURVEY.md §8f row 4).

    python -m katago_b200.match_cli -config match.cfg -sgf-output-dir DIR [-log-file FILE] [-games-per-gpu N] [-override-config k=v,..]

Reads the reference's match configuration: `numBots = 2`, `botName0/1`, `nnModelFile0/1` (or one `nnModelFile` for both),
`numGamesTotal`, the shared search / rules / board-size / komi keys of the selfplay mapping, and per-bot search keys with the bot's index
appended (`maxVisits0`, `cpuctExploration1`, ... - Setup::loadParams with SETUP_FOR_MATCH).  The bots alternate colours; results are
logged in the reference's words and written one record per line to `<sgf-output-dir>/<16 hex>.sgfs`.  Not built: more than two bots,
`secondaryBots` / `extraPairs` pairing tables, per-bot time controls."""
import argparse
import os
import sys


def bot_cfg(cfg, idx):
    """The configuration bot `idx` sees: a search key with the bot's index appended (`maxVisits0`) overrides the shared one
    (Setup::loadParams with SETUP_FOR_MATCH, program/setup.cpp); keys of other bots, bot names and model files are left out."""
    import re
    from . import selfplay_cli as C
    per_bot = set(C._SEARCH_KEYS) | {"botName", "nnModelFile"}
    out = {}
    for k, v in cfg.items():
        m = re.match(r"^(.*?)(\d+)$", k)
        if k in ("botName", "nnModelFile") or (m and m.group(1) in per_bot):
            continue
        out[k] = v
    for k in C._SEARCH_KEYS:
        if k + str(idx) in cfg:
            out[k] = cfg[k + str(idx)]
    return out


def match_default_note(cfg):
    """The log line for uncertainty weighting / noise pruning left unset: the reference's `katago match` loads its bots with
    SETUP_FOR_MATCH, where both default to true (program/setup.cpp:522-544); here an unset key stays off, so that existing match
    configurations keep playing the same games.  None when every bot sets both."""
    import re
    absent = [k for k in ("useUncertainty", "useNoisePruning") if not any(c == k or re.fullmatch(k + r"\d+", c) for c in cfg)]
    if not absent:
        return None
    return (f"[config] {' and '.join(absent)} not set: off here, while the reference's katago match defaults "
            f"{'them' if len(absent) > 1 else 'it'} to true; set {', '.join(k + ' = true' for k in absent)} to search like it")


def main(argv=None):
    ap = argparse.ArgumentParser(prog="katago_b200.match_cli", description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("-config", required=True)
    ap.add_argument("-sgf-output-dir", required=True)
    ap.add_argument("-log-file", default="")
    ap.add_argument("-games-per-gpu", type=int, default=128)
    ap.add_argument("-override-config", default="")
    ap.add_argument("-seed", type=int, default=0)
    a = ap.parse_args(argv)
    from . import selfplay_cli as C
    from .game_initializer import GameInitializer
    from .match_play import MatchPlay
    from .nn_backend import NeuralNet, SelfPlay
    from .npz_writer import write_sgf
    cfg = C.parse_cfg(a.config)
    for kv in [s for s in a.override_config.split(",") if s.strip()]:
        k, v = kv.split("=", 1)
        cfg[k.strip()] = v.strip()
    logf = open(a.log_file, "a") if a.log_file else None

    def log(s):
        print(s, file=sys.stderr, flush=True)
        if logf:
            logf.write(s + "\n"); logf.flush()
    if int(cfg.get("numBots", 2)) != 2:
        raise ValueError("match: exactly two bots are built (numBots = 2)")
    for k in ("secondaryBots", "extraPairs", "includeBots"):
        if k in cfg:
            raise ValueError(f"match: {k} is not built")
    names = [cfg.get(f"botName{i}") for i in range(2)]
    if None in names:
        raise ValueError("If more than one bot, must specify botName0, botName1,... individually")
    files = [cfg.get(f"nnModelFile{i}", cfg.get("nnModelFile")) for i in range(2)]
    if None in files:
        raise ValueError("match: nnModelFile0 / nnModelFile1 (or nnModelFile) required")
    total = int(cfg.get("numGamesTotal", 0))
    if total <= 0:
        raise ValueError("match: numGamesTotal must be positive")
    games = max(2, min(a.games_per_gpu, int(cfg.get("numGameThreads", a.games_per_gpu)), total))
    gpu = int(os.environ.get("LOCAL_RANK", "0"))
    log("Match Engine starting...")
    note = match_default_note(cfg)
    if note:
        log(note)
    loops, owned, data0 = [], [], None
    for i in range(2):
        kw, data, report = C.selfplay_kwargs_from_cfg({k: v for k, v in bot_cfg(cfg, i).items() if k not in ("numBots", "numGamesTotal")})
        if i == 0:
            data0 = data
            for line in report["fixed"]:
                log("[config] " + line)
            if report["not_built"]:
                log("[config] NOT BUILT, ignored: " + "; ".join(report["not_built"]))
        lm = NeuralNet.loadModelFile(files[i])
        ctx = NeuralNet.createComputeContext([gpu], data0["board_size"], data0["board_size"], True, lm)
        h = NeuralNet.createComputeHandle(ctx, lm, games, False, True, gpu)
        owned += [h, ctx]
        max_visits = kw.pop("max_visits", 500)
        loops.append(SelfPlay(h, games, max_visits, komi=data["komi"], seed=a.seed * 7919 + 31 * i + 1, debug_hold_at_max_visits=True, **kw))
        log(f"Loaded neural net {i} from: {files[i]} for bot {names[i]} (maxVisits {max_visits})")
    sink = C.SgfSink(a.sgf_output_dir, f"match{a.seed}", names[0], names[1])
    wins = {n: 0 for n in names}
    draws = [0]

    def on_game(slot, game, b_name, w_name, result):
        with open(sink.path, "a") as f:
            f.write(write_sgf(game, b_name, w_name) + "\n")
        if result.startswith("B"):
            wins[b_name] += 1
        elif result.startswith("W"):
            wins[w_name] += 1
        else:
            draws[0] += 1
        log(f"Game {mp.games_tallied - 1}: {b_name} (black) vs {w_name} (white): {result} in {len(game.moves)} moves")
    mp = MatchPlay(loops, names, total, GameInitializer(seed=a.seed ^ 0x4D617463, **data0["game_init"]), on_game=on_game,
                   draw_equivalent_wins_for_white=0.5, no_result_utility_for_white=0.0, allow_resignation=C._B(cfg.get("allowResignation", "false")),
                   resign_threshold=float(cfg.get("resignThreshold", -0.90)), resign_consec_turns=int(cfg.get("resignConsecTurns", 5)))
    try:
        mp.run()
    except KeyboardInterrupt:
        pass
    log("Match finished: " + ", ".join(f"{n} {w} wins" for n, w in wins.items()) + f", {draws[0]} draws or void; points {mp.win_points[0]:.1f} - {mp.win_points[1]:.1f} in {mp.games_tallied} games")
    for sp in loops:
        sp.free()
    for o in owned:
        o.free()
    if logf:
        logf.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
