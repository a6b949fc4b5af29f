"""Generates tests/golden/ladders_*.npz: NNInputs::fillRowV7 rows of the REFERENCE (oracle/_ref/kgref_driver ladderrows) for positions
chosen to exercise the ladder reader (planes 14-17, iterLadders / searchIsLadderCaptured): every legal position of the tiny boards,
sampled small boards, constructed ladders under every symmetry and in several frames, dense boards with many searches, and positions
right after a ko capture (a set-up move list never captures, so only these have a simple-ko point).

Every position is set up by a move list that places its stones in alternating colours (passes for the side with fewer stones, never two
in a row): when every chain of the final position has a liberty, no partial position captures anything, because the missing stones and
the final empty points are all still empty.  The side to move is set by which colour plays last.  The generator checks that the dumped
planes 1/2 equal the intended diagram.

Per position the npz holds X, Y, the frame NX x NY, ko rule, multi-stone suicide, the move list (int8, padded with -128), the reference
row (22 planes, bit-packed with np.packbits, padded to the 19x19 frame), the 19 globals, whether the position has a simple-ko point, a name,
and designed outcomes (`exp`: (position, x, y, plane, value) rows at points a diagram was built to decide; `exact17`: the number of
plane-17 points) that the CPU test checks against the reference.
Run after build(): python tests/golden/make_ladder_fixtures.py"""
import itertools, os, subprocess, tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
DRIVER = os.path.join(HERE, "..", "..", "oracle", "_ref", "kgref_driver")
ROWBITS = 19 * 19 * 22
PAD = -128


# ---------------------------------------------------------------- boards
def chains(board):
    """[(colour, set of points, set of liberties)] of a [Y, X] int array (0 empty, 1 black, 2 white)."""
    Y, X = board.shape
    seen = np.zeros_like(board, bool)
    out = []
    for y in range(Y):
        for x in range(X):
            c = board[y, x]
            if c == 0 or seen[y, x]:
                continue
            pts, libs, stack = set(), set(), [(x, y)]
            seen[y, x] = True
            while stack:
                px, py = stack.pop()
                pts.add((px, py))
                for qx, qy in ((px - 1, py), (px + 1, py), (px, py - 1), (px, py + 1)):
                    if 0 <= qx < X and 0 <= qy < Y:
                        if board[qy, qx] == 0:
                            libs.add((qx, qy))
                        elif board[qy, qx] == c and not seen[qy, qx]:
                            seen[qy, qx] = True
                            stack.append((qx, qy))
            out.append((int(c), pts, libs))
    return out


def is_legal_position(board):
    return all(libs for _, _, libs in chains(board))


def setup_moves(board, black_to_move):
    """Alternating-colour move list that builds `board` from the empty board and leaves the given side to move."""
    Y, X = board.shape
    stones = {1: [(x, y) for y in range(Y) for x in range(X) if board[y, x] == 1],
              2: [(x, y) for y in range(Y) for x in range(X) if board[y, x] == 2]}
    moves, turn = [], 1
    while stones[1] or stones[2]:
        moves.append(stones[turn].pop(0) if stones[turn] else None)
        turn = 3 - turn
    if (turn == 1) != black_to_move:
        moves.append(None)   # the last move was a stone (or the list is empty): one pass flips the side to move
    return moves


def parse(diagram):
    rows = [r.split() for r in diagram.strip().splitlines()]
    return rows


# ---------------------------------------------------------------- constructed ladders
# A diagram is the corner region of the board at (0, 0) (its top and left sides are board edges).  X / O are black / white stones, '.'
# empty; B / W are black / white stones of a chain whose ladder status is designed ("lad" = laddered, "free" = not); lowercase letters
# mark empty points, and "work" lists the letters that must be exactly plane 17 (working moves against the opponent's 2-liberty chains,
# for the side to move).  `chase` lists the first moves of the chase (diagram coordinates): each prefix is played after the set-up
# as a further position.
def _long_ladder():
    """The working ladder's shape started at the far corner of 19x19: the chase runs the full diagonal."""
    g = [["."] * 19 for _ in range(19)]
    g[17][17] = "W"; g[17][18] = "X"; g[18][16] = "X"; g[18][17] = "X"; g[16][17] = "a"
    return "\n".join(" ".join(r) for r in g)


# the first moves of the working ladder's chase (diagram coordinates), for the history variants: planes 15/16 then come from boards
# that hold ladders
CHASE = [(7, 4), (6, 5), (5, 5), (6, 4), (6, 3), (5, 4), (4, 4), (5, 3)]
CONSTRUCTED = [
    # a working ladder: white's 2-liberty stone, black to move; the chase runs to the top-left corner, 'a' is the one working move
    dict(name="working", black=True, lad="W", work="a", chase=CHASE, d="""
        . . . . . . . . . .
        . . . . . . . . . .
        . . . . . . . . . .
        . . . . . . . . . .
        . . . . . . . a . .
        . . . . . . . W X .
        . . . . . . X X . .
        . . . . . . . . . ."""),
    dict(name="working_long", black=True, lad="W", work="a", chase=[(x + 10, y + 12) for x, y in CHASE], d=_long_ladder()),
    # the same ladder broken by a white stone on the diagonal: not laddered, no working move
    dict(name="breaker_near", black=True, free="W", work="", d="""
        . . . . . . . . . .
        . . . . . . . . . .
        . . . O . . . . . .
        . . . . . . . . . .
        . . . . . . . . . .
        . . . . . . . W X .
        . . . . . . X X . .
        . . . . . . . . . ."""),
    dict(name="breaker_far", black=True, free="W", work="", d="""
        . . . . . . . . . .
        . . O . . . . . . .
        . . . . . . . . . .
        . . . . . . . . . .
        . . . . . . . . . .
        . . . . . . . W X .
        . . . . . . X X . .
        . . . . . . . . . ."""),
    # a black stone on the path makes the ladder work sooner
    dict(name="attacker_on_path", black=True, lad="W", work="a", d="""
        . . . . . . . . . .
        . . . . . . . . . .
        . . . X . . . . . .
        . . . . . . . . . .
        . . . . . . . a . .
        . . . . . . . W X .
        . . . . . . X X . .
        . . . . . . . . . ."""),
    # white in atari whose extension fails, but it captures a black stone in atari next to it ('c'): escaped.  The control without the
    # capture is laddered.
    dict(name="escape_capture_single", black=True, free="W", d="""
        . . . . . . . .
        . . . . . . . .
        . . . . . c . .
        . . . . O X O .
        . . . . X W X .
        . . . . X . X .
        . . . . . . . ."""),
    dict(name="escape_capture_control", black=True, lad="W", d="""
        . . . . . . . .
        . . . . . . . .
        . . . . . . . .
        . . . . . X . .
        . . . . X W X .
        . . . . X . X .
        . . . . . . . ."""),
    # ... capturing a two-stone black chain in atari
    dict(name="escape_capture_chain", black=True, free="W", d="""
        . . . . . . . .
        . . . . . c . .
        . . . . O X O .
        . . . . O X O .
        . . . . X W X .
        . . . . X . X .
        . . . . . . . ."""),
    # the working ladder in a smaller corner region, so that it also fits the 13x7 and 7x13 boards and a 5x5 board inside a 19x19 frame
    dict(name="working_compact", black=True, lad="W", work="a", d="""
        . . . . .
        . . . . .
        . . . a .
        . . . W X
        . . X X ."""),
    # a 2-liberty stone on the edge that both attacker moves capture: two working moves
    dict(name="two_working_moves", black=True, lad="W", work="ab", d="""
        . X W a . .
        . X b X . .
        . . . . . ."""),
    # non-adjacent liberties that both have 3 empty neighbours: the attacker's pruning gives up at once
    dict(name="pruning_both_open", black=True, free="W", work="", d="""
        . . . . . . .
        . . . . . . .
        . . . . . . .
        . . X W X . .
        . . . . . . .
        . . . . . . ."""),
    # a 2-liberty white chain whose liberty 'b' works and whose other liberty (the corner) is suicide for black
    dict(name="first_move_suicide", black=True, lad="W", work="b", d="""
        . W X . . .
        W W X . . .
        b X . . . .
        X . . . . .
        . . . . . ."""),
]


def transforms(X, Y):
    """Board symmetries as point maps; rectangles keep only the four that preserve the shape."""
    out = []
    for t in range(8):
        flip_x, flip_y, swap = t & 1, (t >> 1) & 1, (t >> 2) & 1
        if swap and X != Y:
            continue
        def f(x, y, fx=flip_x, fy=flip_y, sw=swap):
            if sw:
                x, y = y, x
            return (X - 1 - x if fx else x, Y - 1 - y if fy else y)
        out.append((t, f))
    return out


def constructed_positions():
    """(name, X, Y, NX, NY, ko, multi, board, black_to_move, then, checks, exact17)"""
    out = []
    frames = [(19, 19, 19, 19), (13, 7, 13, 7), (7, 13, 7, 13), (9, 9, 19, 19), (13, 7, 19, 19), (10, 10, 10, 10), (5, 5, 19, 19)]
    for c in CONSTRUCTED:
        rows = parse(c["d"])
        h, w = len(rows), len(rows[0])
        for (X, Y, NX, NY) in frames:
            if w > X or h > Y:
                continue
            for t, f in transforms(X, Y):
                board = np.zeros((Y, X), np.int8)
                labels = {}
                for y in range(h):
                    for x in range(w):
                        ch = rows[y][x]
                        px, py = f(x, y)
                        if ch in "XB":
                            board[py, px] = 1
                        elif ch in "OW":
                            board[py, px] = 2
                        if ch not in ".XO":
                            labels.setdefault(ch, []).append((px, py))
                checks = []
                for key, val in (("lad", 1), ("free", 0)):
                    for ch in c.get(key, ""):
                        checks += [(px, py, 14, val) for px, py in labels[ch]]
                exact17 = -1
                if "work" in c:
                    pts = [p for ch in c["work"] for p in labels[ch]]
                    checks += [(px, py, 17, 1) for px, py in pts]
                    exact17 = len(pts)
                assert is_legal_position(board), c["name"]
                ko = t % 2
                name = f"{c['name']}:{X}x{Y}in{NX}x{NY}:t{t}"
                out.append((name, X, Y, NX, NY, ko, 1, board, c["black"], [], checks, exact17))
                # history: a few moves into the chase, the hunted chain is still laddered
                for k in range(1, len(c.get("chase", [])) + 1):
                    then = [f(*m) for m in c["chase"][:k]]
                    out.append((f"{name}:chase{k}", X, Y, NX, NY, ko, 1, board, c["black"], then, [ch for ch in checks if ch[2] == 14], -1))
    return out


# ---------------------------------------------------------------- random positions
def random_position(rng, X, Y, density):
    board = (rng.random((Y, X)) < density).astype(np.int8) * rng.integers(1, 3, size=(Y, X)).astype(np.int8)
    while True:
        dead = [pts for _, pts, libs in chains(board) if not libs]
        if not dead:
            return board
        for x, y in dead[rng.integers(len(dead))]:
            board[y, x] = 0


def low_lib_chains(board):
    return sum(1 for _, _, libs in chains(board) if 1 <= len(libs) <= 2)


# ---------------------------------------------------------------- reference
def run_reference(entries):
    """entries: (X, Y, NX, NY, ko, multi, moves) -> list of (status, slowest_us, (sx, sy), bits[NY*NX*22] uint8, glob[19])."""
    d = tempfile.mkdtemp()
    src, dst = os.path.join(d, "in.txt"), os.path.join(d, "out.bin")
    with open(src, "w") as fh:
        for X, Y, NX, NY, ko, multi, moves in entries:
            fh.write(f"{X} {Y} {NX} {NY} {ko} {multi} " + " ".join("pass" if m is None else f"{m[0]},{m[1]}" for m in moves) + "\n")
    subprocess.check_call([DRIVER, "ladderrows", src, dst], stderr=subprocess.DEVNULL)
    raw = open(dst, "rb").read()
    out, off = [], 0
    for X, Y, NX, NY, *_ in entries:
        n = NX * NY * 22
        status, slow, sx, sy = np.frombuffer(raw, "<i4", 1, off)[0], np.frombuffer(raw, "<f4", 1, off + 4)[0], *np.frombuffer(raw, "<i4", 2, off + 8)
        bits = np.frombuffer(raw, np.uint8, n, off + 16)
        glob = np.frombuffer(raw, "<f4", 19, off + 16 + n)
        out.append((int(status), float(slow), (int(sx), int(sy)), bits, glob))
        off += 16 + n + 19 * 4
    assert off == len(raw)
    return out


def save(tag, items):
    """items: dicts with name X Y NX NY ko multi board black moves checks exact17."""
    entries = [(it["X"], it["Y"], it["NX"], it["NY"], it["ko"], it["multi"], it["moves"]) for it in items]
    ref = run_reference(entries)
    n = len(items)
    maxlen = max(1, max(len(it["moves"]) for it in items))
    moves = np.full((n, maxlen, 2), PAD, np.int8)
    rows = np.zeros((n, ROWBITS // 8 + (ROWBITS % 8 > 0)), np.uint8)
    glob = np.zeros((n, 19), np.float32)
    exp = []
    for i, (it, (status, us, sxy, bits, gl)) in enumerate(zip(items, ref)):
        assert status == 0, (tag, it["name"], "a set-up move was illegal")
        for k, m in enumerate(it["moves"]):
            moves[i, k] = (-1, -1) if m is None else m
        X, Y, NX = it["X"], it["Y"], it["NX"]
        planes = bits.reshape(it["NY"], NX, 22)
        if it.get("board") is not None:
            want = it["board"]
            assert np.array_equal(planes[:Y, :X, 1] + planes[:Y, :X, 2], (want != 0).astype(np.uint8)), (tag, it["name"])
            own = 1 if it["black"] else 2   # plane 1 = the side to move's stones
            assert np.array_equal(planes[:Y, :X, 1], (want == own).astype(np.uint8)), (tag, it["name"])
        rows[i] = np.packbits(np.concatenate([bits, np.zeros(ROWBITS - len(bits), np.uint8)]))
        glob[i] = gl
        for (x, y, pl, val) in it.get("checks", []):
            exp.append((i, x, y, pl, val))
    exp = np.array(exp, np.int16).reshape(-1, 5)
    path = os.path.join(HERE, f"ladders_{tag}.npz")
    np.savez_compressed(path, X=np.array([it["X"] for it in items], np.int8), Y=np.array([it["Y"] for it in items], np.int8),
                        NX=np.array([it["NX"] for it in items], np.int8), NY=np.array([it["NY"] for it in items], np.int8),
                        ko=np.array([it["ko"] for it in items], np.int8), multi=np.array([it["multi"] for it in items], np.int8),
                        moves=moves, rows=rows, glob=glob,
                        simple_ko=np.array([bool(it.get("simple_ko", False)) for it in items]),
                        name=np.array([it["name"] for it in items]), exp=exp,
                        exact17=np.array([it.get("exact17", -1) for it in items], np.int16))
    lad = sum(int(r[3].reshape(-1, 22)[:, 14].sum()) for r in ref)
    p17 = sum(int(r[3].reshape(-1, 22)[:, 17].sum()) for r in ref)
    print(f"ladders_{tag}.npz: {n} positions, plane-14 bits {lad}, plane-17 bits {p17}, slowest search {max(r[1] for r in ref):.0f} us (printed only), "
          f"{os.path.getsize(path) // 1024} KB")
    return ref


def item(name, board, black, X, Y, NX=None, NY=None, ko=0, multi=1, then=(), **kw):
    return dict(name=name, X=X, Y=Y, NX=NX or X, NY=NY or Y, ko=ko, multi=multi, board=board if not then else None, black=black,
                moves=setup_moves(board, black) + list(then), **kw)


def tiny():
    items = []
    for (X, Y) in ((2, 2), (3, 2), (3, 3)):
        count = 0
        for cells in itertools.product((0, 1, 2), repeat=X * Y):
            board = np.array(cells, np.int8).reshape(Y, X)
            if not is_legal_position(board):
                continue
            for black in (True, False):
                items.append(item(f"tiny{X}x{Y}:{count}:{'b' if black else 'w'}", board, black, X, Y, 3, 3, ko=count % 2,
                                  multi=(count // 2) % 2))
            count += 1
        print(f"{X}x{Y}: {count} legal positions")
    return items


def sampled(n_per_size, seed=5):
    rng = np.random.default_rng(seed)
    items = []
    for (X, Y) in ((4, 3), (4, 4), (5, 5)):
        k = 0
        while k < n_per_size:
            board = random_position(rng, X, Y, rng.uniform(0.45, 0.85))
            if low_lib_chains(board) == 0 and rng.random() < 0.8:
                continue
            items.append(item(f"small{X}x{Y}:{k}", board, bool(rng.integers(2)), X, Y, ko=int(rng.integers(3)), multi=int(rng.integers(2))))
            k += 1
    return items


def ko_capture(board, colour):
    """Points where `colour` captures exactly one single stone and leaves a simple ko (its stone alone, with that one liberty)."""
    Y, X = board.shape
    out = []
    for y in range(Y):
        for x in range(X):
            if board[y, x]:
                continue
            # the capturing stone ends up alone with the captured point as its one liberty: every neighbour is an opponent stone
            if any(board[qy, qx] != 3 - colour for qx, qy in ((x - 1, y), (x + 1, y), (x, y - 1), (x, y + 1)) if 0 <= qx < X and 0 <= qy < Y):
                continue
            b = board.copy()
            b[y, x] = colour
            dead = [pts for c, pts, libs in chains(b) if c != colour and not libs]
            if len(dead) != 1 or len(dead[0]) != 1:
                continue
            (dx, dy), = dead[0]
            b[dy, dx] = 0
            mine = [(pts, libs) for c, pts, libs in chains(b) if (x, y) in pts][0]
            if len(mine[0]) == 1 and mine[1] == {(dx, dy)}:
                out.append(((x, y), (dx, dy), b))
    return out


def ko_positions(n, seed=13):
    """Random positions whose last move captured a single stone and left a simple-ko point, mostly ones where a 2-liberty chain of the
    capturer has the ko point as a liberty: the attacker's first move there is illegal for the reference (iterLadders does not clear
    the game's ko before searchIsLadderCapturedAttackerFirst2Libs).  Boards from 4x4 to 19x19, some inside a 19x19 frame, all ko rules."""
    rng = np.random.default_rng(seed)
    shapes = [(4, 4, 4, 4), (5, 5, 5, 5), (6, 5, 6, 5), (7, 7, 7, 7), (9, 9, 9, 9), (5, 5, 19, 19), (9, 9, 19, 19), (13, 7, 19, 19),
              (19, 19, 19, 19)]
    items, k = [], 0
    while len(items) < n:
        X, Y, NX, NY = shapes[k % len(shapes)]
        k += 1
        board = random_position(rng, X, Y, rng.uniform(0.5, 0.8))
        colour = int(rng.integers(1, 3))
        kos = ko_capture(board, colour)
        if not kos:
            continue
        (mx, my), kp, after = kos[int(rng.integers(len(kos)))]
        on_ko = any(len(libs) == 2 and kp in libs for c, _, libs in chains(after) if c == colour)
        if not on_ko and rng.random() < 0.7:
            continue
        items.append(item(f"ko{X}x{Y}in{NX}x{NY}:{k}{':kolib' if on_ko else ''}", board, colour == 1, X, Y, NX, NY,
                          ko=int(rng.integers(3)), multi=int(rng.integers(2)), then=[(mx, my)], simple_ko=True))
    return items


def constructed():
    items = []
    for (name, X, Y, NX, NY, ko, multi, board, black, then, checks, exact17) in constructed_positions():
        items.append(item(name, board, black, X, Y, NX, NY, ko=ko, multi=multi, then=then, checks=checks, exact17=exact17))
    return items


def heavy(n_try, keep, seed=9):
    """Dense random 19x19 and 13x13 positions; keeps the ones with the most 1-2 liberty chains (40 or more each), i.e. the most
    searches per position, so that every one of the device's 8 warps takes several.  The choice uses nothing but the boards: the
    searches' times would not regenerate the same fixture twice."""
    rng = np.random.default_rng(seed)
    cand = []
    for i in range(n_try):
        S = 19 if i % 2 == 0 else 13
        board = random_position(rng, S, S, rng.uniform(0.6, 0.8))
        cand.append(item(f"dense{S}:{i}", board, bool(rng.integers(2)), S, S, 19, 19, ko=0, multi=1))
    nlow = [low_lib_chains(it["board"]) for it in cand]
    order = np.argsort([-k for k in nlow], kind="stable")[:keep]
    assert min(nlow[i] for i in order) >= 40
    return [cand[i] for i in sorted(order)]


if __name__ == "__main__":
    save("tiny", tiny())
    save("small", sampled(3000))
    save("constructed", constructed())
    save("heavy", heavy(400, 64))
    save("ko", ko_positions(3000))
