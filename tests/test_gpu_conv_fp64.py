"""The wgmma convolution and its fused epilogue against a float64 reference, with error bounds derived from an error model.

The reference is computed in float64 from exactly the operands the kernel receives: fp16(x) and fp16(w) in fp16 mode, and in split
mode (fp32-equivalent) the halves ah = fp16(x), al = fp16(x - ah), wh = fp16(w), wl = fp16(w - wh) that the input packing and the
weight packing write.  numpy's float16 rounds to nearest even and keeps subnormals, as __float2half_rn does; that matters, since wl is
subnormal for every weight with |w| < 0.25.  From those operands, in order:

    ideal = sum over taps of (ah*wh + al*wh + ah*wl)        (al = wl = 0 in fp16 mode)
    V     = ideal + ncbias[image] + R                        (R = the residual as the stream holds it: fp32, or rounded to fp16)
    raw   = mask * V,   z = V * bn_scale + bn_bias,   act = mask ? act(z) : 0

and sigma = sqrt(conv(x^2, w^2)) per output, the scale of the accumulation's rounding errors.

Bounds (every output; a row or channel the mask zeroes must be exactly zero):
  raw:  |got - raw| <= C_ACC * U * 2^-23 * sigma + 2^-22 * (|ideal| + |ncbias| + |R|) + half an ulp of the stored dtype at |V|.
        The first term is the tensor core's fp32 accumulation, which is not IEEE round-to-nearest: it truncates toward zero.  One
        output receives U = ceil(cin / 16) * taps * parts accumulator updates (parts = 3 in split mode), and each update can lose up
        to one fp32 ulp of a partial sum of size ~sigma, 2^-23 sigma, always toward zero, so the losses add up linearly in U.
        accumulate() emulates that hardware: each 16-channel step adds the exact sum of its products to the fp32 accumulator and
        truncates, in the kernel's order.  Over the case matrix its worst error is 0.5-1.9 U 2^-23 sigma, and C_ACC = 8 keeps it
        within a quarter of the bound.  On the H100 the ratio lands at 0.7-1.4x of the emulated one, case by case.  An IEEE fp32 GEMM
        would sit some 20x lower on the 3x3 split layers.  The second term is the fp32 rounding of the two epilogue additions.  The
        fp16 ulp includes the subnormal spacing 2^-24.
  split terms: the max bound cannot tell a lost split cross term from truncation on every layer: dropping al*wh or ah*wl costs
        up to 1e-3 sigma, and on a 3x3 192-channel split layer the bound is 3e-4 sigma.  Each cross term T (computed apart in
        float64) is therefore checked by its least-squares coefficient in the raw error, weighted by 1/sigma: c = <e, T> / <T, T>.
        A correct kernel's error is truncation, biased toward zero but unrelated to T, so c ~ 0.  A kernel that loses the term
        gives c = -1, and one that loses it on some taps or tiles gives minus that share.  |c| <= PROJ_BOUND = 1/16.  Kind 1 has no
        raw output, so there T is carried to the activation by act'(z) * bn_scale.
  lo:   in split mode, the coefficient of the reference's lo half, fp16(act - fp16(act)), in the activation error, with the same
        limit: a dropped or misplaced lo half gives about -1.
  act:  the error of z, ACT_LIPSCHITZ * (|bn_scale| * e_v + Z_ROUND |z|), with e_v the raw bound before storage; plus the
        activation formula's own error; plus the storage: half an fp16 ulp of |act| in fp16 mode, 2^-22 |act| + 2^-25 for hi + lo in
        split mode (lo is rounded to fp16 once; 2^-25 is half its subnormal spacing).
        Formula error, for mish and SiLU (identity and relu are exact): with r = act(z) / z in [0, 1],
            2^-20 * |z| * (1 + (|z| + 8) * r * (1 - r)).
        ex2.approx and rcp.approx are off by a few 2^-23 relatively, and the argument z * log2(e) is rounded: together an
        exponential of z + dz with |dz| <= (|z| + 8) * 2^-23, which moves act by |z| |r'(z)| |dz| <= 2 |z| r (1 - r) |dz|.  The rest
        is rounding of the products, at most a few 2^-23 |z|.  For z << 0 mish is computed as z - 2z / (e(e+2)+2), which cancels: its
        error is of order ulp(|z|), not ulp(|mish(z)|), and the |z| factor carries that.
  own:  where the kernel returns its fp32 raw (kind 4, and kinds 2-3 in split mode), act is also checked against the float64
        activation of the kernel's own raw, with the same bound minus the accumulation term: tight enough to see a dropped lo half.
  split structure: hi == fp16(hi + lo) and |lo| <= ulp(hi) / 2.  When |lo| is exactly ulp(hi) / 2 (lo rounded up to the halfway
        point), hi + lo is a tie and fp16 may round it to the even neighbour instead; that case only has to satisfy the second part.
Every check allows the rounding to the stored dtype in full and reports the rest of the error over the computation's bound: a
correctly rounded output may sit anywhere up to half an ulp from the exact value, so that rounding has no margin to give.

Epilogue kinds (kgb_test_conv_ex): 0 raw fp32 only, 1 act only, 2 residual + raw stream + act, 3 raw stream + act, 4 kind 2 with an
fp32 stream in fp16 mode, 5 and 6 kinds 2 and 4 without the raw output (residual in, act out: the last block of a level).  Each case
names the kernel the launcher must take (kgb_conv_wg_kernel or kgb_conv_wg_epi_kernel) and the GPU test asserts it, so that a change
to a stage count or a flag list cannot move a case to the other kernel unnoticed.

test_bounds_separate_correct_from_broken (no GPU) rehearses every case of the GPU matrix.  The emulation of the correct kernel
(accumulate() followed by the epilogue in fp32) must stay within a quarter of every bound.  Each emulated mutant must exceed a bound
at least 8x, unless the case cannot show that mutant (named in _exempt).  The mutants are: a dropped split term, a dropped lo half,
an fp32 residual rounded through fp16, the residual read from the neighbouring 32-column slice, the neighbouring image's ncbias, and
an off-board position left unmasked.  Cases of more than 24 images are rehearsed on their first 24.
"""
import numpy as np
import pytest

F16, F32, F64 = np.float16, np.float32, np.float64
C_ACC = 8.0           # accumulation bound, in units of one truncation per accumulator update (see the module docstring)
PROJ_BOUND = 1.0 / 16  # largest coefficient of a split term or of the lo half allowed in the error (see the module docstring)
ACT_LIPSCHITZ = {0: 1.0, 1: 1.0, 2: 1.1, 3: 1.1}   # max |act'|: mish 1.089, SiLU 1.100
Z_ROUND = 2.0 ** -22   # the fma's rounding of z is at most 2^-24 |z|: 4x, so that no check can be exhausted by one exact rounding
REHEARSAL_MAX_N = 24


WG, WG_EPI = "kgb_conv_wg_kernel", "kgb_conv_wg_epi_kernel"


def _case(cid, ky, cin, cout, n, X, Y, kind, fp16, act, boards=None, ncbias=False, bias=1.0, check_images=None, kernel=WG, env=None):
    """kernel: the kernel the launcher must choose (split mode and 1x1 layers always take kgb_conv_wg_kernel); env: variables set
    for the launch."""
    return pytest.param(dict(ky=ky, cin=cin, cout=cout, n=n, X=X, Y=Y, kind=kind, fp16=fp16, act=act, boards=boards, ncbias=ncbias,
                             bias=bias, check_images=check_images, kernel=kernel, env=env or {}), id=cid)


MIXED = ((19, 19), (9, 9), (13, 13), (7, 11))   # repeated over the batch
CASES = [
    # the b18 3x3 192 -> 192 in every epilogue kind, both modes
    _case("3x3-192-k1-split-mish", 3, 192, 192, 6, 19, 19, 1, False, 2, bias=12.0),
    _case("3x3-192-k1-fp16-mish-mixed", 3, 192, 192, 8, 19, 19, 1, True, 2, boards=MIXED, bias=12.0, kernel=WG_EPI),
    _case("3x3-192-k2-split-identity", 3, 192, 192, 6, 19, 19, 2, False, 0),
    _case("3x3-192-k2-fp16-relu-mixed", 3, 192, 192, 8, 19, 19, 2, True, 1, boards=MIXED),
    _case("3x3-192-k3-split-silu", 3, 192, 192, 6, 19, 19, 3, False, 3, bias=12.0),
    _case("3x3-192-k3-fp16-mish-13x7", 3, 192, 192, 10, 19, 19, 3, True, 2, boards=((13, 7),), kernel=WG_EPI),
    _case("3x3-192-k4-split-silu", 3, 192, 192, 6, 19, 19, 4, False, 3, bias=12.0),
    _case("3x3-192-k4-fp16-silu", 3, 192, 192, 6, 19, 19, 4, True, 3, bias=12.0),
    _case("3x3-192-k0-split-mixed", 3, 192, 192, 8, 19, 19, 0, False, 0, boards=MIXED),
    _case("3x3-192-k0-fp16-9x9", 3, 192, 192, 8, 9, 9, 0, True, 0, boards=((7, 5),), kernel=WG_EPI),
    # every tile width: cout 32, 64, 128, 256 and two n-tiles of 160, 224 and 192
    _case("1x1-cout32-k2-split-mish-13x7", 1, 192, 32, 20, 13, 7, 2, False, 2, bias=12.0),
    _case("3x3-cout64-k1-fp16-silu-9x9", 3, 64, 64, 24, 9, 9, 1, True, 3, boards=((9, 9), (5, 7)), bias=12.0),
    _case("1x1-cout128-k4-split-mish-9x9", 1, 128, 128, 24, 9, 9, 4, False, 2, bias=12.0),
    _case("3x3-cout256-k2-split-relu", 3, 256, 256, 3, 19, 19, 2, False, 1),
    _case("3x3-cout256-k4-fp16-mish-9x9", 3, 256, 256, 12, 9, 9, 4, True, 2, bias=12.0),
    _case("1x1-cout320-k4-fp16-relu", 1, 128, 320, 6, 19, 19, 4, True, 1),
    _case("1x1-cout448-k2-split-silu", 1, 128, 448, 6, 19, 19, 2, False, 3, bias=12.0),
    _case("1x1-cout384-k3-split-identity", 1, 192, 384, 6, 19, 19, 3, False, 0),
    # the initial conv: 5x5, 22 input channels, per-image global bias, kind 3, as the evaluator emits it
    _case("5x5-initial-k3-split-mish-mixed", 5, 22, 192, 8, 19, 19, 3, False, 2, boards=MIXED, ncbias=True, bias=12.0),
    _case("5x5-initial-k3-fp16-mish", 5, 22, 192, 8, 19, 19, 3, True, 2, ncbias=True, bias=12.0, kernel=WG_EPI),
    _case("5x5-initial-k3-split-relu-9x9", 5, 22, 96, 16, 9, 9, 3, False, 1, ncbias=True),
    # frames with fewer than 128 rows in all: one partial tile
    _case("2x2-frame-k2-split-mish", 3, 64, 64, 8, 2, 2, 2, False, 2, bias=12.0),
    _case("3x3-frame-k1-fp16-silu-2x3", 3, 64, 64, 6, 3, 3, 1, True, 3, boards=((2, 3), (3, 3)), bias=12.0),
    # many tiles per CTA (rings wrap across tiles) in split mode with full-precision data
    _case("b18-3x3-k4-split-b128", 3, 192, 192, 128, 19, 19, 4, False, 2, bias=12.0),
    _case("exit1x1-k2-split-b256-two-n-tiles", 1, 192, 384, 256, 19, 19, 2, False, 2, bias=12.0),
    _case("n160-five-slices-k2-split", 1, 128, 320, 100, 19, 19, 2, False, 3, bias=12.0),
    _case("n224-seven-slices-k4-split", 1, 128, 448, 100, 19, 19, 4, False, 1),
    # b28c512nbt (trunk 512, mid 256, gpool 64) as the evaluator emits its layers, in both modes (fp16 mode keeps every stream in fp16):
    # the entry 1x1 (8 k-blocks), the mid 3x3, the exit 1x1 and the 3x3 initial conv (two 256-wide n-tiles), and the gpool unit's first
    # conv with its 3x3 256 -> 64 gpool conv packed in as channels 256-319
    _case("b28-entry1x1-512-k3-split-mish", 1, 512, 256, 24, 19, 19, 3, False, 2, bias=12.0),
    _case("b28-entry1x1-512-k3-fp16-mish-mixed", 1, 512, 256, 24, 19, 19, 3, True, 2, boards=MIXED, bias=12.0),
    _case("b28-3x3-256-k1-fp16-mish-b64-mixed", 3, 256, 256, 64, 19, 19, 1, True, 2, boards=MIXED, bias=12.0),
    _case("b28-3x3-256-k2-fp16-mish-b64-mixed", 3, 256, 256, 64, 19, 19, 2, True, 2, boards=MIXED, bias=12.0),
    _case("b28-exit1x1-512-k2-split-mish", 1, 256, 512, 24, 19, 19, 2, False, 2, bias=12.0),
    _case("b28-exit1x1-512-k2-fp16-mish-mixed", 1, 256, 512, 24, 19, 19, 2, True, 2, boards=MIXED, bias=12.0),
    _case("b28-initial3x3-512-k3-split-mish-mixed", 3, 22, 512, 16, 19, 19, 3, False, 2, boards=MIXED, ncbias=True, bias=12.0),
    _case("b28-initial3x3-512-k3-fp16-mish-mixed", 3, 22, 512, 16, 19, 19, 3, True, 2, boards=MIXED, ncbias=True, bias=12.0),
    _case("b28-gpool3x3-256-320-k0-split-mixed", 3, 256, 320, 24, 19, 19, 0, False, 0, boards=MIXED),
    _case("b28-gpool3x3-256-320-k0-fp16-mixed", 3, 256, 320, 24, 19, 19, 0, True, 0, boards=MIXED, kernel=WG_EPI),
    # b28's batch: 1024 images of 400 rows are 3200 whole 128-row tiles, about 24 per CTA; at 1021 image 1020 holds the partial last tile.
    # Checked on the first images, both sides of 511 / 512 and the last ones (the padding rows between images are zero, so they are
    # independent)
    _case("b28-3x3-256-k2-split-mish-b1024", 3, 256, 256, 1024, 19, 19, 2, False, 2, bias=12.0,
          check_images=(0, 1, 510, 511, 512, 513, 1022, 1023)),
    _case("b28-3x3-256-k2-split-silu-b1021", 3, 256, 256, 1021, 19, 19, 2, False, 3, bias=12.0,
          check_images=(0, 1, 510, 511, 512, 513, 1019, 1020)),
    # kgb_conv_wg_epi_kernel (fp16 mode, mish, 3x3 and 5x5 tiles of 128, 160 and 192 columns) where its CTAs take more than one tile:
    # the accumulator tile's t_full / t_empty phases, the one residual slot's reuse and the operand ring carried across tiles.  A
    # 19x19 image is 400 rows, 3.125 tiles; the H100 has 132 SMs.  b18's commonest 3x3 epilogue at 800 tiles, all of them checked,
    # and the same case on kgb_conv_wg_kernel as the float64 anchor of the bit-identity tests between the two
    _case("3x3-192-k2-fp16-mish-b256", 3, 192, 192, 256, 19, 19, 2, True, 2, bias=12.0, kernel=WG_EPI),
    _case("3x3-192-k2-fp16-mish-b256-no-epilogue-wg", 3, 192, 192, 256, 19, 19, 2, True, 2, bias=12.0, env={"KGB_EPILOGUE_WG": "0"}),
    _case("3x3-192-k2-fp16-mish-b1021", 3, 192, 192, 1021, 19, 19, 2, True, 2, bias=12.0, kernel=WG_EPI,
          check_images=(0, 1, 330, 331, 660, 661, 1019, 1020)),
    _case("3x3-192-k2-fp16-mish-b43-mixed", 3, 192, 192, 43, 19, 19, 2, True, 2, boards=MIXED, bias=12.0, kernel=WG_EPI),
    _case("3x3-192-k0-fp16-b43-mixed", 3, 192, 192, 43, 19, 19, 0, True, 0, boards=MIXED, kernel=WG_EPI),
    # cout is padded to 64 channels: 96 runs at 128 columns with 32 padded ones, and 160 columns are two n-tiles of 320
    _case("3x3-96-k2-fp16-mish-b48", 3, 96, 96, 48, 19, 19, 2, True, 2, bias=12.0, kernel=WG_EPI),
    _case("3x3-128-k1-fp16-mish-b48-mixed", 3, 128, 128, 48, 19, 19, 1, True, 2, boards=MIXED, bias=12.0, kernel=WG_EPI),
    _case("3x3-160-320-k3-fp16-mish-b48-mixed", 3, 160, 320, 48, 19, 19, 3, True, 2, boards=MIXED, bias=12.0, kernel=WG_EPI),
    _case("5x5-initial-22-96-k3-fp16-mish-b48-mixed", 5, 22, 96, 48, 19, 19, 3, True, 2, boards=MIXED, ncbias=True, bias=12.0,
          kernel=WG_EPI),
    # kinds 5 and 6: the residual in, no raw output, as the last block of every level runs (b18: the second conv of each nested
    # block's last inner block, and the trunk's last exit 1x1).  fp16 mode on the epilogue-warpgroup kernel; split mode, the fp32
    # stream and the 1x1 on kgb_conv_wg_kernel's EPI_RES | EPI_MISH copies
    _case("3x3-192-k5-fp16-mish-b48-mixed", 3, 192, 192, 48, 19, 19, 5, True, 2, boards=MIXED, bias=12.0, kernel=WG_EPI),
    _case("3x3-192-k5-split-mish", 3, 192, 192, 6, 19, 19, 5, False, 2, bias=12.0),
    _case("3x3-192-k6-fp16-mish-mixed", 3, 192, 192, 8, 19, 19, 6, True, 2, boards=MIXED, bias=12.0),
    _case("exit1x1-192-384-k5-fp16-mish-b24", 1, 192, 384, 24, 19, 19, 5, True, 2, bias=12.0),
]


# ---- data -------------------------------------------------------------------------------------------------------------------------

def select_images(d, idx):
    """The per-image inputs of the images idx (weights and BN are shared by all images)."""
    return {k: v[idx] if k in ("x", "res", "ncb", "board_xy", "mask") and v is not None else v for k, v in d.items()}


def make_data(c, n=None):
    """Seeded inputs of one case; nothing is fp16-exact, and the input is nonzero off the board."""
    n = c["n"] if n is None else n
    seed = [c["ky"], c["cin"], c["cout"], c["X"], c["Y"], c["kind"], int(c["fp16"]), c["act"], int(c["ncbias"])]
    rng = np.random.default_rng(seed)
    ky, cin, cout, X, Y = c["ky"], c["cin"], c["cout"], c["X"], c["Y"]
    d = dict(w=(rng.standard_normal((ky, ky, cin, cout)) / np.sqrt(ky * ky * cin)).astype(F32),
             x=rng.standard_normal((c["n"], Y, X, cin)).astype(F32)[:n])
    d["res"] = (4.0 * rng.standard_normal((c["n"], Y, X, cout))).astype(F32)[:n] if has_residual(c) else None
    d["ncb"] = rng.standard_normal((c["n"], cout)).astype(F32)[:n] if c["ncbias"] else None
    # BN: scales of both signs; biases in three widths so that some channels sit near zero and others deep in the activation's tails
    d["sc"] = (rng.uniform(0.25, 1.5, cout) * rng.choice([-1.0, 1.0], cout, p=[0.25, 0.75])).astype(F32)
    d["bi"] = (rng.uniform(-1.0, 1.0, cout) * rng.choice([0.5, 4.0, c["bias"]], cout)).astype(F32)
    boards = c["boards"] or ((X, Y),)
    d["board_xy"] = np.array([boards[i % len(boards)] for i in range(n)], np.int32)
    mask = np.zeros((n, Y, X), F64)
    for i, (bx, by) in enumerate(d["board_xy"]):
        mask[i, :by, :bx] = 1.0
    d["mask"] = mask
    return d


# ---- float64 reference ------------------------------------------------------------------------------------------------------------

def _h(a):
    return a.astype(F16).astype(F64)


def split_halves(a32):
    hi = _h(a32)
    return hi, _h(a32.astype(F64) - hi)


def conv64(x, w):
    """'same' zero-padded cross-correlation, NHWC, accumulated tap by tap in the dtype of x and w."""
    n, Y, X, cin = x.shape
    ky, kx, _, cout = w.shape
    py, px = ky // 2, kx // 2
    xp = np.zeros((n, Y + 2 * py, X + 2 * px, cin), x.dtype)
    xp[:, py:py + Y, px:px + X] = x
    out = np.zeros((n * Y * X, cout), x.dtype)
    for dy in range(ky):
        for dx in range(kx):
            out += xp[:, dy:dy + Y, dx:dx + X].reshape(-1, cin) @ w[dy, dx]
    return out.reshape(n, Y, X, cout)


def act64(z, act):
    if act == 0:
        return z
    if act == 1:
        return np.maximum(z, 0.0)
    if act == 2:
        return z * np.tanh(np.logaddexp(0.0, z))
    if act == 3:
        return z * 0.5 * (1.0 + np.tanh(0.5 * z))   # z * sigmoid(z), without overflow
    raise ValueError(act)


def operands(c, d):
    """(ah, al, wh, wl) as the kernel receives them; al, wl None in fp16 mode."""
    if c["fp16"]:
        return _h(d["x"]), None, _h(d["w"]), None
    return split_halves(d["x"]) + split_halves(d["w"])


def has_residual(c):
    return c["kind"] in (2, 4, 5, 6)


def has_raw(c):
    """Kinds 5 and 6 read the residual and write no raw output (kinds 2 and 4 without it)."""
    return c["kind"] in (0, 2, 3, 4)


def stream_residual(c, d):
    """The residual as the stream holds it: fp32 for kinds 4 and 6 and in split mode, fp16 otherwise."""
    if d["res"] is None:
        return 0.0
    return d["res"].astype(F64) if stream_fp32(c) else _h(d["res"])


def reference(c, d):
    ah, al, wh, wl = operands(c, d)
    ideal = conv64(ah, wh)
    terms = {}
    if al is not None:   # the split's two cross terms, kept apart for the projection checks
        terms = {"al*wh": conv64(al, wh), "ah*wl": conv64(ah, wl)}
        ideal = ideal + terms["al*wh"] + terms["ah*wl"]
    x64, w64 = d["x"].astype(F64), d["w"].astype(F64)
    sigma = np.sqrt(conv64(x64 * x64, w64 * w64))
    nb = d["ncb"].astype(F64)[:, None, None, :] if d["ncb"] is not None else 0.0
    R = stream_residual(c, d)
    V = ideal + nb + R
    m = d["mask"][..., None]
    z = V * d["sc"].astype(F64) + d["bi"].astype(F64)
    act = m * act64(z, c["act"])
    return dict(ideal=ideal, terms=terms, sigma=sigma, sum_abs=np.abs(ideal) + np.abs(nb) + np.abs(R), V=V, raw=m * V, z=z, act=act,
                lo=_h(act - _h(act)), mask=m)


# ---- bounds -----------------------------------------------------------------------------------------------------------------------

def ulp16(a):
    """fp16 spacing at |a|, the subnormal spacing 2^-24 below 2^-14."""
    a = np.abs(a)
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return np.exp2(e - 10.0)


def ulp32(a):
    a = np.abs(a)
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -126)))
    return np.exp2(e - 23.0)


def accumulator_updates(c):
    """Accumulator updates one output receives: one per 16 input channels, tap and split part (padding channels add exact zeros)."""
    return -(-c["cin"] // 16) * c["ky"] * c["ky"] * (1 if c["fp16"] else 3)


def stream_fp32(c):
    """Whether the raw output or the stream is fp32: kind 0's raw output, the fp32 stream of kinds 4 and 6, split mode; a case's "raw32"
    overrides it (an fp32 stream in fp16 mode, as KGB_STREAM_FP32=all runs the inner streams)."""
    return c.get("raw32", c["kind"] in (0, 4, 6) or not c["fp16"])


def raw_fp32(c):
    return has_raw(c) and stream_fp32(c)


def formula_error(z, act):
    if act in (0, 1):
        return np.zeros_like(z)
    az = np.abs(z)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(az > 0, act64(z, act) / np.where(az > 0, z, 1.0), 0.0)
    r = np.clip(r, 0.0, 1.0)
    return 2.0 ** -20 * az * (1.0 + (az + 8.0) * r * (1.0 - r))


def store_error(a, fp16):
    return 0.5 * ulp16(a) if fp16 else 2.0 ** -22 * np.abs(a) + 2.0 ** -25


def bounds(c, d, ref):
    """(raw bound or None, act bound or None), each a pair (computation, storage): the first bounds the error of the value the
    kernel computes, the second the rounding to the stored dtype.  Both are zero where the mask is zero."""
    m = ref["mask"]
    # An operand computed by an earlier layer inside the same kernel (the fused boundary's entry) brings that layer's error in, carried
    # through the weights: e_operand from its computation bound, joining this layer's computation term, and s_operand from its
    # storage rounding, which has no margin to give and joins the storage term in full.  Both are zero for an operand given exactly.
    s_op = ref.get("s_operand", 0.0)
    e_v = C_ACC * accumulator_updates(c) * 2.0 ** -23 * ref["sigma"] + 2.0 ** -22 * ref["sum_abs"] + ref.get("e_operand", 0.0)
    V = np.abs(ref["V"])
    store = s_op + 0.5 * (ulp32(V * (1 + 2.0 ** -20) + e_v + s_op) if raw_fp32(c) else ulp16(V * (1 + 2.0 ** -9) + e_v + s_op))
    raw_b = (m * e_v, m * store) if has_raw(c) else None
    act_b = None
    if c["kind"] != 0:
        z, a = ref["z"], np.abs(act64(ref["z"], c["act"]))
        e_a = ACT_LIPSCHITZ[c["act"]] * (np.abs(d["sc"]).astype(F64) * e_v + Z_ROUND * np.abs(z)) + formula_error(z, c["act"])
        s_a = ACT_LIPSCHITZ[c["act"]] * np.abs(d["sc"]).astype(F64) * s_op
        act_b = (m * e_a, m * (s_a + store_error((a + e_a + s_a) * (1 + 2.0 ** -9), c["fp16"])))
    return raw_b, act_b


def _ratio(err, bound):
    """Worst (|err| - storage rounding) / computation bound: a value <= 1 passes.  Where both bounds are zero, only an exact zero
    passes."""
    pre, store = bound
    excess = np.maximum(np.abs(err) - store, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(pre > 0, excess / np.where(pre > 0, pre, 1.0), np.where(excess > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def _projection(err, direction, weight, mask):
    """Least-squares coefficient of `direction` in `err` (weighted, over the rows the mask keeps), over PROJ_BOUND."""
    e, g = (err * weight)[mask], (direction * weight)[mask]
    den = float(np.sum(g * g))
    return abs(float(np.sum(e * g)) / den) / PROJ_BOUND if den > 0 else 0.0


def check(c, d, ref, raw, hi, lo):
    """Worst ratio of each check (> 1 is a failure; the split structure is 0 or inf)."""
    raw_b, act_b = bounds(c, d, ref)
    out = {}
    on = np.broadcast_to(ref["mask"] > 0, ref["V"].shape)
    w = 1.0 / np.maximum(ref["sigma"], 1e-30)
    if raw_b is not None:
        out["raw"] = _ratio(raw.astype(F64) - ref["raw"], raw_b)
    for name, t in ref["terms"].items():
        if raw is not None:   # split mode: raw is fp32
            out[name] = _projection(raw.astype(F64) - ref["raw"], t, w, on)
        else:                 # kind 1: the term as it reaches the activation
            zh = 2.0 ** -20 * np.maximum(np.abs(ref["z"]), 1.0)
            slope = (act64(ref["z"] + zh, c["act"]) - act64(ref["z"] - zh, c["act"])) / (2 * zh) * d["sc"].astype(F64)
            out[name] = _projection(hi.astype(F64) + lo.astype(F64) - ref["act"], slope * t, w, on)
    if act_b is not None:
        a = hi.astype(F64) + (lo.astype(F64) if lo is not None else 0.0)
        out["act"] = _ratio(a - ref["act"], act_b)
        if raw is not None and raw_fp32(c):
            # the activation of the kernel's own fp32 raw: no accumulation term
            z = raw.astype(F64) * d["sc"].astype(F64) + d["bi"].astype(F64)
            own = ref["mask"] * act64(z, c["act"])
            e_a = ACT_LIPSCHITZ[c["act"]] * Z_ROUND * np.abs(z) + formula_error(z, c["act"])
            out["own"] = _ratio(a - own, (ref["mask"] * e_a, ref["mask"] * store_error((np.abs(own) + e_a) * (1 + 2.0 ** -9), c["fp16"])))
        if lo is not None:
            out["lo"] = _projection(a - ref["act"], ref["lo"], 1.0, on)
            h64, l64 = hi.astype(F64), lo.astype(F64)
            half = 0.5 * ulp16(h64)
            ok = ((_h(h64 + l64) == h64) | (np.abs(l64) == half)) & (np.abs(l64) <= half)
            out["split"] = 0.0 if ok.all() else np.inf
    return out


# ---- emulation of the kernel (no GPU), and its mutants ------------------------------------------------------------------------------

def accumulate(c, d):
    """The kernel's accumulation as the H100 performs it, in the kernel's order (k-block of 64 channels, split part, tap, 16
    channels): each step adds the exact sum of 16 products to the fp32 accumulator and truncates the result toward zero."""
    ah, al, wh, wl = operands(c, d)
    n, Y, X, cin = ah.shape
    k, cout = c["ky"], c["cout"]
    p = k // 2

    def taps(a):
        ap = np.zeros((n, Y + 2 * p, X + 2 * p, cin), F64)
        ap[:, p:p + Y, p:p + X] = a
        return [ap[:, dy:dy + Y, dx:dx + X].reshape(-1, cin) for dy in range(k) for dx in range(k)]

    A = taps(ah)
    parts = [(A, wh.reshape(k * k, cin, cout))]
    if al is not None:
        parts += [(taps(al), wh.reshape(k * k, cin, cout)), (A, wl.reshape(k * k, cin, cout))]
    acc = np.zeros((n * Y * X, cout), F64)
    for k0 in range(0, cin, 64):
        for xs, ws in parts:
            for t in range(k * k):
                for j in range(k0, min(k0 + 64, cin), 16):
                    s = acc + xs[t][:, j:j + 16] @ ws[t, j:j + 16]
                    r = s.astype(F32)
                    acc = np.where(np.abs(r) > np.abs(s), np.nextafter(r, F32(0)), r).astype(F64)
    return acc.reshape(n, Y, X, cout)


def emulate(c, d, ref, acc, drop=None):
    """The kernel from its accumulator on: the epilogue in fp32 (z by a single rounding, as the fma does; an accurate activation),
    hi = fp16(a), lo = fp16(a - hi).  `drop` names a mutant, applied to the correct kernel's accumulator or epilogue."""
    if drop in ("al*wh", "ah*wl"):
        acc = acc - ref["terms"][drop]
    v = acc.astype(F32)
    if d["ncb"] is not None:
        ncb = np.roll(d["ncb"], 1, axis=0) if drop == "ncbias-neighbour" else d["ncb"]
        v = (v + ncb[:, None, None, :]).astype(F32)
    if d["res"] is not None:
        R = stream_residual(c, d)
        if drop == "residual-via-fp16":
            R = _h(d["res"])
        if drop == "residual-neighbour-slice":
            R = neighbour_slice(R)
        v = (v + R.astype(F32)).astype(F32)
    m = d["mask"][..., None].copy()
    if drop == "unmasked":
        i, (bx, by) = next((i, b) for i, b in enumerate(d["board_xy"]) if b[0] < c["X"] or b[1] < c["Y"])
        if bx < c["X"]:
            m[i, 0, bx] = 1.0
        else:
            m[i, by, 0] = 1.0
    raw = None
    if has_raw(c):
        raw = (v * m.astype(F32)).astype(F32)
        if not raw_fp32(c):
            raw = raw.astype(F16).astype(F32)
    hi = lo = None
    if c["kind"] != 0:
        z = (v.astype(F64) * d["sc"].astype(F64) + d["bi"].astype(F64)).astype(F32)
        a = np.where(m > 0, act64(z.astype(F64), c["act"]), 0.0).astype(F32)
        hi = a.astype(F16).astype(F32)
        if not c["fp16"]:
            lo = (a.astype(F64) - hi.astype(F64)).astype(F16).astype(F32)
            if drop == "act-lo":
                lo = np.zeros_like(lo)
    return raw, hi, lo


def neighbour_slice(a):
    """a's channels each read from the neighbouring 32-column slice (slices 2k and 2k + 1 swapped; the padded channels up to the next
    64 are zero)."""
    c = a.shape[-1]
    pad = np.zeros(a.shape[:-1] + (-(-c // 64) * 64,), a.dtype)
    pad[..., :c] = a
    return pad[..., np.arange(c) ^ 32]


MUTANTS = ("al*wh", "ah*wl", "act-lo", "residual-via-fp16", "residual-neighbour-slice", "ncbias-neighbour", "unmasked")


def _exempt(c, mutant):
    """Why this case cannot show `mutant`, or None."""
    split = not c["fp16"]
    if mutant in ("al*wh", "ah*wl") and not split:
        return "fp16 mode has no lo operands"
    if mutant == "act-lo" and (not split or c["kind"] == 0):
        return "no activated operand in split mode"
    if mutant == "residual-via-fp16" and not (has_residual(c) and stream_fp32(c)):
        return "no fp32 residual stream"
    if mutant == "residual-neighbour-slice" and not has_residual(c):
        return "no residual"
    if mutant == "ncbias-neighbour" and not c["ncbias"]:
        return "no ncbias"
    if mutant == "unmasked" and not any(b[0] < c["X"] or b[1] < c["Y"] for b in (c["boards"] or ())):
        return "every image covers the whole frame"
    return None


@pytest.mark.parametrize("c", CASES)
def test_bounds_separate_correct_from_broken(c):
    n = min(c["n"], REHEARSAL_MAX_N)
    d = make_data(c, n)
    ref = reference(c, d)
    acc = accumulate(c, d)
    r = check(c, d, ref, *emulate(c, d, ref, acc))
    print("correct emulation, worst error / bound:", {k: f"{v:.3g}" for k, v in r.items()})
    assert r and max(r.values()) <= 0.25, f"the emulated correct kernel uses more than a quarter of a bound: {r}"
    tried = 0
    for mutant in MUTANTS:
        if _exempt(c, mutant):
            continue
        tried += 1
        rm = check(c, d, ref, *emulate(c, d, ref, acc, drop=mutant))
        print(f"mutant {mutant}: worst {max(rm.values()):.3g}x")
        assert max(rm.values()) >= 8.0, f"mutant {mutant} stays within 8x of the bounds: {rm}"
    assert tried > 0, "no mutant can be told apart on this case"


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES)
def test_conv_against_fp64(c, monkeypatch):
    from katago_b200 import nn_backend
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    d = make_data(c)
    raw, hi, lo = nn_backend.test_conv_ex(c["ky"], c["ky"], c["cin"], c["cout"], d["w"], c["n"], c["X"], c["Y"], c["fp16"], c["kind"],
                                          d["x"], board_xy=d["board_xy"], ncbias=d["ncb"], residual=d["res"], bn_scale=d["sc"],
                                          bn_bias=d["bi"], activation=c["act"])
    assert nn_backend.test_last_conv_kernel() == c["kernel"]
    assert (hi is None) == (c["kind"] == 0) and (lo is None) == (c["fp16"] or c["kind"] == 0) and (raw is None) == (not has_raw(c))
    if c["check_images"] is not None:
        idx = np.array(c["check_images"])
        d = select_images(d, idx)
        raw, hi, lo = (a[idx] if a is not None else None for a in (raw, hi, lo))
    r = check(c, d, reference(c, d), raw, hi, lo)
    print("worst error / bound:", {k: f"{v:.3g}" for k, v in r.items()})
    assert max(r.values()) <= 1.0, r
