"""The wgmma GEMM of csrc/gemm.cu (``cb_gemm_f16_ex``): its dispatch restated as plain functions, a sweep of shapes built from the
boundaries of that dispatch, inputs whose product the fp32 accumulator holds exactly, a bit-exact model of the epilogues given that
exact product, and the error bound of the three activations.

``C[M][N] = epilogue(A[M][K] . W[N][K]^T + bias)``.  A launch is one instantiation ``gemm_wgmma_kernel<BN, ACT, OUT_F32, SCALE>``
over a persistent grid of ``min(tiles, sm_count)`` CTAs; CTA b runs tiles b, b + grid, ... (n fastest).  Each of its two consumer
warpgroups owns 64 rows of a 128 x BN tile and writes them in slices of 128 bytes (64 fp16 or 32 fp32 columns) through two
shared-memory buffers; the buffer index and the residual barriers' parities carry from one tile to the next.

Exactness: with fp16 operands that are small integers, every product and every partial sum is an integer below 2^24, so the fp32
accumulator holds ``z = A . W^T`` exactly whatever order the tensor cores add in.  What the epilogue then does to z is a short chain
of IEEE float32 operations, which ``emulate`` reproduces bit for bit.  The activations use approximate intrinsics; ``act_bound``
bounds their error.  The functions take torch tensors on any device.
"""

from __future__ import annotations

import math
from dataclasses import dataclass

import torch

BM, BK = 128, 64
EPI_NONE, EPI_QUICK_GELU, EPI_GELU_TANH, EPI_GELU_ERF = 0, 1, 2, 3
ACTIVATIONS = (EPI_QUICK_GELU, EPI_GELU_TANH, EPI_GELU_ERF)
EPI_NAME = {EPI_NONE: "NONE", EPI_QUICK_GELU: "QUICK_GELU", EPI_GELU_TANH: "GELU_TANH", EPI_GELU_ERF: "GELU_ERF"}
SM_COUNTS = (132, 114)  # H100 SXM, H100 PCIe


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


# --------------------------------------------------------------------------------------------------------------------- dispatch
def tile_width(m: int, n: int, k: int, gamma: bool, out_f32: bool, epilogue: int, sm_count: int) -> int:
    """BN: 128 x 256 tiles when that still gives every SM a tile and N splits into them evenly or is wide; never with gamma."""
    tiles256 = cdiv(m, BM) * cdiv(n, 256)
    return 256 if not gamma and (n % 256 == 0 or n > 1024) and tiles256 >= sm_count else 128


def stages(bn: int) -> int:
    """Depth of the TMA -> wgmma mbarrier ring."""
    return 4 if bn == 256 else 6


def slice_cols(out_f32: bool) -> int:
    """Columns of one 128-byte epilogue slice."""
    return 32 if out_f32 else 64


def instantiation(bn: int, epilogue: int, out_f32: bool, gamma: bool) -> str:
    out = "f32" if out_f32 else "f16"
    return f"<{bn},{EPI_NAME[epilogue]},{out}{',SCALE' if gamma else ''}>"


# the 11 kernels the library holds: BN x {fp16 out x 4 epilogues, fp32 out}, and the LayerScale kernel at BN = 128;
# name -> (BN, epilogue, out_f32, gamma)
INSTANTIATION_ARGS = {instantiation(*a): a for a in
                      [(bn, e, False, False) for bn in (128, 256) for e in (EPI_NONE, *ACTIVATIONS)]
                      + [(bn, EPI_NONE, True, False) for bn in (128, 256)] + [(128, EPI_NONE, True, True)]}  # fmt: skip
INSTANTIATIONS = tuple(INSTANTIATION_ARGS)


@dataclass(frozen=True)
class Plan:
    """What cb_gemm_f16_ex launches for one call."""

    inst: str
    bn: int
    stages: int
    m_tiles: int
    n_tiles: int
    grid: int
    num_kb: int
    slice_cols: int

    @property
    def tiles(self) -> int:
        return self.m_tiles * self.n_tiles

    def tiles_of_cta(self, b: int) -> range:
        return range(b, self.tiles, self.grid)

    @property
    def max_tiles_per_cta(self) -> int:
        return len(self.tiles_of_cta(0))


def plan(m: int, n: int, k: int, gamma: bool, out_f32: bool, epilogue: int, sm_count: int) -> Plan:
    bn = tile_width(m, n, k, gamma, out_f32, epilogue, sm_count)
    m_tiles, n_tiles = cdiv(m, BM), cdiv(n, bn)
    return Plan(instantiation(bn, EPI_NONE if out_f32 else epilogue, out_f32, gamma), bn, stages(bn), m_tiles, n_tiles,
                min(m_tiles * n_tiles, sm_count), cdiv(k, BK), slice_cols(out_f32))  # fmt: skip


def nslices(p: Plan, m: int, n: int, tile: int, c: int) -> int:
    """Slices consumer warpgroup c stores of this tile: none when its 64 rows are all past M, else the ones with columns < N."""
    m_blk, n_blk = divmod(tile, p.n_tiles)
    row0, col0 = m_blk * BM + 64 * c, n_blk * p.bn
    return 0 if row0 >= m else min(p.bn // p.slice_cols, cdiv(n - col0, p.slice_cols))


def epilogue_states(p: Plan, m: int, n: int) -> set[tuple[int, int]]:
    """(eb, rphase) at the start of every tile a consumer warpgroup stores slices of: eb is the buffer of its next slice, rphase
    the parity bits of the two residual barriers; both move by one per slice and carry across the CTA's tiles."""
    seen = set()
    for b in range(p.grid):
        for c in (0, 1):
            eb, rphase = 0, 0
            for t in p.tiles_of_cta(b):
                ns = nslices(p, m, n, t, c)
                if ns:
                    seen.add((eb, rphase))
                for _ in range(ns):
                    rphase ^= 1 << eb
                    eb ^= 1
    return seen


def starts_with_both_parities(p: Plan, m: int, n: int) -> bool:
    """Some tile starts on each buffer, and the residual barrier of its first slice waits for each parity."""
    states = epilogue_states(p, m, n)
    return {eb for eb, _ in states} == {0, 1} and {rphase >> eb & 1 for eb, rphase in states} == {0, 1}


# ------------------------------------------------------------------------------------------------------------------ the sweep
@dataclass(frozen=True)
class Point:
    name: str
    m: int
    n: int
    k: int


# every Linear of the four towers (N, K) and the patch embeddings, at a modest M
TOWERS = [
    ("clip_qkv", 257, 3072, 1024), ("clip_out", 257, 1024, 1024), ("clip_fc1", 257, 4096, 1024), ("clip_fc2", 257, 1024, 4096),
    ("siglip_fc1", 729, 4304, 1152), ("siglip_fc2", 729, 1152, 4304),
    ("iv2_qkv", 1025, 4224, 1408), ("iv2_fc1", 513, 6144, 1408), ("iv2_fc2", 513, 1408, 6144), ("iv2_proj", 1025, 1408, 1408),
    ("bert_qkv", 77, 3072, 1024), ("bert_out", 77, 1024, 1024), ("bert_fc1", 77, 4096, 1024), ("bert_fc2", 77, 1024, 4096),
    ("patch_clip", 256, 1024, 640), ("patch_siglip", 729, 1152, 640), ("patch_iv2", 2048, 1408, 640), ("patch_b16", 196, 768, 768),
]  # fmt: skip
N_TAILS = (8, 32, 40, 64, 72)  # and BN - 8: N mod BN
M_TAILS = (0, 1, 63, 64, 65, 127)  # M mod 128


def m_with(m_tiles: int, tail: int) -> int:
    """M with this many 128-row tiles and M mod 128 = tail."""
    return 128 * m_tiles if tail == 0 else 128 * (m_tiles - 1) + tail


def _odd_tail_rows(n: int, bn: int, sm: int) -> int:
    """M tiles for an N tail: the fewest, from those giving a CTA >= 3 tiles, with which every output type whose tail slice count is
    odd starts tiles on both buffers and both residual parities (tiles are walked n-fastest with a step of the SM count, so which
    CTAs meet the tail column twice depends on both)."""
    nt = cdiv(n, bn)
    mt = cdiv(2 * sm + 1, nt)
    while True:
        ps = [plan(m_with(mt, 1), n, 64, False, f32, EPI_NONE, sm) for f32 in (False, True)]
        assert all(p.bn == bn for p in ps), (n, bn, sm)
        if all(starts_with_both_parities(p, m_with(mt, 1), n) for p in ps if cdiv(n % bn, p.slice_cols) % 2):
            return mt
        mt += 1


def sweep(sm: int) -> list[Point]:
    """Shapes at the boundaries of every dispatch decision for a device of `sm` SMs; each runs every instantiation it reaches."""
    pts: list[Point] = []
    # 128-wide tiles (N <= 1024, not a multiple of 256): every N tail, each with >= 3 tiles on some CTA so that eb and rphase start
    # tiles with both parities; K over the 6-stage ring's boundaries, with and without a K tail
    narrow_k = (8, 320, 384, 448, 832, 312, 440, 776)
    for i, r in enumerate((*N_TAILS, 120)):
        n = 128 * (i % 3) + r
        pts.append(Point(f"narrow_n%128={r}", m_with(_odd_tail_rows(n, 128, sm), M_TAILS[i]), n, narrow_k[i]))
    # tile counts just under, at and over one and two waves: 1, 2 and 3 tiles per CTA
    waves = {"sm-1": sm - 1, "sm": sm, "sm+1": sm + 1, "2sm+1": 2 * sm + 1}
    for (label, t), tail, k in zip(waves.items(), (63, 64, 1, 127), (narrow_k[6], narrow_k[7], 64, 200)):
        pts.append(Point(f"narrow_tiles={label}", m_with(t, tail), 128, k))
    # 256-wide tiles: N > 1024 with every N tail (6 column tiles), K over the 4-stage ring's boundaries
    wide_k = (8, 192, 256, 320, 576, 184, 248)
    for i, r in enumerate((*N_TAILS, 248)):
        n = 1280 + r
        pts.append(Point(f"wide_n%256={r}", m_with(_odd_tail_rows(n, 256, sm), M_TAILS[(i + 3) % 6]), n, wide_k[i]))
    for label, tail, k in (("sm", 0, wide_k[6]), ("sm+1", 65, 568), ("2sm+1", 1, 136)):
        pts.append(Point(f"wide_tiles={label}", m_with(waves[label], tail), 256, k))
    # both sides of the wide predicate: tiles256 the largest reachable value below the SM count and the smallest at or above it
    for n, k in ((512, 136), (1024, 64), (1032, 72), (1408, 120)):
        nt = cdiv(n, 256)
        below, at = (sm - 1) // nt, cdiv(sm, nt)
        pts.append(Point(f"predicate_n={n}_below", m_with(below, 65), n, k))
        pts.append(Point(f"predicate_n={n}_at", m_with(at, 127), n, k))
    pts.append(Point("predicate_n=1016", m_with(cdiv(2 * sm, 4), 64), 1016, 96))  # never wide, however many tiles
    pts += [Point(name, m, n, k) for name, m, n, k in TOWERS]
    return pts


def boundary_classes(p: Plan, m: int, n: int, k: int, sm: int) -> set[str]:
    """The boundaries of the launch that this call sits on."""
    cls = set()
    for name, t in (("sm-1", sm - 1), ("sm", sm), ("sm+1", sm + 1), ("2sm+1", 2 * sm + 1)):
        if p.tiles == t:
            cls.add(f"tiles={name}")
    if p.max_tiles_per_cta <= 3:
        cls.add(f"tiles/cta={p.max_tiles_per_cta}")
    s = p.stages
    for name, kb in (("1", 1), ("S-1", s - 1), ("S", s), ("S+1", s + 1), ("2S+1", 2 * s + 1)):
        if p.num_kb == kb:
            cls.add(f"num_kb={name}")
    if k % BK:
        cls.add("k_tail")
        if k % BK > BK - 16:
            cls.add("k_tail_in_last_k16")  # a K tail that reaches the last k16 step of its k-block
    if m % BM in M_TAILS:
        cls.add(f"m%128={m % BM}")
    r = n % p.bn
    if r in N_TAILS or r == p.bn - 8:
        cls.add(f"n%BN={'BN-8' if r == p.bn - 8 else r}")
    if starts_with_both_parities(p, m, n):
        cls.add("eb_both_parities")
    return cls


def required_classes(bn: int) -> set[str]:
    """Every boundary class an instantiation of this tile width can sit on (a 256-wide launch always has >= sm tiles)."""
    cls = {"tiles=sm", "tiles=sm+1", "tiles=2sm+1", "tiles/cta=1", "tiles/cta=2", "tiles/cta=3", "k_tail", "k_tail_in_last_k16",
           "eb_both_parities"}  # fmt: skip
    cls |= {f"num_kb={x}" for x in ("1", "S-1", "S", "S+1", "2S+1")} | {f"m%128={r}" for r in M_TAILS}
    cls |= {f"n%BN={r}" for r in N_TAILS} | {"n%BN=BN-8"}
    return cls | ({"tiles=sm-1"} if bn == 128 else set())


def launches(pt: Point, sm: int) -> list[tuple[Plan, int, bool, bool]]:
    """(plan, epilogue, out_f32, gamma) of every instantiation a sweep point runs."""
    out = [(plan(pt.m, pt.n, pt.k, False, False, e, sm), e, False, False) for e in (EPI_NONE, *ACTIVATIONS)]
    out.append((plan(pt.m, pt.n, pt.k, False, True, EPI_NONE, sm), EPI_NONE, True, False))
    out.append((plan(pt.m, pt.n, pt.k, True, True, EPI_NONE, sm), EPI_NONE, True, True))
    return out


def coverage(sm: int) -> dict[str, set[str]]:
    """instantiation -> the boundary classes the sweep runs it at."""
    cov: dict[str, set[str]] = {name: set() for name in INSTANTIATIONS}
    for pt in sweep(sm):
        for p, _, _, _ in launches(pt, sm):
            cov[p.inst] |= boundary_classes(p, pt.m, pt.n, pt.k, sm)
    return cov


# ----------------------------------------------------------------------------------------------------------- exact inputs
def _gen(seed: int, device) -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed)


def int_operands(m: int, n: int, k: int, seed: int, device="cpu"):
    """A, W with integer entries in [-8, 8] (fp16): |z| <= 64 K < 2^24 for K <= 2^18, every partial sum too."""
    g = _gen(seed, device)
    a = torch.randint(-8, 9, (m, k), generator=g, device=device).half()
    w = torch.randint(-8, 9, (n, k), generator=g, device=device).half()
    return a, w


def sparse_operands(m: int, n: int, k: int, seed: int, device="cpu"):
    """A, W in {-1, 0, 1} with density min(1, 3 / sqrt(K)): z is an integer of standard deviation about 3 whatever K is, so z + bias
    falls where the activations curve, and every k position still reaches some outputs."""
    g = _gen(seed, device)
    p = min(1.0, 3.0 / math.sqrt(k))

    def one(rows):
        sign = torch.randint(0, 2, (rows, k), generator=g, device=device) * 2 - 1
        return (sign * (torch.rand(rows, k, generator=g, device=device) < p)).half()

    return one(m), one(n)


def position_operands(m: int, n: int, k: int, out_f32: bool, device="cpu"):
    """A, W with three nonzero k positions (0, K / 2 and the last) whose product codes the output's place.  fp32: z = 4096 (m mod
    2048) + (n mod 4096); fp16, where only integers of magnitude <= 2048 are exact: z = 32 (m mod 128) + (n mod 32) - 2048, the
    row within its tile and the column within half a slice."""
    assert k >= 8
    ka, kb, kc = k - 1, 0, k // 2
    rows, cols = torch.arange(m, device=device), torch.arange(n, device=device)
    a = torch.zeros(m, k, device=device)
    w = torch.zeros(n, k, device=device)
    if out_f32:
        a[:, ka], w[:, ka] = rows % 2048, 4096.0
        a[:, kb], w[:, kb] = 64.0, (cols % 4096) // 64
        a[:, kc], w[:, kc] = 1.0, cols % 64
    else:
        a[:, ka], w[:, ka] = rows % 128, 32.0
        a[:, kb], w[:, kb] = 1.0, cols % 32
        a[:, kc], w[:, kc] = -1.0, 2048.0
    return a.half(), w.half()


def decode_position(value: float, out_f32: bool) -> str:
    """Where a position-coded output (no bias) came from."""
    v = int(value)
    if out_f32:
        return f"row = {v // 4096} (mod 2048), column = {v % 4096} (mod 4096)"
    v += 2048
    return f"row = {v // 32} (mod 128), column = {v % 32} (mod 32)"


def grid_bias(n: int, seed: int, device="cpu") -> torch.Tensor:
    """fp32 bias of multiples of 2^-6 in [-1, 1]: with an integer z, z + bias is exact in fp32 (|z| < 2^17) and lands on a fine grid."""
    return torch.randint(-64, 65, (n,), generator=_gen(seed, device), device=device).float() / 64


def exact_product(a: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """z = A W^T in float64: exact for the generators' integer operands (every partial sum < 2^24 < 2^53)."""
    return a.double() @ w.double().t()


# -------------------------------------------------------------------------------------------------------------- the epilogue
def emulate(z: torch.Tensor, bias, gamma, residual, out_f32: bool) -> torch.Tensor:
    """What the kernel stores for an exactly known fp32 accumulator z (float64 [M][N]) with the NONE epilogue:
    fp16 out: f16(f32(z + b));  fp32 out: f32(f32(z + b) + r);  SCALE: f32(f32(f32(z + b) * g) + r).
    z + b is formed in float64 (exact for integer z < 2^24 and fp32 b; otherwise a double rounding that is innocuous, 53 >= 2 * 24 + 2)
    and rounded once; the rest are float32 operations, one rounding each.  A missing bias adds +0; a missing residual adds nothing."""
    v = z + (bias.double() if bias is not None else 0.0)
    v = v.float()
    if not out_f32:
        return v.half()
    if gamma is not None:
        v = v * gamma.float()
    if residual is not None:
        v = v + residual.float()
    return v


# ------------------------------------------------------------------------------------------------------------ the activations
def act64(v: torch.Tensor, epilogue: int) -> torch.Tensor:
    """The activation in float64 (the function the kernel approximates, with the kernel's constants)."""
    v = v.double()
    if epilogue == EPI_QUICK_GELU:
        return v * torch.sigmoid(1.702 * v)
    if epilogue == EPI_GELU_TANH:
        return 0.5 * v * (1 + torch.tanh(0.7978845608028654 * (v + 0.044715 * v**3)))
    if epilogue == EPI_GELU_ERF:
        return 0.5 * v * (1 + torch.erf(v * 0.7071067811865476))
    assert epilogue == EPI_NONE, epilogue
    return v


def ulp16(y: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 numbers in the binade of |y|; 2^-24 (the subnormal spacing) below 2^-14."""
    e = torch.floor(torch.log2(y.double().abs().clamp_min(2.0**-14)))
    return torch.exp2(e - 10)


def act_bound(v: torch.Tensor, epilogue: int) -> torch.Tensor:
    """|kernel - act64(v)| allowed for the fp16 output of an activation of v = f32(z + b), known exactly:
    ulp16(act64(v)) + E(v).

    The fp16 rounding of the kernel's float32 y' costs <= ulp16(y) / 2 + |y' - y| (where y' crosses up into the next binade, the
    result is that binade's first fp16 number, within |y' - y| of y).  So ulp16(y) covers the rounding plus any error of y' that is
    relative and <= 2^-12, and E(v) is what is left:

    * QUICK_GELU, __fdividef(x, 1 + exp2f(-1.702 log2(e) x)): the rounded argument (2^-24 relative, times |1.702 x| ln 2 <= 2^-19.5
      for |x| <= 10), exp2f (2 ulp), the add (2^-24) and rcp.approx inside __fdividef (1 ulp) give y' within about 2^-20 of y,
      relatively, for any x where y is not negligible: E = 0.
    * GELU_TANH, 0.5 x (1 + (1 - __fdividef(2, e + 1))), e = exp2f(2 log2(e) u): 1 + t = 2 - 2 / (e + 1) loses all relative precision
      where e is small (x below about -2.5), so the error is absolute; 1 - q and 1 + t are exact there (Sterbenz).  The rounding of
      e + 1 (2^-24, so 2^-23 in q = 2 / (e + 1)) and __fdividef (div.approx: 2 ulp of q, 2^-22) move 1 + t by <= 3 2^-23 wherever x
      is; exp2f (2 ulp of e) and the rounded argument (u and its scaling by 2 log2(e): about 6 roundings, 2^-21.4 relative, times
      |2u| ln 2 relative in e) move t by (1 - t^2) / 2 times e's relative error: (1 - t^2) (2^-23 + |u| 2^-21.4).  E is |x| / 2 times
      3 2^-23 + (1 - t^2) (2^-23 + |u| 2^-21), about |v| 2^-22.4 in the tail.
    * GELU_ERF, 0.5 x (1 + erff(x / sqrt(2))): erff is within 2 ulp (2^-23 absolute near -1), and the rounded argument moves erf by
      <= 2 / sqrt(pi) a e^{-a^2} 2^-23 < 2^-23.5; 1 + erf is exact (Sterbenz) where erf <= -1/2, else a relative rounding.  So
      |y' - y| <= |x| / 2 (2^-23 + 2^-23.5) + relative terms < |x| 2^-23.2: E = |v| 2^-22 (twice that).
    """
    y = act64(v, epilogue)
    if epilogue == EPI_QUICK_GELU:
        e = torch.zeros_like(y)
    elif epilogue == EPI_GELU_TANH:
        x = v.double()
        u = 0.7978845608028654 * (x + 0.044715 * x**3)
        e = 0.5 * x.abs() * (3 * 2.0**-23 + (1 - torch.tanh(u) ** 2) * (2.0**-23 + u.abs() * 2.0**-21))
    else:
        assert epilogue == EPI_GELU_ERF, epilogue
        e = v.double().abs() * 2.0**-22
    return ulp16(y) + e


def act32(v: torch.Tensor, epilogue: int, k1: float = 0.044715) -> torch.Tensor:
    """The kernel's formulas in float32 torch (exact division and torch's exp2 / erf in place of the intrinsics)."""
    x = v.float()
    if epilogue == EPI_QUICK_GELU:
        return x / (1.0 + torch.exp2(-2.4554669595930156 * x))
    if epilogue == EPI_GELU_TANH:
        u = 0.7978845608028654 * (x + k1 * x * x * x)
        e = torch.exp2(2.885390081777927 * u)
        t = 1.0 - 2.0 / (e + 1.0)
        return 0.5 * x * (1.0 + t)
    if epilogue == EPI_GELU_ERF:
        return 0.5 * x * (1.0 + torch.erf(x * 0.7071067811865476))
    assert epilogue == EPI_NONE, epilogue
    return x


def v_grid(lo: float = -12.0, hi: float = 12.0) -> torch.Tensor:
    """Every multiple of 2^-6 in [lo, hi]: the pre-activations z + bias the sparse inputs produce."""
    return torch.arange(int(lo * 64), int(hi * 64) + 1, dtype=torch.float64) / 64
