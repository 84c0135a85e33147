"""The GEMM oracle (oracle/gemm.py) is well-posed: its dispatch is the one written in csrc/gemm.cu, its sweep puts every kernel
instantiation on every boundary of that dispatch for both H100 SM counts, its inputs make the fp32 accumulator exact, its epilogue
model rounds as float64 step-by-step arithmetic says, and its activation bound holds for the kernel's formulas while catching
small changes to them."""

from __future__ import annotations

import re
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import gemm as G

GEMM_CU = Path(__file__).resolve().parent.parent / "cosmos_curate_b200" / "csrc" / "gemm.cu"


def _c_expr(pattern: str, names: str):
    """A function of `names` evaluating the C expression that `pattern`'s first group captures in gemm.cu (integer division, one
    ternary, &&, ||, !, std::min, member access dropped)."""
    src = GEMM_CU.read_text()
    m = re.search(pattern, src)
    assert m, f"gemm.cu no longer contains {pattern!r}: restate the rule in oracle/gemm.py and here"
    e = m.group(1)
    e = e.replace("ctx->", "").replace("g.", "").replace("std::min", "min").replace("&&", " and ").replace("||", " or ")
    e = re.sub(r"!(?!=)", " not ", e).replace("/", "//")
    t = re.fullmatch(r"(.+?)\s*\?\s*(.+?)\s*:\s*(.+)", e)
    if t:
        e = f"(({t.group(2)}) if ({t.group(1)}) else ({t.group(3)}))"
    return eval(f"lambda {names}: {e}")  # noqa: S307 - the expression is the repository's own source


def test_dispatch_matches_gemm_cu():
    tiles256 = _c_expr(r"const int tiles256 = ([^;]+);", "M, N, BM")
    wide = _c_expr(r"const bool wide = ([^;]+);", "gamma, N, tiles256, sm_count")
    kstages = _c_expr(r"kStages = ([^;]+);", "BN")
    tiles = _c_expr(r"const int tiles = ([^;]+);", "M, N, BM, BN")
    grid = _c_expr(r"kern<<<(.+?), kGemmThreads", "tiles, sm_count")
    kslice = _c_expr(r"kSliceCols = ([^;]+);", "OUT_F32")
    nsl = _c_expr(r"const int nslices = ([^;]+);", "row0, M, N, col0, kSlices, kSliceCols")
    num_kb = _c_expr(r"const int num_kb = ([^;]+);", "K, BK")
    for sm in (*G.SM_COUNTS, 100, 7):
        for m in (1, 63, 64, 65, 128, 129, 1000, 4095, 4225, 8000, 17000):
            for n in (8, 120, 128, 248, 256, 264, 512, 1016, 1024, 1032, 1280, 1408, 4304):
                for gamma in (False, True):
                    for out_f32 in (False, True):
                        k = 8 * (m % 97 + 1)
                        p = G.plan(m, n, k, gamma, out_f32, G.EPI_NONE, sm)
                        bn = 256 if wide(gamma, n, tiles256(m, n, G.BM), sm) else 128
                        case = (sm, m, n, gamma, out_f32)
                        assert p.bn == bn and p.stages == kstages(bn), case
                        assert p.tiles == tiles(m, n, G.BM, bn) and p.grid == grid(p.tiles, sm), case
                        assert p.slice_cols == kslice(out_f32) and p.num_kb == num_kb(k, G.BK), case
                        for t in {0, p.n_tiles - 1, p.tiles - 1}:
                            m_blk, n_blk = divmod(t, p.n_tiles)
                            for c in (0, 1):
                                want = nsl(m_blk * G.BM + 64 * c, m, n, n_blk * bn, bn // p.slice_cols, p.slice_cols)
                                assert G.nslices(p, m, n, t, c) == want, (case, t, c)


def test_instantiations_match_gemm_cu():
    src = GEMM_CU.read_text()
    names = set()
    for bn, epi, out_f32, scale in re.findall(r"launch_gemm<(\w+), CB_EPI_(\w+), (true|false)(?:, (true))?>\(ctx", src):
        e = {v: k for k, v in G.EPI_NAME.items()}[epi]
        for b in ((128, 256) if bn == "BN" else (int(bn),)):
            names.add(G.instantiation(b, e, out_f32 == "true", scale == "true"))
    assert names == set(G.INSTANTIATIONS) and len(names) == 11


def test_plan_examples():
    assert G.plan(257, 3072, 1024, False, False, G.EPI_NONE, 132).bn == 128  # 3 x 12 = 36 wide tiles: too few
    p = G.plan(1025, 4224, 1408, False, False, G.EPI_GELU_ERF, 132)  # 9 x 17 = 153 wide tiles
    assert (p.inst, p.stages, p.grid, p.num_kb, p.max_tiles_per_cta) == ("<256,GELU_ERF,f16>", 4, 132, 22, 2)
    assert G.plan(1025, 4224, 1408, True, True, G.EPI_NONE, 132).inst == "<128,NONE,f32,SCALE>"
    p = G.plan(65, 8, 8, False, True, G.EPI_NONE, 132)
    assert (p.tiles, G.nslices(p, 65, 8, 0, 0), G.nslices(p, 65, 8, 0, 1)) == (1, 1, 1)
    assert G.nslices(G.plan(64, 8, 8, False, True, G.EPI_NONE, 132), 64, 8, 0, 1) == 0  # the M tail: the second warpgroup stores nothing


@pytest.mark.parametrize("sm", G.SM_COUNTS)
def test_sweep_reaches_every_instantiation_and_boundary(sm):
    cov = G.coverage(sm)
    print(f"\nSM count {sm}: boundary classes each instantiation runs at")
    for inst in G.INSTANTIATIONS:
        print(f"  {inst:22s} {' '.join(sorted(cov[inst]))}")
    for inst in G.INSTANTIATIONS:
        missing = G.required_classes(int(inst[1:4])) - cov[inst]
        assert not missing, (inst, sorted(missing))
    pts = {p.name: p for p in G.sweep(sm)}
    assert len(pts) == len(G.sweep(sm))
    # both sides of every clause of the wide predicate
    for n in (512, 1024, 1032, 1408):
        nt = G.cdiv(n, 256)
        below, at = pts[f"predicate_n={n}_below"], pts[f"predicate_n={n}_at"]
        assert (below.n, at.n) == (n, n)
        t_below, t_at = G.cdiv(below.m, 128) * nt, G.cdiv(at.m, 128) * nt
        assert t_below == (sm - 1) // nt * nt and t_at == G.cdiv(sm, nt) * nt, n  # the largest below, the smallest at or above
        assert G.tile_width(below.m, n, below.k, False, False, 0, sm) == 128 and G.tile_width(at.m, n, at.k, False, False, 0, sm) == 256
        assert G.tile_width(at.m, n, at.k, True, True, 0, sm) == 128  # gamma: never wide
    p = pts["predicate_n=1016"]
    assert G.cdiv(p.m, 128) * 4 >= sm and G.tile_width(p.m, 1016, p.k, False, False, 0, sm) == 128
    assert {(n, k) for _, _, n, k in G.TOWERS} <= {(p.n, p.k) for p in pts.values()}
    assert {640, 768} <= {p.k for p in pts.values() if p.name.startswith("patch")}
    for p in pts.values():
        assert p.n % 8 == 0 and p.k % 8 == 0 and p.m > 0


@pytest.mark.parametrize("sm", G.SM_COUNTS)
def test_odd_slice_tails_start_tiles_with_both_buffers(sm):
    """Every N tail of the sweep that leaves an odd slice count runs, for each instantiation of its tile width and output type, at
    a point with >= 3 tiles on a CTA where tiles start on both buffers and on both parities of that buffer's residual barrier."""
    want, got = set(), set()
    for pt in G.sweep(sm):
        for p, _, _, _ in G.launches(pt, sm):
            tail = pt.n % p.bn
            if tail in (*G.N_TAILS, p.bn - 8) and G.cdiv(tail, p.slice_cols) % 2 == 1:
                want.add((p.inst, tail))
                if p.max_tiles_per_cta >= 3 and G.starts_with_both_parities(p, pt.m, pt.n):
                    got.add((p.inst, tail))
    assert want and want == got, sorted(want - got)


def _worst_partial_sum(a: torch.Tensor, w: torch.Tensor) -> float:
    """max over outputs and over k of |sum_{j <= k} a_j w_j|, and the sum of |a_j w_j| that bounds any order's partial sums."""
    prods = a.double()[:, None, :] * w.double()[None, :, :]
    return max(prods.cumsum(-1).abs().max().item(), prods.abs().sum(-1).max().item())


@pytest.mark.parametrize("sm", G.SM_COUNTS)
def test_generators_are_exact(sm):
    for i, k in enumerate(sorted({p.k for p in G.sweep(sm)})):
        for a, w in (G.int_operands(9, 7, k, seed=i), G.sparse_operands(9, 7, k, seed=i)):
            assert torch.equal(a.float().half(), a) and torch.equal(w.float().half(), w)
            assert a.abs().max() <= 8 and w.abs().max() <= 8
            assert 64 * k < 2**24 and _worst_partial_sum(a, w) < 2**24
            assert torch.equal(a.float().round(), a.float()) and torch.equal(w.float().round(), w.float())
        for out_f32, m, n in ((True, 2050, 4100), (False, 130, 70)):
            rows = torch.tensor([0, 1, 63, 64, 127, 128, 2047, 2048, 2049][: 9 if out_f32 else 6])
            cols = torch.tensor([0, 7, 31, 32, 63, 64, 4095, 4096][: 8 if out_f32 else 4])
            a, w = G.position_operands(m, n, k, out_f32)
            a, w = a[rows], w[cols]
            z = G.exact_product(a, w)
            assert _worst_partial_sum(a, w) < 2**24
            assert torch.equal(z.float().double(), z)  # exact in fp32
            if not out_f32:
                assert torch.equal(z.half().double(), z) and z.abs().max() <= 2048  # exact in fp16
            for ri, r in enumerate(rows.tolist()):
                for ci, c in enumerate(cols.tolist()):
                    want = f"row = {r % 2048} (mod 2048), column = {c % 4096}" if out_f32 else f"row = {r % 128} (mod 128), column = {c % 32}"
                    assert G.decode_position(z[ri, ci].item(), out_f32).startswith(want)
    b = G.grid_bias(1000, seed=1)
    assert torch.equal((b * 64).round(), b * 64) and b.abs().max() <= 1
    z = torch.arange(-2**17 + 1, 2**17, 977, dtype=torch.float64)
    assert torch.equal((z[:, None] + b.double()[None]).float().double(), z[:, None] + b.double()[None])  # z + b exact in fp32


def _f32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def test_emulation_matches_float64_steps():
    """emulate() against a float64 evaluation rounded to the target type after each kernel operation, with general (not
    power-of-two) fp32 bias, gamma and residual, including tiny, huge and subnormal values."""
    g = torch.Generator().manual_seed(7)
    m, n = 300, 200
    z = torch.randint(-2**23, 2**23, (m, n), generator=g).double()
    z[0] = torch.randint(-50, 50, (n,), generator=g).double()
    z[1] = 0.0
    bias = torch.randn(n, generator=g) * torch.exp2(torch.randint(-30, 10, (n,), generator=g).float())
    gamma = torch.rand(n, generator=g) * 1.45 + 0.05
    gamma[:5] = torch.tensor([1e-5, 2.0**-130, 3e-38, -0.7, 1.0])
    res = torch.randn(m, n, generator=g) * torch.exp2(torch.randint(-20, 25, (m, n), generator=g).float())
    res[2] = -(z[2] + bias.double()).float()  # exact cancellation: +0
    zn, bn, gn, rn = z.numpy(), bias.double().numpy(), gamma.double().numpy(), res.double().numpy()
    v = _f32(zn + bn)
    with np.errstate(over="ignore"):  # |z| >= 65520 overflows fp16 to +-inf, in the kernel's conversion too
        want16 = (zn + bn).astype(np.float32).astype(np.float16)
        want16_nobias = zn.astype(np.float32).astype(np.float16)
    assert np.array_equal(G.emulate(z, bias, None, None, False).numpy().view(np.int16), want16.view(np.int16))
    assert np.array_equal(G.emulate(z, None, None, None, False).numpy().view(np.int16), want16_nobias.view(np.int16))
    for gam, r in ((None, None), (None, res), (gamma, None), (gamma, res)):
        want = v
        if gam is not None:
            want = _f32(want * gn)  # the product of two fp32 numbers is exact in float64
        if r is not None:
            want = _f32(want + rn)  # float64 then fp32: an innocuous double rounding (53 >= 2 * 24 + 2)
        got = G.emulate(z, bias, gam, r, True).numpy()
        assert np.array_equal(got.view(np.int32), want.astype(np.float32).view(np.int32)), (gam is None, r is None)


V = G.v_grid()


def _exceeds(y: torch.Tensor, epi: int) -> int:
    """Grid points where fp16(y) (y an alternative activation in float64) is outside the bound of `epi`."""
    return int(((y.half().double() - G.act64(V, epi)).abs() > G.act_bound(V, epi)).sum())


def test_activation_bound_is_not_vacuous():
    def tanh_form(x, k1=0.044715):
        return 0.5 * x * (1 + torch.tanh(0.7978845608028654 * (x + k1 * x**3)))

    assert _exceeds(V * torch.sigmoid(1.70 * V), G.EPI_QUICK_GELU) > 0  # 1.702 written as 1.70
    assert _exceeds(tanh_form(V, 0.0447), G.EPI_GELU_TANH) > 0  # k1 written as 0.0447
    assert _exceeds(tanh_form(V), G.EPI_GELU_ERF) > 0  # the tanh form where erf is expected
    for epi in G.ACTIVATIONS:
        assert _exceeds(G.act64(V, epi), epi) == 0
        assert _exceeds(G.act64(V, epi) + 2 * G.ulp16(G.act64(V, epi)), epi) > 0  # 2 ulp off: out


def test_activation_bound_holds_for_the_kernel_formulas_in_float32():
    """The kernel's formulas in float32, as written and with the intrinsics' worst errors (exp2f 2 ulp, div.approx 2 ulp, erff 2
    ulp) applied in either direction, rounded to fp16: within the bound on the whole grid."""
    x = V.float()
    for epi in G.ACTIVATIONS:
        assert (G.act32(V, epi).half().double() - G.act64(V, epi)).abs().le(G.act_bound(V, epi)).all(), epi
    worst = {}
    for se in (1 + 2.0**-22, 1 - 2.0**-22):
        for sq in (1 + 2.0**-23, 1 - 2.0**-23):
            u = 0.7978845608028654 * (x + 0.044715 * x * x * x)
            e = torch.exp2(2.885390081777927 * u) * se
            t = 1.0 - (2.0 / (e + 1.0)) * sq
            cand = {G.EPI_GELU_TANH: 0.5 * x * (1.0 + t), G.EPI_QUICK_GELU: x / (1.0 + torch.exp2(-2.4554669595930156 * x) * se) * sq}
            erf = torch.erf(x * 0.7071067811865476)
            cand[G.EPI_GELU_ERF] = 0.5 * x * (1.0 + erf + torch.where(erf.abs() >= 0.5, torch.sign(erf) * (sq - 1) * 2, erf * (sq - 1)))
            for epi, y in cand.items():
                r = ((y.half().double() - G.act64(V, epi)).abs() / G.act_bound(V, epi)).max().item()
                worst[epi] = max(worst.get(epi, 0.0), r)
    print({G.EPI_NAME[k]: round(v, 3) for k, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst
