"""The wgmma GEMM (cb_gemm_f16_ex) against oracle/gemm.py, every instantiation at every boundary of its dispatch.

* exact: integer operands make the fp32 accumulator exact, so fp16 NONE, fp32 (no residual, a separate residual, the residual
  aliasing the output) and SCALE (general gamma and residual) must equal the oracle's emulation of the epilogue bit for bit;
  position-coded operands say where a misplaced element came from;
* bounded: the three activations on the same inputs, within the oracle's per-element bound (the worst err/bound per instantiation
  is printed when the module ends);
* every call reads A, W and the residual with NaN rows after them and writes into a NaN-filled buffer: nothing outside [M][N] may be
  written, no NaN may reach the output;
* slot invariance: rolling A's rows rolls the output's rows, rolling W's rows (with bias and gamma) rolls its columns, bit for bit;
* repeat launches; the host's argument checks, each before any launch.
"""

from __future__ import annotations

import zlib

import pytest
import torch

from gpu_helpers import ctx  # noqa: F401
from oracle import gemm as G

pytestmark = pytest.mark.gpu

PAD = 3  # NaN rows after A, W and a separate residual; NaN rows before and after the output
NAMES = [p.name for p in G.sweep(G.SM_COUNTS[0])]


def _sm(ctx) -> int:
    return ctx.device_info()["sm_count"]


def _nan_after(x: torch.Tensor) -> torch.Tensor:
    """x [R][C] as the first R rows of a buffer whose PAD rows after it are NaN."""
    buf = torch.full((x.shape[0] + PAD, x.shape[1]), float("nan"), dtype=x.dtype, device="cuda")
    buf[: x.shape[0]] = x
    return buf[: x.shape[0]]


def _bits(x: torch.Tensor) -> torch.Tensor:
    return x.view(torch.int32 if x.dtype == torch.float32 else torch.int16)


def _call(ctx, a, w, bias, gamma, residual, o32, o16, m, n, k, epi) -> int:
    from cosmos_curate_b200.runtime import _stream_ptr

    return ctx.lib.cb_gemm_f16_ex(ctx.h, a, w, bias, gamma, residual, o32, o16, m, n, k, epi, _stream_ptr())


def _run(ctx, a, w, bias=None, gamma=None, residual=None, out_f32=False, epi=G.EPI_NONE, alias=False) -> torch.Tensor:
    """cb_gemm_f16_ex with a and w copied to _nan_after buffers, the output PAD rows into a NaN-filled buffer (prefilled with the residual when
    `alias`, else the residual from its own _nan_after buffer); asserts nothing outside [M][N] changed, the separate residual is as
    it was and the output holds no NaN, and returns the output."""
    from cosmos_curate_b200.runtime import check

    m, k = a.shape
    n = w.shape[0]
    a, w = _nan_after(a), _nan_after(w)
    dt = torch.float32 if out_f32 else torch.float16
    buf = torch.full(((m + 2 * PAD) * n,), float("nan"), dtype=dt, device="cuda")
    out = buf[PAD * n : (PAD + m) * n].view(m, n)
    rptr, r_sep = None, None
    if residual is not None:
        if alias:
            out.copy_(residual)
            rptr = out.data_ptr()
        else:
            r_sep = _nan_after(residual)
            rptr = r_sep.data_ptr()
    before = buf.clone()
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    o32, o16 = (out.data_ptr(), None) if out_f32 else (None, out.data_ptr())
    check(_call(ctx, a.data_ptr(), w.data_ptr(), ptr(bias), ptr(gamma), rptr, o32, o16, m, n, k, epi), "cb_gemm_f16_ex", ctx.h)
    torch.cuda.synchronize()
    assert torch.equal(_bits(buf[: PAD * n]), _bits(before[: PAD * n])), "rows before the output were written"
    assert torch.equal(_bits(buf[(PAD + m) * n :]), _bits(before[(PAD + m) * n :])), "rows after the output were written"
    if r_sep is not None:
        assert torch.equal(_bits(r_sep), _bits(residual)), "the separate residual was written"
    assert not torch.isnan(out).any(), f"NaN in the output: {torch.isnan(out).nonzero()[0].tolist()} is the first"
    return out


def _assert_bitwise(got: torch.Tensor, want: torch.Tensor, what: str, position: bool | None = None) -> None:
    bad = (_bits(got) != _bits(want)).nonzero()
    if len(bad):
        m, n = bad[0].tolist()
        g, w = got[m, n].item(), want[m, n].item()
        where = f" (got decodes to {G.decode_position(g, position)})" if position is not None else ""
        pytest.fail(f"{what}: {len(bad)} of {got.numel()} elements differ; first at (m={m}, n={n}): got {g!r} want {w!r}{where}")


@pytest.fixture(scope="module")
def worst():
    """Worst err/bound per activation instantiation, printed when the module ends."""
    w: dict[str, float] = {}
    yield w
    for name, r in sorted(w.items()):
        print(f"\ngemm {name}: worst err/bound {r:.3f}", end="")
    print()


def test_sweep_names_do_not_depend_on_the_sm_count(ctx):
    assert [p.name for p in G.sweep(_sm(ctx))] == NAMES


@pytest.mark.parametrize("name", NAMES)
def test_gemm_sweep(ctx, worst, name):
    sm = _sm(ctx)
    pt = {p.name: p for p in G.sweep(sm)}[name]
    m, n, k = pt.m, pt.n, pt.k
    seed = zlib.crc32(name.encode())
    g = torch.Generator(device="cuda").manual_seed(seed)
    bias = G.grid_bias(n, seed, "cuda")
    gamma = torch.rand(n, generator=g, device="cuda") * 1.45 + 0.05
    res = torch.randn(m, n, generator=g, device="cuda") * 4
    at = f"at {name} (M={m} N={n} K={k}, {sm} SMs)"
    for kind, gen in (("integer", G.int_operands), ("sparse", G.sparse_operands)):
        a, w = gen(m, n, k, seed + 1, "cuda")
        z = G.exact_product(a, w)
        for p, epi, out_f32, scale in G.launches(pt, sm):
            what = f"{p.inst} {at}, {kind} inputs"
            if not out_f32:
                got = _run(ctx, a, w, bias, epi=epi)
                if epi == G.EPI_NONE:
                    _assert_bitwise(got, G.emulate(z, bias, None, None, False), what)
                    continue
                v = G.emulate(z, bias, None, None, True)  # f32(z + b), the activation's exact argument
                ratio = (got.double() - G.act64(v, epi)).abs() / G.act_bound(v, epi)
                r = ratio.max().item()
                worst[p.inst] = max(worst.get(p.inst, 0.0), r)
                if r > 1.0:
                    i, j = divmod(int(ratio.argmax()), n)
                    pytest.fail(f"{what}: err/bound {r:.3f} at (m={i}, n={j}): v = {v[i, j].item()!r}, got {got[i, j].item()!r}, "
                                f"want {G.act64(v[i, j], epi).item()!r}")  # fmt: skip
                continue
            gam = gamma if scale else None
            for mode in ("none", "separate", "aliased") if not scale else ("separate", "aliased"):
                r = None if mode == "none" else res
                got = _run(ctx, a, w, bias, gam, r, out_f32=True, alias=mode == "aliased")
                _assert_bitwise(got, G.emulate(z, bias, gam, r, True), f"{what}, residual {mode}")
    for out_f32 in (False, True):
        a, w = G.position_operands(m, n, k, out_f32, "cuda")
        z = G.exact_product(a, w)
        got = _run(ctx, a, w, out_f32=out_f32)
        p = G.plan(m, n, k, False, out_f32, G.EPI_NONE, sm)
        _assert_bitwise(got, G.emulate(z, None, None, None, out_f32), f"{p.inst} {at}, position-coded inputs", position=out_f32)


def _slot_case(inst: str, sm: int):
    """A shape this instantiation runs at with >= 3 tiles on a CTA, and random real-valued operands."""
    bn, epi, out_f32, scale = G.INSTANTIATION_ARGS[inst]
    n, k = (1280, 200) if bn == 256 else (640, 200)  # five 256-wide column tiles / 640 is never wide
    m = G.m_with(G.cdiv(2 * sm + 1, 5), 77)
    assert G.plan(m, n, k, scale, out_f32, epi, sm).inst == inst
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(inst.encode()))
    a = torch.randn(m, k, generator=g, device="cuda").half()
    w = (torch.randn(n, k, generator=g, device="cuda") / k**0.5).half()
    bias = torch.randn(n, generator=g, device="cuda")
    gamma = torch.rand(n, generator=g, device="cuda") + 0.1 if scale else None
    res = torch.randn(m, n, generator=g, device="cuda") if out_f32 else None
    return a, w, bias, gamma, res, out_f32, epi


ROLL_ROWS, ROLL_COLS = 37, 40  # 40: a multiple of 8 and of neither slice width (32 fp32 / 64 fp16 columns)


@pytest.mark.parametrize("inst", G.INSTANTIATIONS)
def test_slot_invariance(ctx, inst):
    """An output element does not depend on where in its tile, slice or accumulator registers it is computed."""
    a, w, bias, gamma, res, out_f32, epi = _slot_case(inst, _sm(ctx))
    base = _run(ctx, a, w, bias, gamma, res, out_f32, epi)
    roll = lambda t, s, d=0: t.roll(s, d) if t is not None else None  # noqa: E731
    rows = _run(ctx, a.roll(ROLL_ROWS, 0), w, bias, gamma, roll(res, ROLL_ROWS), out_f32, epi)
    _assert_bitwise(rows, base.roll(ROLL_ROWS, 0), f"{inst}: A's rows rolled by {ROLL_ROWS} vs the output's rows rolled")
    cols = _run(ctx, a, w.roll(ROLL_COLS, 0), bias.roll(ROLL_COLS), roll(gamma, ROLL_COLS), roll(res, ROLL_COLS, 1), out_f32, epi)
    _assert_bitwise(cols, base.roll(ROLL_COLS, 1), f"{inst}: W's rows rolled by {ROLL_COLS} vs the output's columns rolled")


@pytest.mark.parametrize("inst", G.INSTANTIATIONS)
def test_repeat_launches_bitwise_equal(ctx, inst):
    a, w, bias, gamma, res, out_f32, epi = _slot_case(inst, _sm(ctx))
    first = _run(ctx, a, w, bias, gamma, res, out_f32, epi, alias=True)
    for _ in range(2):
        _assert_bitwise(_run(ctx, a, w, bias, gamma, res, out_f32, epi, alias=True), first, f"{inst}: a repeat launch")


ARG, UNSUPPORTED = -2, -3
_ERRORS = [  # name, changes to a valid 64 x 64 x 64 fp16-output call, code
    ("n_not_multiple_of_8", {"N": 60}, ARG),
    ("k_not_multiple_of_8", {"K": 36}, ARG),
    ("a_misaligned", {"A": 8}, ARG),
    ("w_misaligned", {"W": 8}, ARG),
    ("out_f16_misaligned", {"out16": 8}, ARG),
    ("out_f32_misaligned", {"out16": None, "out32": 8}, ARG),
    ("residual_misaligned", {"out16": None, "out32": 0, "residual": 8}, ARG),
    ("gamma_misaligned", {"out16": None, "out32": 0, "gamma": 4}, ARG),
    ("quick_gelu_with_f32_out", {"out16": None, "out32": 0, "epi": G.EPI_QUICK_GELU}, UNSUPPORTED),
    ("gelu_tanh_with_f32_out", {"out16": None, "out32": 0, "epi": G.EPI_GELU_TANH}, UNSUPPORTED),
    ("gelu_erf_with_f32_out", {"out16": None, "out32": 0, "epi": G.EPI_GELU_ERF}, UNSUPPORTED),
    ("residual_with_f16_out", {"residual": 0}, UNSUPPORTED),
    ("gamma_with_f16_out", {"gamma": 0}, UNSUPPORTED),
    ("m_zero", {"M": 0}, ARG),
    ("m_negative", {"M": -1}, ARG),
    ("n_zero", {"N": 0}, ARG),
    ("n_negative", {"N": -8}, ARG),
    ("k_zero", {"K": 0}, ARG),
    ("k_negative", {"K": -64}, ARG),
    ("unknown_epilogue", {"epi": 4}, ARG),
    ("negative_epilogue", {"epi": -1}, ARG),
    ("null_output", {"out16": None}, ARG),
]


@pytest.mark.parametrize(("changes", "code"), [e[1:] for e in _ERRORS], ids=[e[0] for e in _ERRORS])
def test_rejected_on_the_host(ctx, changes, code):
    """Each bad argument returns its code before anything is launched.  Every buffer is 1 MB, so that even the misaligned and
    mis-sized calls name memory a kernel could read and write without leaving it."""
    bufs = {name: torch.full((1 << 18,), float("nan"), device="cuda") for name in ("A", "W", "bias", "gamma", "residual", "out32", "out16")}
    before = {name: b.clone() for name, b in bufs.items()}
    call = {"A": 0, "W": 0, "bias": 0, "gamma": None, "residual": None, "out32": None, "out16": 0, "M": 64, "N": 64, "K": 64, "epi": 0}
    call.update(changes)
    ptr = {name: None if call[name] is None else bufs[name].data_ptr() + call[name] for name in bufs}
    launches = ctx.launch_count()
    rc = _call(ctx, ptr["A"], ptr["W"], ptr["bias"], ptr["gamma"], ptr["residual"], ptr["out32"], ptr["out16"], call["M"], call["N"],
               call["K"], call["epi"])  # fmt: skip
    torch.cuda.synchronize()
    assert rc == code
    assert ctx.launch_count() == launches, "a kernel was launched"
    for name, b in bufs.items():
        assert torch.equal(_bits(b), _bits(before[name])), f"{name} was written"
