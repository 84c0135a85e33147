"""The shot network's kernels (csrc/transnet.cu) through the C ABI, against oracle/transnet_kernels.py.

* conv (every instantiation, at every sweep point of `conv_sweep`), shortcut_pool, spatial_mean, l2_normalize_rows,
  window_similarity_fc and window_gather: bit for bit equal to their float32 models on the exact and the random input classes, and
  on the exact class equal to the float64 reference too, up to full 100-frame windows x max_windows;
* head: bit for bit equal to one of its expf candidates per row; the histogram of the candidates used is printed when the module ends;
* inputs have NaN guard rows after them (and NaN in the columns a launch must not read); outputs go into NaN-filled buffers with guard
  rows on both sides: nothing outside the output may change and no NaN may reach it;
* a poisoned window next to a clean one leaves the clean one's bits unchanged, for every dilation;
* the same rows give the same bits under every instantiation and at any row offset;
* ShotNet.forward equals a replay of run_windows' schedule through the entry points, bit for bit, and predict's stitching equals
  forward on each window alone;
* every argument error returns its code before any launch; repeat launches are bitwise equal.
"""

from __future__ import annotations

import ctypes as C
import zlib
from collections import Counter

import numpy as np
import pytest
import torch

from gpu_helpers import ctx  # noqa: F401
from oracle import transnet_kernels as K
from oracle import transnetv2 as tn

pytestmark = pytest.mark.gpu

F32 = np.float32
PAD = 3  # NaN rows after every input, NaN guard rows before and after every output
MAX_WINDOWS = 4
CB_ERR_ARG, CB_ERR_UNSUPPORTED = -2, -3


def _stream():
    from cosmos_curate_b200.runtime import _stream_ptr

    return _stream_ptr()


def _seed(name: str) -> int:
    return zlib.crc32(name.encode())


def _bits(a: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=F32).view(np.int32)


def _ok(ctx, rc: int, what: str) -> None:  # noqa: F811
    from cosmos_curate_b200.runtime import check

    check(rc, what, ctx.h)


def _assert_bitwise(got: np.ndarray, want: np.ndarray, what: str) -> None:
    bad = np.argwhere(_bits(got) != _bits(want))
    if len(bad):
        i = tuple(bad[0])
        pytest.fail(f"{what}: {len(bad)} of {got.size} elements differ; first at {list(i)}: got {got[i]!r} want {want[i]!r}")


_LIVE: list[torch.Tensor] = []


@pytest.fixture(autouse=True)
def _inputs_live_until_the_test_ends():
    yield
    torch.cuda.synchronize()
    _LIVE.clear()


def _in(a: np.ndarray, dtype=None) -> torch.Tensor:
    """a on the device as the first rows of a buffer whose PAD rows after it are NaN (0xff bytes for uint8)."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    fill = 255 if t.dtype == torch.uint8 else (-1 if t.dtype == torch.int32 else float("nan"))
    buf = torch.full((t.shape[0] + PAD, *t.shape[1:]), fill, dtype=t.dtype, device="cuda")
    buf[: t.shape[0]] = t.cuda()
    _LIVE.append(buf)
    return buf[: t.shape[0]]


class Out:
    """A NaN-filled fp32 output [rows][cols] with PAD guard rows before and after; `mask` [cols] marks the columns the launch writes."""

    def __init__(self, rows: int, cols: int, mask: np.ndarray | None = None):
        self.buf = torch.full((rows + 2 * PAD, cols), float("nan"), dtype=torch.float32, device="cuda")
        self.t = self.buf[PAD : PAD + rows]
        self.rows, self.mask = rows, (np.ones(cols, bool) if mask is None else mask)
        self.before = self.buf.clone()

    @property
    def ptr(self) -> int:
        return self.t.data_ptr()

    def get(self, what: str, nan_ok: bool = False) -> np.ndarray:
        """The output after the guards are checked; nan_ok where the inputs themselves are poisoned."""
        torch.cuda.synchronize()
        b, a = _bits(self.buf.cpu().numpy()), _bits(self.before.cpu().numpy())
        assert np.array_equal(b[:PAD], a[:PAD]), f"{what}: rows before the output were written"
        assert np.array_equal(b[PAD + self.rows :], a[PAD + self.rows :]), f"{what}: rows after the output were written"
        assert np.array_equal(b[PAD : PAD + self.rows][:, ~self.mask], a[PAD : PAD + self.rows][:, ~self.mask]), f"{what}: columns outside the output were written"
        out = self.t.cpu().numpy()
        w = out[:, self.mask]
        assert nan_ok or not np.isnan(w).any(), f"{what}: NaN in the output at {np.argwhere(np.isnan(w))[0].tolist()}"
        return out

    def untouched(self, what: str) -> None:
        torch.cuda.synchronize()
        assert np.array_equal(_bits(self.buf.cpu().numpy()), _bits(self.before.cpu().numpy())), f"{what}: the buffer was written"


@pytest.fixture(scope="module")
def record(pytestconfig):
    r = {"expf": Counter()}
    yield r
    total = sum(r["expf"].values())
    line = "head expf candidate per row (ulps from the correctly rounded exp): " + ", ".join(
        f"{k:+d}: {r['expf'][k]}" for k in range(-K.EXPF_ULP, K.EXPF_ULP + 1)) + f" (rows {total})"  # fmt: skip
    capman = pytestconfig.pluginmanager.get_plugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print("\n" + line)


# ------------------------------------------------------------------------------------------------ conv
def _conv_args(a: dict, inp: int, w: int, out: int, scale: int | None, shift: int | None):
    from cosmos_curate_b200._lib import TransnetConvArgs

    s = TransnetConvArgs()
    s.in_, s.w, s.out, s.scale, s.shift = inp, w, out, scale, shift
    for k in ("M", "N", "cin", "in_ld", "in_coff", "w_ld", "out_ld", "out_coff", "T", "H", "W", "mode", "dil", "relu", "z_in_coff",
              "z_out_coff", "z_dil_shift", "z_w"):  # fmt: skip
        setattr(s, k, int(a[k]))
    return s


def _out_mask(a: dict) -> np.ndarray:
    m = np.zeros(a["out_ld"], bool)
    for z in range(a["z"]):
        m[a["out_coff"] + z * a["z_out_coff"] :][: a["N"]] = True
    return m


def _conv(ctx, a, inp, w, scale, shift, in_rows_off: int = 0, nan_ok: bool = False) -> np.ndarray:  # noqa: F811
    """One cb_transnet_conv launch on host arrays; returns the output [M][out_ld] (guards checked)."""
    lib = ctx.lib
    x = _in(inp.reshape(-1, a["in_ld"]))
    wd, sd, hd = _in(w), (_in(scale) if scale is not None else None), (_in(shift) if shift is not None else None)
    out = Out(a["M"], a["out_ld"], _out_mask(a))
    args = _conv_args(a, x.data_ptr() + in_rows_off * a["in_ld"] * 4, wd.data_ptr(), out.ptr, sd.data_ptr() if sd is not None else None,
                      hd.data_ptr() if hd is not None else None)  # fmt: skip
    _ok(ctx, lib.cb_transnet_conv(ctx.h, C.byref(args), a["z"], _stream()), "cb_transnet_conv")
    return out.get("conv", nan_ok)


def _pick(out: np.ndarray, a: dict, rows) -> np.ndarray:
    """The written columns of `rows` as [len(rows)][z][N]."""
    return np.stack([out[rows, a["out_coff"] + z * a["z_out_coff"] :][:, : a["N"]] for z in range(a["z"])], 1)


def _conv_ref_all(a, inp, w_ref, scale, shift) -> np.ndarray:
    """float64 reference on the device, [M][z][N]."""
    x = inp.reshape(a["M"], a["in_ld"])
    ys = []
    for z in range(a["z"]):
        c0 = a["in_coff"] + z * a["z_in_coff"]
        acc = K.conv_ref(x[:, c0 : c0 + a["cin"]], w_ref[z], a["mode"], a["T"], a["H"], a["W"], dil=(a["dil"] << z) if a["z_dil_shift"] else a["dil"],
                         device="cuda")  # fmt: skip
        c = a["out_coff"] + z * a["z_out_coff"] + np.arange(a["N"])
        ys.append(K.epilogue_ref(acc, None if scale is None else scale[c], None if shift is None else shift[c], bool(a["relu"])).cpu().numpy())
    return np.stack(ys, 1)


SWEEP = K.conv_sweep()


@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("p", SWEEP, ids=lambda p: p.name)
def test_conv_matches_model_bitwise(ctx, p, kind):  # noqa: F811
    a = p.args()
    rng = np.random.default_rng(_seed(p.name + kind))
    inp, w, scale, shift, w_ref = K.conv_inputs(kind, p, a, rng)
    got = _conv(ctx, a, inp, w, scale, shift)
    rows = K.select_rows(p.M, p.inst, p.T, p.H, p.W, rng) if kind == "random" else np.arange(p.M)
    if kind == "exact":
        ref = _conv_ref_all(a, inp, w_ref, scale, shift)
        _assert_bitwise(_pick(got, a, rows), ref.astype(F32), f"{p.name} exact vs float64")
        assert np.array_equal(ref.astype(F32).astype(np.float64), ref)
    rows = rows if kind == "random" else K.select_rows(p.M, p.inst, p.T, p.H, p.W, rng, extra=8)
    _assert_bitwise(_pick(got, a, rows), K.conv_f32(inp, w, scale, shift, a, rows), f"{p.name} {kind} vs model")


@pytest.mark.parametrize("name", [l["name"] for l in K.schedule(1, 1) if l["kind"] == "conv"])
def test_conv_exact_class_at_full_windows(ctx, name):  # noqa: F811
    """Every conv launch of the network at B = max_windows 100-frame windows on the exact class: kernel == float64 reference."""
    L = next(l for l in K.schedule(MAX_WINDOWS, 100) if l.get("name") == name)
    p = K.ConvPoint(L["cin"], L["N"], L["M"], L["mode"], T=L["T"], H=L["H"], W=L["W"], z=L["z"],
                    epi="scale" if L["scale"] else ("shift" if L["shift"] else "none"), relu=L["relu"])  # fmt: skip
    a = dict(p.args(), in_ld=L["in_ld"], in_coff=0, w_ld=L["w_ld"], out_ld=L["out_ld"], out_coff=0, z_in_coff=L["z_in_coff"],
             z_out_coff=L["z_out_coff"], z_dil_shift=L["z_dil_shift"], z_w=L["z_w"])  # fmt: skip
    inp, w, scale, shift, w_ref = K.conv_inputs("exact", p, a, np.random.default_rng(_seed(name)))
    got = _conv(ctx, a, inp, w, scale, shift)
    ref = _conv_ref_all(a, inp, w_ref, scale, shift)
    _assert_bitwise(_pick(got, a, np.arange(p.M)), ref.astype(F32), f"{name} B={MAX_WINDOWS} T=100")


@pytest.mark.parametrize("T", [1, 8, 9, 100])
def test_conv_temporal_taps_stay_inside_their_window(ctx, T):  # noqa: F811
    """Window 0 all NaN, window 1 clean, four dilation branches (1, 2, 4, 8): window 1 equals its own launch bit for bit; relu off,
    no scale, so a NaN read would reach the output."""
    p = K.ConvPoint(32, 16, 2 * T * 2, 2, T=T, H=1, W=2, z=4, epi="shift")
    a = p.args()
    inp, w, scale, shift, _ = K.conv_inputs("random", p, a, np.random.default_rng(T))
    x = inp.reshape(p.M, a["in_ld"]).copy()
    win = T * 2
    x[:win] = np.nan
    got = _conv(ctx, a, x.reshape(-1), w, scale, shift, nan_ok=True)[win:]
    alone = _conv(ctx, dict(a, M=win), x[win:].reshape(-1), w, scale, shift)
    _assert_bitwise(_pick(got, a, np.arange(win)), _pick(alone, a, np.arange(win)), f"T={T} clean window next to a NaN one")
    # and with the clean window first
    x2 = np.concatenate([x[win:], x[:win]])
    got2 = _conv(ctx, a, x2.reshape(-1), w, scale, shift, nan_ok=True)[:win]
    _assert_bitwise(_pick(got2, a, np.arange(win)), _pick(alone, a, np.arange(win)), f"T={T} clean window before a NaN one")


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_conv_bits_do_not_depend_on_tile_shape_or_row_offset(ctx, mode):  # noqa: F811
    """The first 16 output columns of the same rows under all five instantiations (N = 16, 32, 64, 128 at cin 16; cin 20 with zero
    weights on channels 16..19 for <16,8,4>), and with the rows moved across tile boundaries, are bit-identical."""
    rng = np.random.default_rng(mode)
    T, H, W = 3, 4, 5
    M = 2 * T * H * W * 9  # 18 windows: several 128- and 256-row tiles
    taps = {0: 1, 1: 9, 2: 3}[mode]
    x = rng.standard_normal((M + 600, 20)).astype(F32)
    w16 = rng.standard_normal((taps, 16, 128)).astype(F32) * F32(0.1)
    sh = (rng.standard_normal(128) * 0.1).astype(F32)
    results = {}
    for cin, N in ((16, 16), (16, 32), (16, 64), (16, 128), (20, 128)):
        w = np.zeros((taps, cin, N), F32)
        w[:, :16] = w16[:, :, :N]
        a = dict(M=M, N=N, cin=cin, in_ld=20, in_coff=0, w_ld=N, out_ld=N, out_coff=0, T=T, H=H, W=W, mode=mode, dil=1, relu=0, z=1,
                 z_in_coff=0, z_out_coff=0, z_dil_shift=0, z_w=0)  # fmt: skip
        xi = x.copy()
        if cin == 16:
            xi[:, 16:] = np.nan  # never read
        for off in (0, 60, 300):  # whole windows, so mode 2 sees the same frames; output row i is input row off + i
            o = _conv(ctx, a, xi[off : off + M].reshape(-1), w.reshape(-1), None, sh[:N])
            results[(K.conv_inst(cin, N), off)] = o[300 - off : M - off, :16]  # input rows 300 .. M - 1
    base = results[((16, 8, 16), 0)]
    for key, v in results.items():
        _assert_bitwise(v, base, f"mode {mode} {key}")


# ------------------------------------------------------------------------------------------------ row kernels
def _gather(ctx, frames, first, pad, T):  # noqa: F811
    B = len(first)
    fr = _in(frames)
    fi, pa = _in(np.array(first, np.int32)), _in(np.array(pad, np.int32))
    x0, hist = Out(B * T, 1296 * 4), Out(B * T, 512)
    _ok(ctx, ctx.lib.cb_transnet_window_gather(ctx.h, fr.data_ptr(), fi.data_ptr(), pa.data_ptr(), B, T, x0.ptr, hist.ptr, _stream()), "window_gather")
    return x0.get("x0").reshape(B * T, 1296, 4), hist.get("hist")


@pytest.mark.parametrize("T", [1, 8, 9, 100])
def test_window_gather_bitwise_and_window_isolation(ctx, T):  # noqa: F811
    rng = np.random.default_rng(T)
    n = 2 * T + 3
    frames = rng.integers(0, 256, (n, 27, 48, 3), dtype=np.uint8)
    frames[: T + 3] = 255  # saturated frames: every pixel in one bin
    frames[1] = 0
    first, pad = [0, T + 3], [min(2, T - 1), 0]
    x0, hist = _gather(ctx, frames, first, pad, T)
    mx0, mh = K.window_gather_f32(frames, first, pad, T)
    _assert_bitwise(x0, mx0, "x0")
    _assert_bitwise(hist, mh, "hist")
    r0, rh = K.window_gather_ref(frames, first, pad, T)
    assert np.array_equal(x0[..., :3], r0.astype(F32)) and (np.abs(hist - rh) <= 3 * K.U * rh + 1e-45).all()
    a0, ah = _gather(ctx, frames, first[1:], pad[1:], T)
    _assert_bitwise(x0[T:], a0, "clean window x0")
    _assert_bitwise(hist[T:], ah, "clean window hist")


POOL_SHAPES = [(1, 27, 48, 64), (3, 13, 24, 128), (2, 6, 12, 256), (2, 1, 5, 4), (5, 3, 3, 12)]


@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("shape", POOL_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_shortcut_pool_and_spatial_mean_bitwise(ctx, shape, kind):  # noqa: F811
    fr, H, W, Cc = shape
    rng = np.random.default_rng(_seed(f"{shape}{kind}"))
    mk = (lambda: rng.integers(-6, 7, shape)) if kind == "exact" else (lambda: rng.standard_normal(shape))
    x2, x1 = mk().astype(F32), mk().astype(F32)
    hp, wp = H // 2, W // 2
    stride = hp * wp * Cc + 8
    out = Out(fr, stride, np.arange(stride) < hp * wp * Cc)
    _ok(ctx, ctx.lib.cb_transnet_shortcut_pool(ctx.h, _in(x2).data_ptr(), _in(x1).data_ptr(), out.ptr, fr, H, W, Cc, stride, _stream()), "pool")
    if hp * wp == 0:  # a one-row frame pools to nothing (floor): nothing is written
        out.untouched("pool of a one-row frame")
        return
    got = out.get("pool")[:, : hp * wp * Cc].reshape(fr, hp, wp, Cc)
    want = K.shortcut_pool_f32(x2, x1)
    _assert_bitwise(got, want, "shortcut_pool")
    if kind == "exact":
        assert np.array_equal(want.astype(np.float64), K.shortcut_pool_ref(x2, x1))
    feats = Out(fr, Cc + 12, (np.arange(Cc + 12) >= 4) & (np.arange(Cc + 12) < 4 + Cc))
    src = _in(out.t.cpu().numpy())
    _ok(ctx, ctx.lib.cb_transnet_spatial_mean(ctx.h, src.data_ptr(), stride, fr, hp * wp, Cc, feats.ptr, Cc + 12, 4, _stream()), "mean")
    mean = feats.get("mean")[:, 4 : 4 + Cc]
    _assert_bitwise(mean, K.spatial_mean_f32(got.reshape(fr, hp * wp, Cc)), "spatial_mean")


@pytest.mark.parametrize("D", [128, 512, 1, 33, 300])
def test_l2_normalize_rows_bitwise(ctx, D):  # noqa: F811
    rng = np.random.default_rng(D)
    x = (rng.standard_normal((37, D)) * rng.uniform(0.01, 30, (37, 1))).astype(F32)
    x[5] = 0  # max(|0|, 1e-12)
    buf = Out(37, D)
    buf.t.copy_(torch.from_numpy(x))
    buf.before = buf.buf.clone()
    _ok(ctx, ctx.lib.cb_transnet_l2_normalize_rows(ctx.h, buf.ptr, 37, D, _stream()), "l2")
    got = buf.get("l2")
    _assert_bitwise(got, K.l2_normalize_f32(x), f"l2 D={D}")
    assert (np.abs(got - K.l2_normalize_ref(x)) <= (2 * D + 8) * K.U * np.abs(K.l2_normalize_ref(x)) + 1e-45).all()


@pytest.mark.parametrize("D,T", [(128, 1), (128, 7), (128, 100), (512, 9), (512, 100), (64, 51)])
def test_window_similarity_fc_bitwise_and_isolated(ctx, D, T):  # noqa: F811
    rng = np.random.default_rng(D * 1000 + T)
    B = 3
    x = K.l2_normalize_f32(rng.standard_normal((B * T, D)).astype(F32))
    wt = (rng.standard_normal((101, 128)) / 10).astype(F32)
    bias = (rng.standard_normal(128) * 0.05).astype(F32)

    def run(xx):
        rows = xx.shape[0]
        out = Out(rows, 300, (np.arange(300) >= 136) & (np.arange(300) < 264))
        _ok(ctx, ctx.lib.cb_transnet_window_similarity_fc(ctx.h, _in(xx).data_ptr(), rows, D, T, _in(wt).data_ptr(), _in(bias).data_ptr(), out.ptr, 300, 136,
                                                         _stream()), "simfc")  # fmt: skip
        return out.get("simfc", nan_ok=np.isnan(xx).any())[:, 136:264]

    got = run(x)
    sel = np.unique(np.r_[0, T - 1, T, 2 * T - 1, B * T - 1, np.random.default_rng(T).integers(0, B * T, 12)])
    _assert_bitwise(got[sel], K.window_similarity_fc_f32(x, T, wt, bias, sel), f"simfc D={D} T={T}")
    ref, terms = K.window_similarity_fc_ref(x, T, wt, bias)
    assert (np.abs(got - ref) <= K.window_similarity_fc_bound(terms, D, ref, bias)).all()
    poisoned = x.copy()
    poisoned[:T] = np.nan
    _assert_bitwise(run(poisoned)[T:], run(x[T:]), "clean windows next to a NaN one")


@pytest.mark.parametrize("rows", [1, 4, 5, 127, 400])
def test_head_matches_an_expf_candidate(ctx, rows, record):  # noqa: F811
    rng = np.random.default_rng(rows)
    h = np.maximum(rng.standard_normal((rows, 1024)), 0).astype(F32)
    w = (rng.standard_normal(1024) * 0.06).astype(F32)
    b = F32(-4.75 + rng.standard_normal() * 0.1)
    out = Out(rows, 1)
    _ok(ctx, ctx.lib.cb_transnet_head(ctx.h, _in(h).data_ptr(), _in(w).data_ptr(), float(b), rows, 1, out.ptr, 0, 0, 0, _stream()), "head")
    got = out.get("head")[:, 0]
    off = K.head_match(got, K.head_candidates(h, w, b))
    assert (off != 99).all(), f"rows {np.flatnonzero(off == 99)[:5].tolist()} match no expf candidate"
    record["expf"].update(off.tolist())
    # stitch mode: windows w0.. of T frames into prob[50 w + t - 25] below n_total, nothing else written
    for T, w0, n_total in ((100, 3, 10_000), (100, 0, 160), (60, 2, 131), (26, 1, 52)):
        B = max(1, rows // T)
        hh = np.maximum(rng.standard_normal((B * T, 1024)), 0).astype(F32)
        tgt = K.stitch_targets(B, T, w0, n_total)
        n_out = 50 * (w0 + B) + 50
        mask = np.zeros(n_out, bool)
        mask[list(tgt.values())] = True
        o = Out(1, n_out, mask)
        _ok(ctx, ctx.lib.cb_transnet_head(ctx.h, _in(hh).data_ptr(), _in(w).data_ptr(), float(b), B * T, T, o.ptr, 1, w0, n_total, _stream()), "stitch")
        g = o.get("stitch")[0]
        plain = Out(B * T, 1)
        _ok(ctx, ctx.lib.cb_transnet_head(ctx.h, _in(hh).data_ptr(), _in(w).data_ptr(), float(b), B * T, T, plain.ptr, 0, 0, 0, _stream()), "plain")
        pv = plain.get("plain")[:, 0]
        src = np.array(list(tgt.keys()), np.int64)
        _assert_bitwise(g[list(tgt.values())], pv[src], f"stitch T={T} w0={w0} n={n_total}")


# ------------------------------------------------------------------------------------------------ network replay and stitching
@pytest.fixture(scope="module")
def net(ctx):  # noqa: F811
    from cosmos_curate_b200.runtime import ShotNet

    sd = tn.random_state_dict(7)
    n = ShotNet(ctx, sd, max_windows=MAX_WINDOWS)
    n.sd = sd
    yield n
    n.close()


def _replay(ctx, packed: dict, frames: np.ndarray, B: int, T: int, first, pad) -> np.ndarray:  # noqa: F811
    """run_windows' schedule through the C entry points, with oracle.transnet_kernels.pack's weights."""
    fr = B * T
    bufs = {k: torch.full((v,), float("nan"), dtype=torch.float32, device="cuda") for k, v in K.workspace_floats(fr).items()}
    bufs["prob"] = torch.full((fr,), float("nan"), dtype=torch.float32, device="cuda")
    W = {k: torch.from_numpy(np.ascontiguousarray(v).reshape(-1)).cuda() for k, v in packed.items()}
    ptr = lambda name, off=0: bufs[name].data_ptr() + 4 * off  # noqa: E731
    lib, st = ctx.lib, _stream()
    dev_frames = torch.from_numpy(frames).cuda()
    fi, pa = torch.tensor(first, dtype=torch.int32, device="cuda"), torch.tensor(pad, dtype=torch.int32, device="cuda")
    for L in K.schedule(B, T):
        k = L["kind"]
        if k == "gather":
            rc = lib.cb_transnet_window_gather(ctx.h, dev_frames.data_ptr(), fi.data_ptr(), pa.data_ptr(), B, T, ptr("x0"), ptr("hist"), st)
        elif k == "conv":
            args = _conv_args(L, ptr(L["inp"], L["in_off"]), W[L["w"]].data_ptr(), ptr(L["out"], L["out_off"]),
                              W[L["scale"]].data_ptr() if L["scale"] else None, W[L["shift"]].data_ptr() if L["shift"] else None)  # fmt: skip
            rc = lib.cb_transnet_conv(ctx.h, C.byref(args), L["z"], st)
        elif k == "pool":
            rc = lib.cb_transnet_shortcut_pool(ctx.h, ptr(L["x2"]), ptr(L["x1"]), ptr(L["out"], L["out_off"]), L["frames"], L["H"], L["W"], L["C"],
                                               L["out_frame_stride"], st)  # fmt: skip
        elif k == "mean":
            rc = lib.cb_transnet_spatial_mean(ctx.h, ptr(L["x"], L["x_off"]), L["frame_stride"], L["frames"], L["npos"], L["C"], ptr(L["feats"]),
                                              L["feats_ld"], L["coff"], st)  # fmt: skip
        elif k == "l2":
            rc = lib.cb_transnet_l2_normalize_rows(ctx.h, ptr(L["x"]), L["rows"], L["D"], st)
        elif k == "simfc":
            rc = lib.cb_transnet_window_similarity_fc(ctx.h, ptr(L["x"]), L["rows"], L["D"], L["T"], W[L["wt"]].data_ptr(), W[L["bias"]].data_ptr(),
                                                      ptr(L["out"]), L["out_ld"], L["out_coff"], st)  # fmt: skip
        else:
            rc = lib.cb_transnet_head(ctx.h, ptr("fc1"), W["cls_w"].data_ptr(), float(packed["cls_b"][0]), L["rows"], L["T"], ptr("prob"), 0, 0, 0, st)
        _ok(ctx, rc, f"replay {k} {L.get('name', '')}")
    torch.cuda.synchronize()
    return bufs["prob"].cpu().numpy()


@pytest.mark.parametrize("B", [1, MAX_WINDOWS])
@pytest.mark.parametrize("T", [1, 7, 45, 100])
def test_forward_equals_a_replay_of_its_schedule(ctx, net, B, T):  # noqa: F811
    video = tn.synthetic_frames(B * T, seed=B * 100 + T, cuts=(T // 2,))
    got = net.forward(torch.from_numpy(video.reshape(B, T, 27, 48, 3)).cuda()).cpu().numpy().reshape(-1)
    want = _replay(ctx, K.pack(net.sd), video, B, T, [b * T for b in range(B)], [0] * B)
    _assert_bitwise(got, want, f"forward B={B} T={T} vs replay")


def _predict_raw(ctx, net, frames: np.ndarray) -> np.ndarray:  # noqa: F811
    n = len(frames)
    out = Out(1, n)
    _ok(ctx, ctx.lib.cb_transnet_predict(net.h, _in(frames).data_ptr(), n, out.ptr, _stream()), "predict")
    return out.get("predict")[0]


STITCH_N = [1, 24, 25, 26, 49, 50, 51, 74, 75, 76, 99, 100, 101, 150, 151] + [50 * (k * MAX_WINDOWS + d) - 10 for k in (1, 2) for d in (-1, 0, 1)]


@pytest.mark.parametrize("n", STITCH_N)
def test_predict_stitching_equals_forward_on_each_window_alone(ctx, net, n):  # noqa: F811
    video = tn.synthetic_frames(n, seed=n, cuts=(n // 3,))
    got = _predict_raw(ctx, net, video)
    wins = tn.windows(video)
    assert len(wins) == len(tn.window_plan(n))
    for i, w in enumerate(wins):
        p = net.forward(torch.from_numpy(w).cuda()[None]).cpu().numpy()[0, :, 0]
        j = np.arange(50 * i, min(50 * i + 50, n))
        _assert_bitwise(got[j], p[j - 50 * i + 25], f"n={n} window {i}")


# ------------------------------------------------------------------------------------------------ argument checks
def test_argument_errors_return_their_code_before_any_launch(ctx):  # noqa: F811
    lib = ctx.lib
    p = K.ConvPoint(16, 32, 64, 2, T=4, H=2, W=2, z=4, epi="scale")
    a = p.args()
    inp, w, sc, sh, _ = K.conv_inputs("random", p, a, np.random.default_rng(0))
    x, wd, sd, hd = _in(inp.reshape(p.M, -1)), _in(w), _in(sc), _in(sh)
    out = Out(p.M, a["out_ld"], _out_mask(a))
    n0 = ctx.launch_count()

    def conv(z=4, **kw):
        d = dict(a, **{k: v for k, v in kw.items() if k in a})
        args = _conv_args(d, kw.get("inp", x.data_ptr()), kw.get("w", wd.data_ptr()), kw.get("out", out.ptr), kw.get("scale", sd.data_ptr()),
                          kw.get("shift", hd.data_ptr()))  # fmt: skip
        return lib.cb_transnet_conv(ctx.h, C.byref(args), z, _stream())

    cases = {"null in": conv(inp=None), "null w": conv(w=None), "null out": conv(out=None), "in +4 bytes": conv(inp=x.data_ptr() + 4),
             "out +8 bytes": conv(out=out.ptr + 8), "w +4 bytes": conv(w=wd.data_ptr() + 4), "scale +2 bytes": conv(scale=sd.data_ptr() + 2),
             "in_ld 2 mod 4": conv(in_ld=a["in_ld"] + 2), "in_coff 1": conv(in_coff=1), "out_ld 6 mod 4": conv(out_ld=a["out_ld"] + 2),
             "out_coff 2": conv(out_coff=2), "w_ld 2 mod 4": conv(w_ld=a["w_ld"] + 2), "z_in_coff 2 mod 4": conv(z_in_coff=a["z_in_coff"] + 2),
             "z_out_coff 2 mod 4": conv(z_out_coff=a["z_out_coff"] + 2), "z_w 2 mod 4": conv(z_w=a["z_w"] + 2), "mode 3": conv(mode=3),
             "mode -1": conv(mode=-1), "z 0": conv(z=0), "z 65536": conv(z=65536), "M not whole windows": conv(M=p.M - 4),
             "M not whole frames (mode 1)": conv(mode=1, M=p.M - 1), "M < 0": conv(M=-4), "T 0": conv(T=0), "H 0": conv(H=0),
             "cin 0": conv(cin=0)}  # fmt: skip
    for what, rc in cases.items():
        assert rc == CB_ERR_ARG, (what, rc)
    for what, rc in {"N 30": conv(N=30), "cin 8 N 64": conv(cin=8, N=64), "cin 6 N 128": conv(cin=6, N=128, mode=0)}.items():
        assert rc == CB_ERR_UNSUPPORTED, (what, rc)
    assert conv(M=0) == 0
    f = _in(np.zeros((4, 27, 48, 3), np.uint8))
    i32 = _in(np.zeros(4, np.int32))
    big = Out(8, 4096)
    row = {"gather null": lib.cb_transnet_window_gather(ctx.h, None, i32.data_ptr(), i32.data_ptr(), 1, 1, big.ptr, big.ptr, _stream()),
           "gather x0 +4": lib.cb_transnet_window_gather(ctx.h, f.data_ptr(), i32.data_ptr(), i32.data_ptr(), 1, 1, big.ptr + 4, big.ptr, _stream()),
           "gather B<0": lib.cb_transnet_window_gather(ctx.h, f.data_ptr(), i32.data_ptr(), i32.data_ptr(), -1, 1, big.ptr, big.ptr, _stream()),
           "pool C 6": lib.cb_transnet_shortcut_pool(ctx.h, big.ptr, big.ptr, big.ptr, 1, 2, 2, 6, 8, _stream()),
           "pool stride 6": lib.cb_transnet_shortcut_pool(ctx.h, big.ptr, big.ptr, big.ptr, 1, 2, 2, 4, 6, _stream()),
           "pool out +4": lib.cb_transnet_shortcut_pool(ctx.h, big.ptr, big.ptr, big.ptr + 4, 1, 2, 2, 4, 8, _stream()),
           "pool null": lib.cb_transnet_shortcut_pool(ctx.h, None, big.ptr, big.ptr, 1, 2, 2, 4, 8, _stream()),
           "mean npos 0": lib.cb_transnet_spatial_mean(ctx.h, big.ptr, 8, 1, 0, 4, big.ptr, 4, 0, _stream()),
           "mean null": lib.cb_transnet_spatial_mean(ctx.h, big.ptr, 8, 1, 1, 4, None, 4, 0, _stream()),
           "l2 D 0": lib.cb_transnet_l2_normalize_rows(ctx.h, big.ptr, 1, 0, _stream()),
           "l2 null": lib.cb_transnet_l2_normalize_rows(ctx.h, None, 1, 4, _stream()),
           "simfc rows % T": lib.cb_transnet_window_similarity_fc(ctx.h, big.ptr, 5, 4, 2, big.ptr, big.ptr, big.ptr, 128, 0, _stream()),
           "simfc null": lib.cb_transnet_window_similarity_fc(ctx.h, big.ptr, 4, 4, 2, None, big.ptr, big.ptr, 128, 0, _stream()),
           "head stitch 2": lib.cb_transnet_head(ctx.h, big.ptr, big.ptr, 0.0, 1, 1, big.ptr, 2, 0, 0, _stream()),
           "head T 0": lib.cb_transnet_head(ctx.h, big.ptr, big.ptr, 0.0, 1, 0, big.ptr, 0, 0, 0, _stream()),
           "head null": lib.cb_transnet_head(ctx.h, None, big.ptr, 0.0, 1, 1, big.ptr, 0, 0, 0, _stream())}  # fmt: skip
    for what, rc in row.items():
        assert rc == CB_ERR_ARG, (what, rc)
    assert lib.cb_transnet_window_similarity_fc(ctx.h, big.ptr, 2, 12300, 2, big.ptr, big.ptr, big.ptr, 128, 0, _stream()) == CB_ERR_UNSUPPORTED
    assert lib.cb_transnet_conv(ctx.h, None, 1, _stream()) == CB_ERR_ARG
    for zero in (lib.cb_transnet_l2_normalize_rows(ctx.h, big.ptr, 0, 4, _stream()), lib.cb_transnet_head(ctx.h, big.ptr, big.ptr, 0.0, 0, 1, big.ptr, 0, 0, 0, _stream()),
                 lib.cb_transnet_window_gather(ctx.h, f.data_ptr(), i32.data_ptr(), i32.data_ptr(), 0, 5, big.ptr, big.ptr, _stream())):  # fmt: skip
        assert zero == 0
    assert ctx.launch_count() == n0, "a refused or empty call launched"
    out.untouched("conv (refused calls)")
    big.untouched("row kernels (refused calls)")
    # repeat launches are bitwise equal
    r1 = _conv(ctx, a, inp, w, sc, sh)
    r2 = _conv(ctx, a, inp, w, sc, sh)
    assert np.array_equal(_bits(_pick(r1, a, np.arange(p.M))), _bits(_pick(r2, a, np.arange(p.M))))
