"""The tower's row kernels (csrc/vit_kernels.cu) through the C ABI, against oracle/rowops.py, at every dispatch and row boundary.

* rsqrtf class (LayerNorm, LayerNorm-post, RMSNorm, qk-RMSNorm, CLIP assemble, clip_tail): one of the <= 5 fp32 rstd candidates per
  row reproduces the whole row bit for bit; the histogram of the candidates used is printed when the module ends;
* exact (SigLIP and InternVideo2 assemble, l2norm_score, affine_score, token_mean, tube_patches; the pools on uniform and one-hot inputs): bit for bit;
* bounded (the pools on random inputs): within oracle.rowops.pool_bound, the worst err/bound printed when the module ends;
* every call reads its inputs with NaN rows after them and writes into a NaN-filled buffer with guard rows: nothing outside the
  output may change and no NaN may reach it;
* repeat launches are bitwise equal; every argument error returns its code before anything is launched.
"""

from __future__ import annotations

import zlib
from collections import Counter

import numpy as np
import pytest
import torch

from gpu_helpers import ctx  # noqa: F401
from oracle import rowops as R

pytestmark = pytest.mark.gpu

F32, F16 = np.float32, np.float16
PAD = 3  # NaN rows after every input, NaN guard rows before and after every output
SM_REF = 132  # the sweep's names use this SM count's rows; the rows themselves come from the device


def _stream():
    from cosmos_curate_b200.runtime import _stream_ptr

    return _stream_ptr()


def _sm(ctx) -> int:
    return ctx.device_info()["sm_count"]


def _seed(name: str) -> int:
    return zlib.crc32(name.encode())


_LIVE: list[torch.Tensor] = []  # inputs whose raw pointers were handed to the library: alive until the test ends


@pytest.fixture(autouse=True)
def _inputs_live_until_the_test_ends():
    yield
    torch.cuda.synchronize()
    _LIVE.clear()


def _in(a: np.ndarray) -> torch.Tensor:
    """a on the device as the first rows of a buffer whose PAD rows after it are NaN.  The buffer is kept alive until the test ends:
    the calls pass `_in(x).data_ptr()`, and a buffer freed there would go back to torch's allocator while the kernel reads it."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    rows = t.shape[0] if t.dim() else 1
    buf = torch.full((rows + PAD, *t.shape[1:]), float("nan"), dtype=t.dtype, device="cuda")
    buf[:rows] = t.cuda().reshape(rows, *t.shape[1:])
    _LIVE.append(buf)
    return buf[:rows] if t.dim() else buf[0]


class Out:
    """A NaN-filled output [rows][...] with PAD guard rows before and after."""

    def __init__(self, shape, dtype, fill: torch.Tensor | None = None):
        self.buf = torch.full((shape[0] + 2 * PAD, *shape[1:]), float("nan"), dtype=dtype, device="cuda")
        self.t = self.buf[PAD : PAD + shape[0]]
        if fill is not None:
            self.t.copy_(fill)
        self.before = self.buf.clone()

    @property
    def ptr(self) -> int:
        return self.t.data_ptr()

    def get(self, what: str) -> np.ndarray:
        torch.cuda.synchronize()
        b, a = _bits(self.buf.cpu().numpy()), _bits(self.before.cpu().numpy())
        assert np.array_equal(b[:PAD], a[:PAD]), f"{what}: rows before the output were written"
        assert np.array_equal(b[PAD + self.t.shape[0] :], a[PAD + self.t.shape[0] :]), f"{what}: rows after the output were written"
        out = self.t.cpu().numpy()
        assert not np.isnan(out).any(), f"{what}: NaN in the output at {np.argwhere(np.isnan(out))[0].tolist()}"
        return out


def _bits(a: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(a).view({2: np.int16, 4: np.int32}[a.dtype.itemsize])


def _ok(ctx, rc: int, what: str) -> None:
    from cosmos_curate_b200.runtime import check

    check(rc, what, ctx.h)


def _assert_bitwise(got: np.ndarray, want: np.ndarray, what: str) -> None:
    bad = np.argwhere(_bits(got) != _bits(want))
    if len(bad):
        i = tuple(bad[0])
        pytest.fail(f"{what}: {len(bad)} of {got.size} elements differ; first at {list(i)}: got {got[i]!r} want {want[i]!r}")


@pytest.fixture(scope="module")
def record(pytestconfig):
    """rstd candidate histogram and worst pool err/bound, written to the terminal (past output capture) when the module ends."""
    r = {"hist": Counter(), "worst": {}}
    yield r
    total = sum(r["hist"].values())
    lines = ["rsqrtf candidate per row (ulps from the correctly rounded rsqrt): "
             + ", ".join(f"{k:+d}: {r['hist'][k]}" for k in range(-R.RSQRT_ULP, R.RSQRT_ULP + 1)) + f" (rows {total})"]  # fmt: skip
    lines += [f"pool {name}: worst err/bound {w:.3f}" for name, w in sorted(r["worst"].items())]
    capman = pytestconfig.pluginmanager.get_plugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print("\n" + "\n".join(lines))


def _accept(record, got: np.ndarray, arg: np.ndarray, apply, what: str) -> None:
    off, best = R.match_rows(got, arg, apply)
    bad = np.flatnonzero(off == 99)
    if len(bad):
        i = bad[0]
        pytest.fail(f"{what}: {len(bad)} of {len(off)} rows match no rsqrtf candidate within {R.RSQRT_ULP} ulp; first row {i}, "
                    f"{best[i]} elements differ for its best candidate")  # fmt: skip
    record["hist"].update(off.tolist())


# ------------------------------------------------------------------------------------------------ norms
def _norm_rows(rows: int, d: int, seed: int) -> np.ndarray:
    """Row classes by index mod 5: random, mean >> sigma, constant (dyadic: the mean is exact), around 1e-20, large (~1e4)."""
    r = np.random.default_rng(seed)
    x = (r.standard_normal((rows, d)) * 3 + 1).astype(F32)
    i = np.arange(rows)
    x[i % 5 == 1] = (1e3 + r.standard_normal((int((i % 5 == 1).sum()), d))).astype(F32)
    x[i % 5 == 2] = ((i[i % 5 == 2] % 7 - 3) * 0.375).astype(F32)[:, None]
    x[i % 5 == 3] = (r.standard_normal((int((i % 5 == 3).sum()), d)) * 1e-20).astype(F32)
    x[i % 5 == 4] = (r.standard_normal((int((i % 5 == 4).sum()), d)) * 1e4).astype(F32)
    return x


NORM_CASES = [(p.kernel, p.d, R.rows_classes(SM_REF).index(p.rows)) for k in R.NORMS for p in R.norm_sweep(k, SM_REF)]
NORM_CASES += [(k, d, -1) for k in R.NORMS for d in (768, 1024, 1408)]  # rc -1: 9 rows, gamma ~1e4 - outputs near the fp16 range


@pytest.mark.parametrize(("kernel", "d", "rc"), NORM_CASES, ids=[f"{k}-d{d}-rc{rc}" for k, d, rc in NORM_CASES])
def test_norm_exact(ctx, record, kernel, d, rc):
    rows = 9 if rc < 0 else R.rows_classes(_sm(ctx))[rc]
    name = f"{kernel}-d{d}-rc{rc}"
    what = f"{R.instantiation(kernel, d)} at d={d}, rows={rows}"
    r = np.random.default_rng(_seed(name))
    x = _norm_rows(rows, d, _seed(name) + 1)
    gamma = (r.random(d) * 1.45 + 0.05).astype(F32) * F32(8e3 if rc < 0 else 1)
    beta = r.standard_normal(d).astype(F32)
    eps = 1e-5 if kernel.startswith("layernorm") else 1e-6
    const = (np.arange(rows) % 5 == 2)[:, None]
    if kernel == "layernorm":
        y = Out((rows, d), torch.float16)
        _ok(ctx, ctx.lib.cb_layernorm_f16(ctx.h, _in(x).data_ptr(), _in(gamma).data_ptr(), _in(beta).data_ptr(), y.ptr, rows, d, eps, _stream()), what)
        got = y.get(what)
        mean, arg = R.ln_stats(x, eps)
        _accept(record, got, arg, lambda rs: R.ln_apply(x, mean, rs, gamma, beta).astype(F16), what)
        _assert_bitwise(np.where(const, got, F16(0)), np.where(const, beta.astype(F16)[None], F16(0)), f"{what}: constant rows -> beta")
    elif kernel == "layernorm_post":
        h = Out((rows, d), torch.float32, torch.from_numpy(x).cuda())
        y = Out((rows, d), torch.float16)
        _ok(ctx, ctx.lib.cb_layernorm_post_f16(ctx.h, h.ptr, _in(gamma).data_ptr(), _in(beta).data_ptr(), y.ptr, rows, d, eps, _stream()), what)
        got32, got16 = h.get(what), y.get(what)
        mean, arg = R.ln_stats(x, eps)
        _accept(record, got32, arg, lambda rs: R.ln_apply(x, mean, rs, gamma, beta), what)
        _assert_bitwise(got16, got32.astype(F16), f"{what}: the fp16 copy is the fp32 result rounded")
        _assert_bitwise(np.where(const, got32, F32(0)), np.where(const, beta[None], F32(0)), f"{what}: constant rows -> beta")
    elif kernel == "rmsnorm":
        y = Out((rows, d), torch.float16)
        _ok(ctx, ctx.lib.cb_rmsnorm_f16(ctx.h, _in(x).data_ptr(), _in(gamma).data_ptr(), y.ptr, rows, d, eps, _stream()), what)
        got = y.get(what)
        _accept(record, got, R.rms_stats(x, eps), lambda rs: R.rms_apply(x, rs, gamma).astype(F16), what)
    else:  # qk_rmsnorm: q and k thirds of fp16 qkv rows in place, v third untouched
        qkv = np.concatenate([x.astype(F16), _norm_rows(rows, d, _seed(name) + 2).astype(F16), r.standard_normal((rows, d)).astype(F16)], 1)
        wk = (r.random(d) + 0.5).astype(F32)
        buf = Out((rows, 3 * d), torch.float16, torch.from_numpy(qkv).cuda())
        _ok(ctx, ctx.lib.cb_qk_rmsnorm_f16(ctx.h, buf.ptr, _in(gamma).data_ptr(), _in(wk).data_ptr(), rows, d, eps, _stream()), what)
        got = buf.get(what)
        for part, w in ((0, gamma), (1, wk)):
            xp = qkv[:, part * d : (part + 1) * d].astype(F32)
            _accept(record, got[:, part * d : (part + 1) * d], R.rms_stats(xp, eps), lambda rs: R.rms_apply(xp, rs, w).astype(F16),  # noqa: B023
                    f"{what}, {'qk'[part]} third")  # fmt: skip
        _assert_bitwise(got[:, 2 * d :], qkv[:, 2 * d :], f"{what}: the v third")


# ------------------------------------------------------------------------------------------------ assemble
# clip: [CLS] + pre-LN; siglip: no [CLS], no norm; iv2 (InternVideo2): [CLS], no norm
ASSEMBLE_CASES = [(arch, n, g, d) for arch in ("clip", "siglip", "iv2") for n, g, d in ((1, 7, 128), (3, 7, 768), (2, 16, 1024), (5, 3, 1152),
                                                                                          (1, 2, 1536))]  # fmt: skip


@pytest.mark.parametrize(("arch", "n", "g", "d"), ASSEMBLE_CASES, ids=[f"{a}-n{n}-g{g}-d{d}" for a, n, g, d in ASSEMBLE_CASES])
def test_assemble(ctx, record, arch, n, g, d):
    what = f"assemble {arch} n={n} grid={g}x{g} d={d}"
    r = np.random.default_rng(_seed(what))
    g2 = g * g
    tokens = g2 + (arch != "siglip")
    patch = (r.standard_normal((n * g2, d)) * 2).astype(F32)
    cls = r.standard_normal(d).astype(F32)
    pos = r.standard_normal((tokens, d)).astype(F32)
    gamma = (r.random(d) + 0.5).astype(F32) if arch == "clip" else None
    beta = r.standard_normal(d).astype(F32) if arch == "clip" else None
    h = Out((n * tokens, d), torch.float32)
    dp = lambda a: _in(a).data_ptr() if a is not None else None  # noqa: E731
    _ok(ctx, ctx.lib.cb_assemble_tokens(ctx.h, dp(patch), dp(cls) if arch != "siglip" else None, dp(pos), dp(gamma), dp(beta), h.ptr, n, tokens, g2,
                                        d, 1e-5, _stream()), what)  # fmt: skip
    got = h.get(what)
    summed, stats = R.assemble_f32(patch, cls, pos, gamma, beta, None, 1e-5, n, tokens, g2)
    if arch != "clip":
        _assert_bitwise(got, summed, what)
    else:
        mean, arg = stats
        _accept(record, got, arg, lambda rs: R.ln_apply(summed, mean, rs, gamma, beta), what)


# ------------------------------------------------------------------------------------------------ CLIP tail
TAIL_CASES = [(d, pd, feat, aes, stride) for d, pd in ((256, 128), (768, 512), (1024, 768), (1024, 0)) for feat, aes in ((True, True), (False, False))
              for stride in ("T*d", "d")]  # fmt: skip


@pytest.mark.parametrize(("d", "proj_dim", "feat", "aes", "stride"), TAIL_CASES,
                         ids=[f"d{d}-p{p}-{'feat' if f else 'nofeat'}-{'aes' if a else 'noaes'}-{s}" for d, p, f, a, s in TAIL_CASES])  # fmt: skip
def test_clip_tail(ctx, record, d, proj_dim, feat, aes, stride):
    what = f"clip_tail d={d} proj_dim={proj_dim} feat={feat} aes={aes} img_stride={stride}"
    r = np.random.default_rng(_seed(what))
    n, T = 9, 50
    h = (r.standard_normal((n, T if stride == "T*d" else 1, d)) * 2 + 0.5).astype(F32)
    x = np.ascontiguousarray(h[:, 0])
    gamma, beta = (r.random(d) + 0.5).astype(F32), (r.standard_normal(d) * 0.1).astype(F32)
    proj = (r.standard_normal((proj_dim, d)) * d**-0.5).astype(F32) if proj_dim else None
    out_dim = proj_dim or d
    aes_w = r.standard_normal(out_dim).astype(F32) if aes else None
    aes_b = 0.375
    emb, fo = Out((n, out_dim), torch.float32), Out((n, out_dim), torch.float32) if feat else None
    score = Out((n,), torch.float32) if aes else None
    dp = lambda a: _in(a).data_ptr() if a is not None else None  # noqa: E731
    _ok(ctx, ctx.lib.cb_clip_tail(ctx.h, dp(h.reshape(n * h.shape[1], d)), h.shape[1] * d, dp(gamma), dp(beta), dp(proj), d, proj_dim, 1e-5,
                                  dp(aes_w), aes_b, emb.ptr, fo.ptr if feat else None, score.ptr if aes else None, n, _stream()), what)  # fmt: skip
    got = [emb.get(what)] + ([fo.get(what)] if feat else []) + ([score.get(what)[:, None]] if aes else [])
    mean, arg = R.clip_tail_stats(x, 1e-5)

    def model(rs):
        e, f, s = R.clip_tail_f32(x, mean, rs, gamma, beta, proj, aes_w, aes_b)
        return np.concatenate([e] + ([f] if feat else []) + ([s[:, None]] if aes else []), 1)

    _accept(record, np.concatenate(got, 1), arg, model, what)
    e64, _, s64 = R.clip_tail_ref(x, gamma, beta, 1e-5, proj, aes_w, aes_b)
    assert np.abs(got[0] - e64).max() < 1e-5, what  # the model itself is the operation


# ------------------------------------------------------------------------------------------------ exact-class kernels
@pytest.mark.parametrize(("n", "d"), [(1, 32), (9, 128), (1057, 512), (7, 1152), (8, 1536)])
def test_l2norm_score_exact(ctx, n, d):
    what = f"l2norm_score n={n} d={d}"
    r = np.random.default_rng(_seed(what))
    feat = (r.standard_normal((n, d)) * 3).astype(F32)
    w = r.standard_normal(d).astype(F32)
    for aes in (False, True):
        emb, fo, sc = Out((n, d), torch.float32), Out((n, d), torch.float32), Out((n,), torch.float32)
        _ok(ctx, ctx.lib.cb_l2norm_score(ctx.h, _in(feat).data_ptr(), d, _in(w).data_ptr() if aes else None, -0.25, emb.ptr, fo.ptr,
                                         sc.ptr if aes else None, n, _stream()), what)  # fmt: skip
        we, ws = R.l2norm_score_f32(feat, w if aes else None, -0.25)
        _assert_bitwise(emb.get(what), we, f"{what} emb")
        _assert_bitwise(fo.get(what), feat, f"{what} feat")
        if aes:
            _assert_bitwise(sc.get(what), ws, f"{what} score")


@pytest.mark.parametrize(("n", "d"), [(1, 512), (9, 768), (1057, 1152)])
def test_affine_score_exact(ctx, n, d):
    what = f"affine_score n={n} d={d}"
    r = np.random.default_rng(_seed(what))
    emb, w = r.standard_normal((n, d)).astype(F32), r.standard_normal(d).astype(F32)
    out = Out((n,), torch.float32)
    _ok(ctx, ctx.lib.cb_affine_score(ctx.h, _in(emb).data_ptr(), _in(w).data_ptr(), 0.125, out.ptr, n, d, _stream()), what)
    _assert_bitwise(out.get(what), R.affine_score_f32(emb, w, 0.125), what)


@pytest.mark.parametrize("tokens", R.TOKENS)
def test_token_mean_exact(ctx, tokens):
    for n, d in ((3, 1408), (1, 128)):
        what = f"token_mean n={n} tokens={tokens} d={d}"
        h = np.random.default_rng(_seed(what)).standard_normal((n, tokens, d)).astype(F32)
        out = Out((n, d), torch.float32)
        _ok(ctx, ctx.lib.cb_token_mean(ctx.h, _in(h.reshape(n * tokens, d)).data_ptr(), out.ptr, n, tokens, d, _stream()), what)
        _assert_bitwise(out.get(what), R.token_mean_f32(h), what)


@pytest.mark.parametrize(("frames", "s", "p", "k_pad"), [(4, 224, 14, 592), (3, 64, 16, 768), (1, 30, 14, 600), (2, 16, 16, 776)])
def test_tube_patches_exact(ctx, frames, s, p, k_pad):
    what = f"tube_patches frames={frames} S={s} P={p} k_pad={k_pad}"
    tubes = np.random.default_rng(_seed(what)).standard_normal((frames, 3, s, s)).astype(F32)
    g = s // p
    out = Out((frames * g * g, k_pad), torch.float16)
    _ok(ctx, ctx.lib.cb_tube_patches(ctx.h, _in(tubes.reshape(frames * 3, s * s)).data_ptr(), out.ptr, frames, s, p, k_pad, _stream()), what)
    _assert_bitwise(out.get(what), R.tube_patches_f32(tubes, p, k_pad).reshape(frames * g * g, k_pad), what)


# ------------------------------------------------------------------------------------------------ pools
HEADS = 2


def _pool_call(ctx, kind: str, k: np.ndarray, v: np.ndarray, q: np.ndarray, what: str) -> np.ndarray:
    """k, v fp16 [n][T][heads][hd], q fp32 [n][heads][hd] (map: q[0] is the one query, pre-scaled) -> out fp16 [n][heads][hd]."""
    n, t, heads, hd = k.shape
    hidden = heads * hd
    out = Out((n, hidden), torch.float16)
    if kind == "map":
        kv = np.concatenate([k.reshape(n, t, hidden), v.reshape(n, t, hidden)], 2).reshape(n * t, 2 * hidden)
        rc = ctx.lib.cb_map_pool(ctx.h, _in(kv).data_ptr(), _in(q[0].reshape(hidden)).data_ptr(), out.ptr, n, t, heads, hd, _stream())
    else:
        rc = ctx.lib.cb_clip_pool(ctx.h, _in(q.reshape(n, hidden)).data_ptr(), _in(k.reshape(n * t, hidden)).data_ptr(),
                                  _in(v.reshape(n * t, hidden)).data_ptr(), out.ptr, n, t, heads, hd, _stream())  # fmt: skip
    _ok(ctx, rc, what)
    return out.get(what).reshape(n, heads, hd)


def _qh(kind: str, q: np.ndarray, hd: int) -> np.ndarray:
    """The query as the kernel multiplies with it: map_pool's is given pre-scaled, clip_pool scales by 1.0f / sqrtf(hd)."""
    return q if kind == "map" else (q * (F32(1) / np.sqrt(F32(hd)))).astype(F32)


POOL_CASES = [(kind, hd, t) for kind in ("map", "clip") for hd, t in R.pool_sweep(kind)]


@pytest.mark.parametrize(("kind", "hd", "t"), POOL_CASES, ids=[f"{k}-hd{h}-t{t}" for k, h, t in POOL_CASES])
def test_pool(ctx, record, kind, hd, t):
    what = f"{kind}_pool hd={hd} tokens={t}"
    n = 2 if kind == "clip" else 1  # map_pool has one query for every image; n > 1 is exercised by the random class
    seed = _seed(what)
    # uniform: every __expf(0) = 1, V's sums exact
    parts = [R.pool_uniform_inputs(n, t, hd, seed + h) for h in range(HEADS)]
    k, v = (np.stack([p[i] for p in parts], 2) for i in range(2))
    q = np.stack([p[2] for p in parts], 1)
    if kind == "map":
        q[:] = q[:1]
    got = _pool_call(ctx, kind, k, v, q, f"{what}, uniform")
    for h in range(HEADS):
        _assert_bitwise(got[:, h], R.pool_f32(k[:, :, h], v[:, :, h], _qh(kind, q[:, h], hd)), f"{what}, uniform, head {h}")
    # one-hot: the output is V[j], j coded in V's values
    scale = 1.0 if kind == "clip" else hd**-0.5
    parts = [R.pool_onehot_inputs(n, t, hd, seed + 10 + h, scale=1.0) for h in range(HEADS)]
    k, v = (np.stack([p[i] for p in parts], 2) for i in range(2))
    q = np.stack([p[2] for p in parts], 1) * F32(scale)
    if kind == "map":
        q[:] = q[:1]
        for h in range(HEADS):  # one query for every image: recode the winning key of image i > 0 against image 0's query
            k[:, :, h] = 0
            k[np.arange(n), parts[h][3], h] = (32 * np.sign(q[0, h])).astype(F16)
    got = _pool_call(ctx, kind, k, v, q.astype(F32), f"{what}, one-hot")
    for h in range(HEADS):
        _assert_bitwise(got[:, h], v[np.arange(n), parts[h][3], h], f"{what}, one-hot, head {h}")
    # random: within the bound
    r = np.random.default_rng(seed + 99)
    nr = 3
    k = (r.standard_normal((nr, t, HEADS, hd)) * 1.5).astype(F16)
    v = r.standard_normal((nr, t, HEADS, hd)).astype(F16)
    q = (r.standard_normal((nr, HEADS, hd)) * (hd**-0.5 if kind == "map" else 1)).astype(F32)
    if kind == "map":
        q[:] = q[:1]
    got = _pool_call(ctx, kind, k, v, q, f"{what}, random").astype(np.float64)
    worst = 0.0
    for h in range(HEADS):
        qh = _qh(kind, q[:, h], hd)
        ratio = np.abs(got[:, h] - R.pool_ref(k[:, :, h], v[:, :, h], qh)) / R.pool_bound(k[:, :, h], v[:, :, h], qh)
        worst = max(worst, float(ratio.max()))
    key = f"{kind} hd={hd}"
    record["worst"][key] = max(record["worst"].get(key, 0.0), worst)
    assert worst <= 1.0, f"{what}, random: err/bound {worst:.3f}"


# ------------------------------------------------------------------------------------------------ repeat launches
def test_repeat_launches_bitwise_equal(ctx):
    r = np.random.default_rng(7)
    rows, d = 8 * _sm(ctx) + 1, 1024
    x, g, b = _norm_rows(rows, d, 8), (r.random(d) + 0.5).astype(F32), r.standard_normal(d).astype(F32)
    xi, gi, bi = _in(x), _in(g), _in(b)
    t, hd = 1025, 88
    k, v = (r.standard_normal((2 * t, 16 * hd)).astype(F16) for _ in range(2))
    q = r.standard_normal((2, 16 * hd)).astype(F32)
    ki, vi, qi = _in(k), _in(v), _in(q)
    first = None
    for _ in range(3):
        y, p = Out((rows, d), torch.float16), Out((2, 16 * hd), torch.float16)
        _ok(ctx, ctx.lib.cb_layernorm_f16(ctx.h, xi.data_ptr(), gi.data_ptr(), bi.data_ptr(), y.ptr, rows, d, 1e-5, _stream()), "layernorm")
        _ok(ctx, ctx.lib.cb_clip_pool(ctx.h, qi.data_ptr(), ki.data_ptr(), vi.data_ptr(), p.ptr, 2, t, 16, hd, _stream()), "clip_pool")
        now = (y.get("layernorm"), p.get("clip_pool"))
        if first is None:
            first = now
        for a, b_, name in zip(now, first, ("layernorm", "clip_pool")):
            _assert_bitwise(a, b_, f"{name}: a repeat launch")


# ------------------------------------------------------------------------------------------------ argument errors
ARG, UNSUPPORTED = -2, -3
_B = ("a", "b", "c", "d", "e", "f", "g", "h")  # eight 1 MB NaN buffers; an argument "a+4" is buffer a's address plus 4 bytes

_VALID = {  # export -> argument list of a valid call (buffer names, ints, floats)
    "cb_layernorm_f16": ["a", "b", "c", "d", 8, 256, 1e-5],
    "cb_layernorm_post_f16": ["a", "b", "c", "d", 8, 256, 1e-5],
    "cb_assemble_tokens": ["a", "b", "c", "d", "e", "f", 2, 50, 49, 256, 1e-5],
    "cb_clip_tail": ["a", 256, "b", "c", "d", 256, 128, 1e-5, "e", 0.5, "f", "g", "h", 2],
    "cb_map_pool": ["a", "b", "c", 2, 257, 4, 64],
    "cb_l2norm_score": ["a", 256, "b", 0.5, "c", "d", "e", 8],
    "cb_token_mean": ["a", "b", 2, 257, 256],
    "cb_clip_pool": ["a", "b", "c", "d", 2, 257, 4, 64],
    "cb_tube_patches": ["a", "b", 2, 28, 14, 592],
}
_ERRORS = [  # (id, export, {argument index: value}, code)
    ("ln_rows_negative", "cb_layernorm_f16", {4: -1}, ARG),
    ("ln_d_zero", "cb_layernorm_f16", {5: 0}, UNSUPPORTED),
    ("ln_d_not_128k", "cb_layernorm_f16", {5: 200}, UNSUPPORTED),
    ("ln_d_too_wide", "cb_layernorm_f16", {5: 1664}, UNSUPPORTED),
    ("ln_x_misaligned", "cb_layernorm_f16", {0: "a+4"}, ARG),
    ("ln_gamma_misaligned", "cb_layernorm_f16", {1: "b+8"}, ARG),
    ("ln_y_misaligned", "cb_layernorm_f16", {3: "d+4"}, ARG),
    ("ln_null_beta", "cb_layernorm_f16", {2: None}, ARG),
    ("ln_post_h_misaligned", "cb_layernorm_post_f16", {0: "a+4"}, ARG),
    ("asm_null_patch", "cb_assemble_tokens", {0: None}, ARG),
    ("asm_null_cls_with_cls_token", "cb_assemble_tokens", {1: None}, ARG),
    ("asm_gamma_without_beta", "cb_assemble_tokens", {4: None}, ARG),
    ("asm_n_negative", "cb_assemble_tokens", {6: -1}, ARG),
    ("asm_tokens_not_grid2", "cb_assemble_tokens", {7: 52}, ARG),
    ("asm_d_not_128k", "cb_assemble_tokens", {9: 320}, UNSUPPORTED),
    ("asm_d_too_wide", "cb_assemble_tokens", {9: 1664}, UNSUPPORTED),
    ("asm_pos_misaligned", "cb_assemble_tokens", {2: "c+4"}, ARG),
    ("tail_null_h", "cb_clip_tail", {0: None}, ARG),
    ("tail_null_emb", "cb_clip_tail", {10: None}, ARG),
    ("tail_n_negative", "cb_clip_tail", {13: -1}, ARG),
    ("tail_stride_below_d", "cb_clip_tail", {1: 128}, ARG),
    ("tail_proj_dim_zero", "cb_clip_tail", {6: 0}, ARG),
    ("tail_d_not_128k", "cb_clip_tail", {5: 200, 1: 200}, UNSUPPORTED),
    ("tail_proj_misaligned", "cb_clip_tail", {4: "d+4"}, ARG),
    ("tail_smem_too_large", "cb_clip_tail", {6: 12100}, UNSUPPORTED),
    ("map_head_dim_258", "cb_map_pool", {6: 258, 5: 2}, UNSUPPORTED),
    ("map_head_dim_odd", "cb_map_pool", {6: 63}, UNSUPPORTED),
    ("map_kv_misaligned", "cb_map_pool", {0: "a+2"}, ARG),
    ("map_tokens_zero", "cb_map_pool", {4: 0}, ARG),
    ("map_n_negative", "cb_map_pool", {3: -1}, ARG),
    ("map_smem_past_the_device", "cb_map_pool", {4: 1 << 20}, UNSUPPORTED),
    ("l2_null_feat", "cb_l2norm_score", {0: None}, ARG),
    ("l2_n_negative", "cb_l2norm_score", {7: -1}, ARG),
    ("l2_d_zero", "cb_l2norm_score", {1: 0}, UNSUPPORTED),
    ("l2_d_too_wide", "cb_l2norm_score", {1: 1537}, UNSUPPORTED),
    ("l2_emb_misaligned", "cb_l2norm_score", {4: "c+2"}, ARG),
    ("mean_tokens_zero", "cb_token_mean", {3: 0}, ARG),
    ("mean_tokens_negative", "cb_token_mean", {3: -5}, ARG),
    ("mean_n_negative", "cb_token_mean", {2: -1}, ARG),
    ("mean_d_not_128k", "cb_token_mean", {4: 100}, UNSUPPORTED),
    ("mean_null_out", "cb_token_mean", {1: None}, ARG),
    ("pool_head_dim_258", "cb_clip_pool", {7: 258, 6: 2}, UNSUPPORTED),
    ("pool_head_dim_odd", "cb_clip_pool", {7: 87}, UNSUPPORTED),
    ("pool_k_misaligned", "cb_clip_pool", {1: "b+2"}, ARG),
    ("pool_null_v", "cb_clip_pool", {2: None}, ARG),
    ("pool_smem_past_the_device", "cb_clip_pool", {5: 1 << 20}, UNSUPPORTED),
    ("tube_k_pad_odd", "cb_tube_patches", {5: 591}, ARG),
    ("tube_k_pad_short", "cb_tube_patches", {5: 586}, ARG),
    ("tube_image_below_patch", "cb_tube_patches", {3: 12}, ARG),
    ("tube_frames_negative", "cb_tube_patches", {2: -1}, ARG),
    ("tube_out_misaligned", "cb_tube_patches", {1: "b+2"}, ARG),
]
_NOOPS = [("cb_layernorm_f16", {4: 0}), ("cb_assemble_tokens", {6: 0}), ("cb_clip_tail", {13: 0}), ("cb_map_pool", {3: 0}),
          ("cb_l2norm_score", {7: 0}), ("cb_token_mean", {2: 0}), ("cb_clip_pool", {4: 0}), ("cb_tube_patches", {2: 0})]  # fmt: skip


def _call_with(ctx, fn: str, changes: dict) -> int:
    bufs = {b: torch.full((1 << 18,), float("nan"), device="cuda") for b in _B}
    before = {b: t.clone() for b, t in bufs.items()}
    args = list(_VALID[fn])
    for i, val in changes.items():
        args[i] = val

    def conv(a):
        if isinstance(a, str):
            name, _, off = a.partition("+")
            return bufs[name].data_ptr() + int(off or 0)
        return a

    launches = ctx.launch_count()
    rc = getattr(ctx.lib, fn)(ctx.h, *[conv(a) for a in args], _stream())
    torch.cuda.synchronize()
    assert ctx.launch_count() == launches, f"{fn}: a kernel was launched"
    for b, t in bufs.items():
        assert torch.equal(t.view(torch.int32), before[b].view(torch.int32)), f"{fn}: buffer {b} was written"
    return rc


@pytest.mark.parametrize(("fn", "changes", "code"), [e[1:] for e in _ERRORS], ids=[e[0] for e in _ERRORS])
def test_rejected_on_the_host(ctx, fn, changes, code):
    """Each bad argument returns its code before anything is launched (every buffer is 1 MB, so even the mis-sized calls name memory a
    kernel could use without leaving it)."""
    assert _call_with(ctx, fn, changes) == code


@pytest.mark.parametrize(("fn", "changes"), _NOOPS, ids=[f[0] for f in _NOOPS])
def test_n_zero_is_a_no_op(ctx, fn, changes):
    assert _call_with(ctx, fn, changes) == 0



# ------------------------------------------------------------------------------------------------ ViT handle replay
REPLAY_MAX_BATCH = 4


def _replay_cfg(arch: str):
    from oracle import vit

    if arch == "clip":
        return vit.CLIP_TINY  # 2 layers, 7 x 7 patches + [CLS], d 256, projection 128
    return vit.VitConfig(image_size=64, patch=16, hidden=128, layers=2, heads=2, mlp=256, proj_dim=0, act="gelu_tanh", ln_eps=1e-6, arch="siglip")


class _Replay:
    """cb_vit_forward's schedule (csrc/vit.cu forward_chunk) restated through the C ABI on the same fp16 / fp32 weights."""

    def __init__(self, ctx, cfg, w: dict, aes_w: np.ndarray, aes_b: float, k_pad: int):
        self.ctx, self.cfg, self.k_pad, self.aes_b = ctx, cfg, k_pad, aes_b
        self.f = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
        self.h = {k: torch.from_numpy(v).half().cuda() for k, v in w.items() if v.ndim == 2 and k not in ("pos",)}
        pw = torch.zeros(cfg.hidden, k_pad, dtype=torch.float16)
        pw[:, : w["patch_w"].shape[1]] = torch.from_numpy(w["patch_w"]).half()
        self.h["patch_w"] = pw.cuda()
        self.aes_w = torch.from_numpy(aes_w).cuda()
        if cfg.arch == "siglip":  # the pooling query, folded as cb_vit_finalize folds it: float64, inputs in order, then * hd^-1/2
            d, hd = cfg.hidden, cfg.hidden // cfg.heads
            terms = w["map_in_w"][:d].astype(np.float64) * w["map_probe"].astype(np.float64)[None]
            acc = np.cumsum(np.concatenate([w["map_in_b"][:d, None].astype(np.float64), terms], 1), axis=1)[:, -1]
            self.map_q = torch.from_numpy((acc * (1.0 / np.sqrt(float(hd)))).astype(F32)).cuda()

    def gemm(self, a, w, bias, out_f32=None, residual=None, epi=0, n_out=None):
        m, k = a.shape
        n = w.shape[0]
        o16 = None if out_f32 is not None else torch.empty(m, n, dtype=torch.float16, device="cuda")
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        _ok(self.ctx, self.ctx.lib.cb_gemm_f16_ex(self.ctx.h, a.data_ptr(), w.data_ptr(), ptr(bias), None, ptr(residual), ptr(out_f32), ptr(o16), m, n,
                                                  k, epi, _stream()), "replay gemm")  # fmt: skip
        return out_f32 if out_f32 is not None else o16

    def ln(self, x, g, b):
        y = torch.empty(x.shape, dtype=torch.float16, device="cuda")
        _ok(self.ctx, self.ctx.lib.cb_layernorm_f16(self.ctx.h, x.data_ptr(), g.data_ptr(), b.data_ptr(), y.data_ptr(), x.shape[0], x.shape[1],
                                                    self.cfg.ln_eps, _stream()), "replay layernorm")  # fmt: skip
        return y

    def chunk(self, patches, gather: str):
        """One chunk of images; gather "cls" is the current schedule ([CLS] rows gathered after the last attention), "none" the one
        before it (every row through the last layer, then the tail reads token 0 of each image at img_stride = T d)."""
        c, ctx, f, h = self.cfg, self.ctx, self.f, self.h
        lib = ctx.lib
        n, d, T, g2 = patches.shape[0], c.hidden, c.tokens, c.grid**2
        rows, hd = n * T, c.hidden // c.heads
        act = 1 if c.act == "quick_gelu" else 2
        patch_out = torch.empty(n * g2, d, device="cuda")
        self.gemm(patches.reshape(n * g2, self.k_pad), h["patch_w"], f.get("patch_b") if c.arch == "siglip" else None, out_f32=patch_out)
        hs = torch.empty(rows, d, device="cuda")
        clip = c.arch == "clip"
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        _ok(ctx, lib.cb_assemble_tokens(ctx.h, patch_out.data_ptr(), ptr(f.get("cls")), f["pos"].data_ptr(), ptr(f.get("pre_ln_w")),
                                        ptr(f.get("pre_ln_b")), hs.data_ptr(), n, T, g2, d, c.ln_eps, _stream()), "replay assemble")  # fmt: skip
        hcur = hs
        for i in range(c.layers):
            p = f"L{i}."
            xn = self.ln(hs, f[p + "ln1_w"], f[p + "ln1_b"])
            qkv = self.gemm(xn, h[p + "qkv_w"], f[p + "qkv_b"])
            attn = torch.empty(rows, d, dtype=torch.float16, device="cuda")
            _ok(ctx, lib.cb_attention_f16(ctx.h, qkv.data_ptr(), attn.data_ptr(), n, T, c.heads, hd, _stream()), "replay attention")
            if clip and i == c.layers - 1 and gather == "cls":
                hcur = hs.view(n, T, d)[:, 0].contiguous()
                attn = attn.view(n, T, d)[:, 0].contiguous()
            self.gemm(attn, h[p + "out_w"], f[p + "out_b"], out_f32=hcur, residual=hcur)
            xn = self.ln(hcur, f[p + "ln2_w"], f[p + "ln2_b"])
            mlp = self.gemm(xn, h[p + "fc1_w"], f[p + "fc1_b"], epi=act)
            self.gemm(mlp, h[p + "fc2_w"], f[p + "fc2_b"], out_f32=hcur, residual=hcur)
        out_dim = c.proj_dim or d
        emb, feat, score = (torch.full(s, float("nan"), device="cuda") for s in ((n, out_dim), (n, out_dim), (n,)))
        if clip:
            stride = d if gather == "cls" else T * d
            _ok(ctx, lib.cb_clip_tail(ctx.h, hcur.data_ptr(), stride, f["post_ln_w"].data_ptr(), f["post_ln_b"].data_ptr(), ptr(f.get("proj_w")), d,
                                      c.proj_dim, c.ln_eps, self.aes_w.data_ptr(), self.aes_b, emb.data_ptr(), feat.data_ptr(), score.data_ptr(), n,
                                      _stream()), "replay clip_tail")  # fmt: skip
        else:
            xn = self.ln(hs, f["post_ln_w"], f["post_ln_b"])
            kv = self.gemm(xn, h["map_in_w"][d:].contiguous(), f["map_in_b"][d:].contiguous())
            pooled = torch.empty(n, d, dtype=torch.float16, device="cuda")
            _ok(ctx, lib.cb_map_pool(ctx.h, kv.data_ptr(), self.map_q.data_ptr(), pooled.data_ptr(), n, T, c.heads, hd, _stream()), "replay map_pool")
            r = self.gemm(pooled, h["map_out_w"], f["map_out_b"], out_f32=torch.empty(n, d, device="cuda"))
            xn = self.ln(r, f["map_ln_w"], f["map_ln_b"])
            mlp = self.gemm(xn, h["map_fc1_w"], f["map_fc1_b"], epi=act)
            self.gemm(mlp, h["map_fc2_w"], f["map_fc2_b"], out_f32=r, residual=r)
            _ok(ctx, lib.cb_l2norm_score(ctx.h, r.data_ptr(), d, self.aes_w.data_ptr(), self.aes_b, emb.data_ptr(), feat.data_ptr(), score.data_ptr(), n,
                                         _stream()), "replay l2norm_score")  # fmt: skip
        torch.cuda.synchronize()
        return emb, feat, score

    def forward(self, patches, gather: str = "cls"):
        outs = [self.chunk(patches[i : i + REPLAY_MAX_BATCH], gather) for i in range(0, patches.shape[0], REPLAY_MAX_BATCH)]
        return tuple(torch.cat([o[j] for o in outs]) for j in range(3))


@pytest.mark.parametrize("arch", ["clip", "siglip"])
def test_vit_handle_replay(ctx, arch):
    """VitTower.forward_patches at n = 1, max_batch and max_batch + 1 (two chunks) equals its schedule replayed through the C ABI, bit
    for bit in emb, feat and score; for CLIP also the schedule before the [CLS] gather (every row through the last layer, the tail at
    img_stride = T d), which the gather must not have changed."""
    from oracle import vit
    from cosmos_curate_b200.runtime import VitTower

    cfg = _replay_cfg(arch)
    w = vit.random_weights(cfg, seed=11)
    out_dim = cfg.proj_dim or cfg.hidden
    aes_w = np.random.default_rng(12).standard_normal(out_dim).astype(F32) * F32(0.1)
    tower = VitTower(ctx, cfg.to_dict(), w, max_batch=REPLAY_MAX_BATCH, aesthetic=(aes_w, 0.25))
    try:
        replay = _Replay(ctx, cfg, w, aes_w, 0.25, tower.k_pad)
        g2, kp = cfg.grid**2, 3 * cfg.patch**2
        for n in (1, REPLAY_MAX_BATCH, REPLAY_MAX_BATCH + 1):
            p = torch.zeros(n, g2, tower.k_pad, dtype=torch.float16)
            p[:, :, :kp] = torch.randn(n, g2, kp, generator=torch.Generator().manual_seed(n)).half()
            p = p.cuda()
            got = [t.cpu().numpy() for t in tower.forward_patches(p, want_features=True)]
            torch.cuda.synchronize()
            schedules = ("cls", "none") if arch == "clip" else ("cls",)
            for gather in schedules:
                want = [t.cpu().numpy() for t in replay.forward(p, gather)]
                for name, a, b in zip(("emb", "feat", "score"), got, want):
                    label = "the schedule before the [CLS] gather" if gather == "none" else "the replayed schedule"
                    _assert_bitwise(a, b, f"{arch} n={n}: {name} vs {label}")
    finally:
        tower.close()
