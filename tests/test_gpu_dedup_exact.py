"""The dedup kernels (csrc/dedup.cu) through the C ABI and the dedup module above them, against oracle/dedup.py.

* cb_rowdot_argmax, exact: on dyadic inputs (oracle.dedup.dyadic_rows: every fp32 partial sum is exact) with ties planted in one
  thread, across thread groups, 64-row halves, row tiles and the diagonal tile, values and indices equal rowdot_reference bit for
  bit over every tile boundary of na, nb and d, with and without bias, UPPER and CLIP, and init_val -inf, -1 and a column's exact
  maximum (that column must come back as (init_val, -1));
* cb_rowdot_argmax, bounded: on random unit rows and tight near-duplicate clusters, the returned value is within
  oracle.dedup.rowdot_bound of the float64 score at the returned index, and no candidate scores above it by more than its bound;
  the worst err/bound is printed when the module ends;
* a candidate row holding a NaN is never returned: every column equals the run without that row.  That is the kernel's behaviour,
  pinned here: NaN fails the `v > best` test, and under CLIP fmaxf turns it into -1, which init_val -1 never takes (a float64
  argmax would pick the NaN instead);
* cb_rows_l2_normalize: bit for bit x / |x| where |x| is exact, the 1e-12 clamp, zero rows, within l2_normalize_bound elsewhere;
* cb_cluster_sums: bit for bit the sequential fp32 sum of oracle.dedup.cluster_sums_sequential, up to 70000 clusters;
* semdedup_cluster, assign_to_centroids and one spherical_kmeans step on unit-exact rows: equal to the oracle exactly;
* inputs are followed by NaN rows, outputs are sentinel-filled with guard elements that must not change; repeat launches are
  bitwise equal; every argument error returns its code before anything is launched.
"""

from __future__ import annotations

import zlib

import numpy as np
import pytest
import torch

from gpu_helpers import ctx  # noqa: F401
from oracle import dedup as od

pytestmark = pytest.mark.gpu

F32 = np.float32
PAD = 3  # NaN rows after every input, sentinel guard elements before and after every output
SENTINEL_I32 = -123456789
ARG, UNSUPPORTED = -2, -3
UPPER, CLIP = 1, 2


def _stream():
    from cosmos_curate_b200.runtime import _stream_ptr

    return _stream_ptr()


def _seed(name: str) -> int:
    return zlib.crc32(name.encode())


def _ok(ctx, rc: int, what: str) -> None:
    from cosmos_curate_b200.runtime import check

    check(rc, what, ctx.h)


_LIVE: list[torch.Tensor] = []  # inputs whose raw pointers were handed to the library: alive until the test ends


@pytest.fixture(autouse=True)
def _inputs_live_until_the_test_ends():
    yield
    torch.cuda.synchronize()
    _LIVE.clear()


def _in(a: np.ndarray) -> torch.Tensor:
    """a on the device as the first rows of a buffer with PAD rows after it: NaN for floats, 0 for integers (an index)."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    fill = float("nan") if t.is_floating_point() else 0
    buf = torch.full((t.shape[0] + PAD, *t.shape[1:]), fill, dtype=t.dtype, device="cuda")
    buf[: t.shape[0]] = t.cuda()
    _LIVE.append(buf)
    return buf[: t.shape[0]]


def _bits(a: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(a).view(np.int32)


class Out:
    """A sentinel-filled output (NaN, or SENTINEL_I32) with PAD guard rows before and after; `fill` replaces the output part."""

    def __init__(self, shape, dtype, fill: np.ndarray | None = None):
        s = float("nan") if dtype == torch.float32 else SENTINEL_I32
        self.buf = torch.full((shape[0] + 2 * PAD, *shape[1:]), s, dtype=dtype, device="cuda")
        self.t = self.buf[PAD : PAD + shape[0]]
        if fill is not None:
            self.t.copy_(torch.from_numpy(np.ascontiguousarray(fill)))
        self.before = self.buf.clone()

    @property
    def ptr(self) -> int:
        return self.t.data_ptr()

    def get(self, what: str, nan_ok: bool = False) -> np.ndarray:
        torch.cuda.synchronize()
        b, a = _bits(self.buf.cpu().numpy()), _bits(self.before.cpu().numpy())
        n = self.t.shape[0]
        assert np.array_equal(b[:PAD], a[:PAD]), f"{what}: elements before the output were written"
        assert np.array_equal(b[PAD + n :], a[PAD + n :]), f"{what}: elements after the output were written"
        out = self.t.cpu().numpy()
        if out.dtype == np.int32:
            assert not (out == SENTINEL_I32).any(), f"{what}: output element {np.argwhere(out == SENTINEL_I32)[0].tolist()} not written"
        elif not nan_ok:
            assert not np.isnan(out).any(), f"{what}: NaN in the output at {np.argwhere(np.isnan(out))[0].tolist()}"
        return out


def _assert_bitwise(got: np.ndarray, want: np.ndarray, what: str) -> None:
    got, want = np.asarray(got), np.asarray(want).astype(got.dtype)
    bad = np.argwhere(_bits(got) != _bits(want))
    if len(bad):
        i = tuple(bad[0])
        pytest.fail(f"{what}: {len(bad)} of {got.size} elements differ; first at {list(i)}: got {got[i]!r} want {want[i]!r}")


@pytest.fixture(scope="module")
def record(pytestconfig):
    """Worst err/bound per kernel, written to the terminal (past output capture) when the module ends."""
    r: dict[str, float] = {}
    yield r
    capman = pytestconfig.pluginmanager.get_plugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print("\n" + "\n".join(f"{k}: worst err/bound {v:.3f}" for k, v in sorted(r.items())))


def _note(record, key: str, worst: float) -> None:
    record[key] = max(record.get(key, 0.0), worst)


# ------------------------------------------------------------------------------------------------ rowdot_argmax
def _rowdot(ctx, a: torch.Tensor, na: int, b: torch.Tensor, nb: int, d: int, bias, flags: int, init: float, what: str):
    val, idx = Out((nb,), torch.float32), Out((nb,), torch.int32)
    _ok(ctx, ctx.lib.cb_rowdot_argmax(ctx.h, a.data_ptr(), na, b.data_ptr(), nb, d, None if bias is None else bias.data_ptr(), flags, init,
                                      val.ptr, idx.ptr, _stream()), what)  # fmt: skip
    return val.get(what), idx.get(what)


NA = (0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1000)
NB = (1, 127, 128, 129, 257, 1000)
M_UPPER = (1, 2, 127, 128, 129, 256, 257, 4097)
DS = (16, 32, 48, 768, 1024)
EXACT_CASES = [(False, na, nb) for na in NA for nb in NB] + [(True, m, m) for m in M_UPPER]


@pytest.mark.parametrize(("upper", "na", "nb"), EXACT_CASES, ids=[f"{'upper' if u else 'full'}-na{a}-nb{b}" for u, a, b in EXACT_CASES])
def test_rowdot_argmax_exact(ctx, upper, na, nb):
    """Every d, bias or not, CLIP or not, init_val -inf / -1 / one column's exact maximum: values and indices bit for bit."""
    for d in DS:
        name = f"rowdot {'upper' if upper else 'full'} na={na} nb={nb} d={d}"
        rng = np.random.default_rng(_seed(name))
        a, bias = od.dyadic_rows(na, d, rng), od.dyadic_bias(na, rng)
        a, bias, b, planted = od.plant_ties(a, bias, None if upper else od.dyadic_rows(nb, d, rng), rng)
        if upper:
            b = a
        if na:
            at, biast = _in(a), _in(bias)
        else:  # a zero-row view has no address: na = 0 rows of a NaN row, which the kernel must not read
            at, biast = _in(np.full((1, d), np.nan, F32)), _in(np.full(1, np.nan, F32))
        bt = at if upper else _in(b)
        prod = np.asarray(a, np.float64) @ np.asarray(b, np.float64).T
        for use_bias in (False, True):
            for clip in (False, True):
                s = od.rowdot_scores(a, b, bias if use_bias else None, upper, clip, prod=prod)
                v_all, _ = od.rowdot_pick(s, -np.inf)
                cols = np.flatnonzero(np.isfinite(v_all))
                j_eq = int(cols[len(cols) // 2]) if len(cols) else None
                inits = [-np.inf, -1.0] + ([float(v_all[j_eq])] if j_eq is not None else [])
                for init in inits:
                    what = f"{name} bias={use_bias} clip={clip} init_val={init}"
                    flags = (UPPER if upper else 0) | (CLIP if clip else 0)
                    got_v, got_i = _rowdot(ctx, at, na, bt, nb, d, biast if use_bias else None, flags, init, what)
                    want_v, want_i = od.rowdot_pick(s, init)
                    _assert_bitwise(got_i, want_i, f"{what}: index")
                    _assert_bitwise(got_v, want_v.astype(F32), f"{what}: value")
                    if j_eq is not None and init == v_all[j_eq]:
                        assert got_i[j_eq] == -1 and got_v[j_eq] == F32(init), f"{what}: column {j_eq}'s maximum equals init_val"
                    if upper:
                        assert got_i[0] == -1 and got_v[0] == F32(init), f"{what}: column 0 has no candidate"
        s = od.rowdot_scores(a, b, None, upper, False, prod=prod)
        for tie, pos, cols_t in planted:  # the planted columns did test a tie: without bias or clip, exactly the copies attain the maximum
            for j in pos[1:] if upper else cols_t:
                ties = np.flatnonzero(s[:, j] == s[:, j].max())
                assert list(ties) == [p for p in pos if not upper or p < j], f"{name}: tie group {tie}, column {j}"


def test_rowdot_argmax_antipodal_and_clipped_ties(ctx):
    """Unit-exact rows +-s x (s in 1, 2.5, 1/8) over 300 rows: under CLIP every same-sign pair with s_i s_j >= 1 ties at exactly 1.0
    (the first index wins), opposite signs score -1 or above; with init_val -1 a column whose earlier rows are all antipodal gets -1."""
    d = 16
    x = np.zeros(d, F32)
    x[[1, 6, 9, 14]] = [0.5, -0.5, 0.5, 0.5]
    y = np.zeros(d, F32)
    y[[0, 2, 3, 4]] = 0.5
    motif = np.stack([x, -x, 2.5 * x, -0.125 * x, x, y, -y]).astype(F32)
    want_i = [-1, -1, 0, 1, 0, 0, 0]
    want_v = [-1.0, -1.0, 1.0, 0.125, 1.0, 0.0, 0.0]
    mt = _in(motif)
    v, i = _rowdot(ctx, mt, 7, mt, 7, d, None, UPPER | CLIP, -1.0, "antipodal motif")
    assert list(i) == want_i and list(v) == want_v
    n = 300
    s = np.array([(1.0, 2.5, 0.125)[k % 3] * (1 if (k // 3) % 2 == 0 else -1) for k in range(n)], F32)
    rows = (s[:, None] * x[None]).astype(F32)
    rt = _in(rows)
    for init in (-1.0, -np.inf):
        got_v, got_i = _rowdot(ctx, rt, n, rt, n, d, None, UPPER | CLIP, init, f"scaled duplicates init_val={init}")
        want_v, want_i = od.rowdot_reference(rows, rows, upper=True, clip=True, init_val=init)
        _assert_bitwise(got_i, want_i, f"scaled duplicates init_val={init}: index")
        _assert_bitwise(got_v, want_v.astype(F32), f"scaled duplicates init_val={init}: value")
    # rows x, 2.5 x, x / 8, -x, -2.5 x, -x / 8, x, ...: 2.5 x clips to a tie at 1.0 on x; -x takes the least negative, -x / 8
    assert (got_i[1], got_v[1], got_i[2], got_v[2], got_i[3], got_v[3]) == (0, 1.0, 1, 0.3125, 2, -0.125)
    assert (got_v == 1.0).sum() > n // 2 and got_i[6] == 0


def _unit_rows(n: int, d: int, rng, near: bool) -> np.ndarray:
    if not near:
        return od.l2_normalize(rng.standard_normal((n, d)))
    c = od.l2_normalize(rng.standard_normal((max(1, n // 40), d)))
    noise = rng.standard_normal((n, d)) / np.sqrt(d) * rng.uniform(0, 0.14, (n, 1))  # cosine to the center ~0.99 .. 1
    return od.l2_normalize(c[rng.integers(0, len(c), n)] + noise)


BOUND_CASES = [(kind, na, nb, d, upper) for kind in ("random", "near") for na, nb, d, upper in
               ((1000, 1000, 768, True), (4097, 4097, 1024, True), (129, 129, 16, True), (257, 129, 1024, False), (600, 1000, 48, False),
                (1000, 257, 768, False))]  # fmt: skip


@pytest.mark.parametrize(("kind", "na", "nb", "d", "upper"), BOUND_CASES,
                         ids=[f"{k}-na{a}-nb{b}-d{d}-{'upper' if u else 'full'}" for k, a, b, d, u in BOUND_CASES])  # fmt: skip
def test_rowdot_argmax_bounded(ctx, record, kind, na, nb, d, upper):
    name = f"rowdot {kind} na={na} nb={nb} d={d} upper={upper}"
    rng = np.random.default_rng(_seed(name))
    a = _unit_rows(na, d, rng, kind == "near")
    b = a if upper else _unit_rows(nb, d, rng, kind == "near")
    bias = (rng.standard_normal(na) * 0.01).astype(F32)
    at = _in(a)
    bt = at if upper else _in(b)
    prod = np.asarray(a, np.float64) @ np.asarray(b, np.float64).T
    cols = np.arange(nb)
    for use_bias in (False, True):
        bv = bias if use_bias else None
        bnd = od.rowdot_bound(a, b, bv)
        for clip in (False, True):
            init = -1.0 if clip else -np.inf
            what = f"{name} bias={use_bias} clip={clip}"
            got_v, got_i = _rowdot(ctx, at, na, bt, nb, d, _in(bv) if use_bias else None, (UPPER if upper else 0) | (CLIP if clip else 0), init, what)
            s = od.rowdot_scores(a, b, bv, upper, clip, prod=prod)
            has = got_i >= 0
            gi = np.where(has, got_i, 0)
            assert np.all(np.isfinite(s[gi[has], cols[has]])), f"{what}: an index outside the candidates"
            err = np.abs(got_v[has].astype(np.float64) - s[gi[has], cols[has]])
            ratio = err / np.maximum(bnd[gi[has], cols[has]], 1e-300)
            worst = float(ratio.max(initial=0.0))
            _note(record, "rowdot_argmax", worst)
            assert worst <= 1.0, f"{what}: err/bound {worst:.3f} at column {cols[has][ratio.argmax()]}"
            # no candidate above the returned value by more than its bound (for (init_val, -1) columns: above init_val)
            ref_v = np.where(has, got_v.astype(np.float64), init)
            with np.errstate(invalid="ignore"):  # -inf - -inf where a column has no candidate at all
                over = s - (ref_v[None, :] + bnd)
            assert not np.any(over > 0), f"{what}: column {np.argwhere(over > 0)[0][1]} has a candidate above the returned value"
            assert np.all(got_v[~has] == F32(init)), f"{what}: (init_val, -1) columns"


@pytest.mark.parametrize(("upper", "clip", "init"), [(False, False, -np.inf), (False, True, -1.0), (False, True, -np.inf), (True, True, -1.0),
                                                      (True, False, -np.inf)])  # fmt: skip
def test_rowdot_argmax_nan_candidate_is_never_returned(ctx, upper, clip, init):
    what = f"NaN candidate upper={upper} clip={clip} init_val={init}"
    rng = np.random.default_rng(_seed(what))
    na, nb, d, k = 300, 300 if upper else 200, 64, 130
    a = _unit_rows(na, d, rng, near=True)
    a[k + 1] = a[k - 1]  # a tie across the NaN row
    b = a if upper else _unit_rows(nb, d, rng, near=True)
    bad = a.copy()
    bad[k, 5] = np.nan
    flags = (UPPER if upper else 0) | (CLIP if clip else 0)
    t = _in(bad)
    got_v, got_i = _rowdot(ctx, t, na, t if upper else _in(b), nb, d, None, flags, init, what)
    keep = np.delete(np.arange(na), k)
    r = _in(a[keep])
    ref_v, ref_i = _rowdot(ctx, r, na - 1, r if upper else _in(b), nb - 1 if upper else nb, d, None, flags, init, f"{what}: without the row")
    assert not np.any(got_i == k), f"{what}: the NaN row was returned"
    cols = np.delete(np.arange(nb), k) if upper else np.arange(nb)
    _assert_bitwise(got_v[cols], ref_v, f"{what}: value")
    _assert_bitwise(got_i[cols], np.where(ref_i >= k, ref_i + 1, ref_i), f"{what}: index")
    if upper:  # the NaN row's own column: every score NaN (-1 under CLIP), nothing taken
        assert got_i[k] == -1 and got_v[k] == F32(init)


# ------------------------------------------------------------------------------------------------ rows_l2_normalize
ND = (1, 3, 16, 127, 128, 129, 768, 1000, 4096)


def _norm_rows(d: int, rng) -> tuple[np.ndarray, np.ndarray, int, int]:
    """Exact rows (the sum of squares and its root exact in fp32), a clamp row [2^-50, 0, ...], a zero row, then random rows of
    scales 1e-3 .. 1e4.  Returns (x, exact-row mask, clamp row, zero row)."""
    exact = []
    for s in (1.0, 2.5, 0.125):
        exact.append(np.r_[3 * s, np.zeros(d - 1)])
        if d >= 2:
            r = np.zeros(d)
            r[rng.choice(d, 2, replace=False)] = [3 * s, -4 * s]
            exact.append(r)
        for nnz in (4, 16):
            if d >= nnz:
                r = np.zeros(d)
                r[rng.choice(d, nnz, replace=False)] = np.where(rng.random(nnz) < 0.5, -s, s)
                exact.append(r)
    clamp = np.zeros(d)
    clamp[0] = 2.0**-50
    rand = rng.standard_normal((20, d)) * 10 ** rng.uniform(-3, 4, (20, 1))
    x = np.concatenate([np.array(exact), clamp[None], np.zeros((1, d)), rand]).astype(F32)
    mask = np.zeros(len(x), bool)
    mask[: len(exact)] = True
    return x, mask, len(exact), len(exact) + 1


@pytest.mark.parametrize("d", ND)
def test_rows_l2_normalize(ctx, record, d):
    what = f"rows_l2_normalize d={d}"
    x, exact, clamp, zero = _norm_rows(d, np.random.default_rng(_seed(what)))
    rows = len(x)
    y, nrm = Out((rows, d), torch.float32, fill=x), Out((rows,), torch.float32)
    _ok(ctx, ctx.lib.cb_rows_l2_normalize(ctx.h, y.ptr, rows, d, nrm.ptr, _stream()), what)
    got, got_n = y.get(what), nrm.get(what)
    want_n = np.sqrt((x[exact].astype(np.float64) ** 2).sum(1)).astype(F32)
    _assert_bitwise(got_n[exact], want_n, f"{what}: exact norms")
    _assert_bitwise(got[exact], x[exact] / want_n[:, None], f"{what}: exact rows")
    assert got_n[clamp] == F32(2.0**-50) and got[clamp, 0] == F32(2.0**-50) / F32(1e-12) and not got[clamp, 1:].any(), f"{what}: clamp"
    assert got_n[zero] == 0 and not got[zero].any() and not np.signbit(got[zero]).any(), f"{what}: zero row"
    rest = ~exact
    rest[[clamp, zero]] = False
    b_y, b_n = od.l2_normalize_bound(x[rest])
    x64 = x[rest].astype(np.float64)
    n64 = np.sqrt((x64 * x64).sum(1))
    wy = float((np.abs(got[rest] - x64 / n64[:, None]) / np.maximum(b_y, 1e-300)).max())
    wn = float((np.abs(got_n[rest] - n64) / b_n).max())
    _note(record, "rows_l2_normalize", max(wy, wn))
    assert wy <= 1.0 and wn <= 1.0, f"{what}: err/bound {wy:.3f} (rows), {wn:.3f} (norms)"
    # norms_out = nullptr: the same rows
    y2 = Out((rows, d), torch.float32, fill=x)
    _ok(ctx, ctx.lib.cb_rows_l2_normalize(ctx.h, y2.ptr, rows, d, None, _stream()), f"{what}, no norms")
    _assert_bitwise(y2.get(f"{what}, no norms"), got, f"{what}: without norms_out")
    # a row of Inf and a row of NaN leave their neighbours bitwise unchanged
    xb = x.copy()
    xb[rows - 5], xb[rows - 3] = np.inf, np.nan
    y3, n3 = Out((rows, d), torch.float32, fill=xb), Out((rows,), torch.float32)
    _ok(ctx, ctx.lib.cb_rows_l2_normalize(ctx.h, y3.ptr, rows, d, n3.ptr, _stream()), f"{what}, Inf / NaN rows")
    ok = np.ones(rows, bool)
    ok[[rows - 5, rows - 3]] = False
    _assert_bitwise(y3.get(f"{what}, Inf / NaN rows", nan_ok=True)[ok], got[ok], f"{what}: neighbours of Inf / NaN rows")
    _assert_bitwise(n3.get(f"{what}, Inf / NaN rows", nan_ok=True)[ok], got_n[ok], f"{what}: neighbours' norms")


# ------------------------------------------------------------------------------------------------ cluster_sums
def _cluster_case(n_clusters: int, d: int, rng, max_len: int = 5, extra: int = 5):
    """Clusters of 0 .. max_len rows (about 10% more of them empty), `extra` NaN rows outside every segment, order a permutation."""
    lens = rng.integers(0, max_len + 1, n_clusters)
    lens[rng.random(n_clusters) < 0.1] = 0
    seg = np.r_[0, np.cumsum(lens)].astype(np.int64)
    n = int(seg[-1]) + extra
    x = (rng.standard_normal((n, d)) * 10 ** rng.uniform(-2, 2, (n, 1))).astype(F32)
    order = rng.permutation(n).astype(np.int64)
    x[order[seg[-1] :]] = np.nan
    sums0 = rng.standard_normal((n_clusters, d)).astype(F32)
    return x, order, seg, sums0


CS_CASES = [(300, d) for d in (1, 16, 255, 256, 257, 768)] + [(k, 257) for k in (1, 65535, 65536, 70000)] + [(2, 65535 * 256 + 300)]


@pytest.mark.parametrize(("n_clusters", "d"), CS_CASES, ids=[f"k{k}-d{d}" for k, d in CS_CASES])
def test_cluster_sums_exact(ctx, n_clusters, d):
    """Bit for bit the sequential fp32 sum per cluster, added once to a non-zero sums (+=, not =), with an arbitrary order, empty
    clusters, NaN rows outside every segment; any number of clusters (grid x), and d past 65535 dimension blocks (grid-y stride)."""
    what = f"cluster_sums n_clusters={n_clusters} d={d}"
    rng = np.random.default_rng(_seed(what))
    x, order, seg, sums0 = _cluster_case(n_clusters, d, rng) if d < 1 << 20 else _cluster_case(n_clusters, d, rng, max_len=2, extra=1)
    out = Out((n_clusters, d), torch.float32, fill=sums0)
    _ok(ctx, ctx.lib.cb_cluster_sums(ctx.h, _in(x).data_ptr(), _in(order).data_ptr(), _in(seg).data_ptr(), n_clusters, d, out.ptr, _stream()), what)
    _assert_bitwise(out.get(what), od.cluster_sums_sequential(x, order, seg, sums0), what)


# ------------------------------------------------------------------------------------------------ the dedup module
SEM_CASES = [(m, d) for d in (72, 768) for m in M_UPPER]


@pytest.mark.parametrize(("m", "d"), SEM_CASES, ids=[f"m{m}-d{d}" for m, d in SEM_CASES])
def test_semdedup_cluster_exact(ctx, m, d):
    """Unit-exact embeddings (normalisation exact, cosines multiples of 1/16): the whole of semdedup_cluster equals pairwise_max
    exactly; d = 72 goes through the pad-to-16 path; sort-key ties; eps = 0.25 puts scores exactly on the 0.75 threshold."""
    from cosmos_curate_b200 import dedup

    rng = np.random.default_rng(_seed(f"semdedup m={m} d={d}"))
    emb = od.unit_exact_rows(m, d, rng)
    dist = (rng.integers(0, 6, m) / 8).astype(F32)
    ids = np.array([f"clip-{i:05d}" for i in range(m)])
    for eps in (0.25, 0.01):
        got = dedup.semdedup_cluster(ids, emb, dist, eps, ctx=ctx)
        want = od.pairwise_max(ids, emb, dist, eps)
        assert np.array_equal(got["id"], want["id"]) and np.array_equal(got["max_id"], want["max_id"])
        _assert_bitwise(got["cosine_sim_score"], want["cosine_sim_score"], f"m={m} d={d} eps={eps}: cosine_sim_score")
        assert got["kept"] == want["kept"] and got["total"] == m
        if m >= 128 and eps == 0.25:
            assert np.any(want["cosine_sim_score"] == F32(0.75))  # on the threshold: kept (<=)


def test_assign_to_centroids_identical_centroids_take_the_first(ctx):
    from cosmos_curate_b200 import dedup

    rng = np.random.default_rng(21)
    c = od.dyadic_rows(6, 32, rng)
    c[4] = c[1]
    x = od.dyadic_rows(700, 32, rng)
    x[::7] = c[1]
    labels, _ = dedup.assign_to_centroids(torch.from_numpy(x).cuda(), torch.from_numpy(c).cuda(), ctx=ctx)
    labels = labels.cpu().numpy()
    _, want = od.rowdot_reference(c, x, -0.5 * (c.astype(np.float64) ** 2).sum(1))
    assert np.array_equal(labels, want) and not np.any(labels == 4) and np.all(labels[::7] == 1)


def test_spherical_kmeans_one_step_exact(ctx):
    """max_iter=1 on unit-exact rows: centroids are bit for bit the float32 sums / counts of the oracle's exact labels; two initial
    centroids coincide (a scaled duplicate), so the second gets no members and keeps its centroid."""
    from cosmos_curate_b200 import dedup

    n, k, d_in, seed = 400, 9, 72, 3
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:k].numpy()
    x = od.unit_exact_rows(n, d_in, np.random.default_rng(22))
    x[perm[1]] = x[perm[0]] * F32(2.5)
    assert np.count_nonzero(x[perm[0]])
    r = dedup.spherical_kmeans(x, k, max_iter=1, seed=seed, tol=0.0, ctx=ctx)
    xu = np.zeros((n, 80), F32)
    xu[:, :d_in] = od.l2_normalize(x)
    cent = xu[perm]
    _, labels = od.rowdot_reference(cent, xu, -0.5 * (cent.astype(np.float64) ** 2).sum(1))
    order = np.argsort(labels, kind="stable")
    counts = np.bincount(labels, minlength=k)
    seg = np.r_[0, np.cumsum(counts)]
    sums = od.cluster_sums_sequential(xu, order, seg, np.zeros((k, 80), F32))
    want = np.where(counts[:, None] > 0, sums / np.maximum(counts, 1).astype(F32)[:, None], cent).astype(F32)
    assert counts[1] == 0 and counts[0] > 0
    _assert_bitwise(r["centroids"].cpu().numpy(), want[:, :d_in], "spherical_kmeans one step: centroids")
    assert r["n_iter"] == 1


# ------------------------------------------------------------------------------------------------ repeat launches
def test_repeat_launches_bitwise_equal(ctx):
    rng = np.random.default_rng(9)
    m, d = 3000, 768
    a = _unit_rows(m, d, rng, near=True)
    at = _in(a)
    x, order, seg, sums0 = _cluster_case(500, 257, rng)
    xt, ot, st = _in(x), _in(order), _in(seg)
    first = None
    for _ in range(3):
        v, i = _rowdot(ctx, at, m, at, m, d, None, UPPER | CLIP, -1.0, "rowdot repeat")
        y = Out((m, d), torch.float32, fill=a * F32(3))
        _ok(ctx, ctx.lib.cb_rows_l2_normalize(ctx.h, y.ptr, m, d, None, _stream()), "normalize repeat")
        s = Out((500, 257), torch.float32, fill=sums0)
        _ok(ctx, ctx.lib.cb_cluster_sums(ctx.h, xt.data_ptr(), ot.data_ptr(), st.data_ptr(), 500, 257, s.ptr, _stream()), "cluster_sums repeat")
        now = (v, i, y.get("normalize repeat"), s.get("cluster_sums repeat"))
        if first is None:
            first = now
        for got, want, name in zip(now, first, ("rowdot value", "rowdot index", "rows_l2_normalize", "cluster_sums")):
            _assert_bitwise(got, want, f"{name}: a repeat launch")


# ------------------------------------------------------------------------------------------------ argument errors
_B = ("a", "b", "c", "d", "e", "f")  # six 1 MB NaN buffers; an argument "a+4" is buffer a's address plus 4 bytes

_VALID = {  # export -> argument list of a valid call (buffer names, ints, floats)
    "cb_rowdot_argmax": ["a", 8, "b", 8, 16, "c", 0, -1.0, "d", "e"],
    "cb_rows_l2_normalize": ["a", 8, 16, "b"],
    "cb_cluster_sums": ["a", "b", "c", 4, 16, "d"],
}
_ERRORS = [  # (id, export, {argument index: value}, code)
    ("rowdot_d_not_16k", "cb_rowdot_argmax", {4: 24}, UNSUPPORTED),
    ("rowdot_d_zero", "cb_rowdot_argmax", {4: 0}, UNSUPPORTED),
    ("rowdot_upper_a_not_b", "cb_rowdot_argmax", {6: UPPER}, ARG),
    ("rowdot_upper_na_not_nb", "cb_rowdot_argmax", {6: UPPER | CLIP, 2: "a", 3: 7}, ARG),
    ("rowdot_null_a", "cb_rowdot_argmax", {0: None}, ARG),
    ("rowdot_null_b", "cb_rowdot_argmax", {2: None}, ARG),
    ("rowdot_null_out_val", "cb_rowdot_argmax", {8: None}, ARG),
    ("rowdot_null_out_idx", "cb_rowdot_argmax", {9: None}, ARG),
    ("rowdot_a_misaligned", "cb_rowdot_argmax", {0: "a+4"}, ARG),
    ("rowdot_b_misaligned", "cb_rowdot_argmax", {2: "b+4"}, ARG),
    ("rowdot_upper_misaligned", "cb_rowdot_argmax", {0: "a+8", 2: "a+8", 6: UPPER}, ARG),
    ("l2_null_x", "cb_rows_l2_normalize", {0: None}, ARG),
    ("l2_d_zero", "cb_rows_l2_normalize", {2: 0}, ARG),
    ("sums_null_x", "cb_cluster_sums", {0: None}, ARG),
    ("sums_null_order", "cb_cluster_sums", {1: None}, ARG),
    ("sums_null_seg", "cb_cluster_sums", {2: None}, ARG),
    ("sums_null_sums", "cb_cluster_sums", {5: None}, ARG),
    ("sums_n_clusters_zero", "cb_cluster_sums", {3: 0}, ARG),
    ("sums_d_zero", "cb_cluster_sums", {4: 0}, ARG),
]
_NOOPS = [("cb_rowdot_argmax", {3: 0}), ("cb_rows_l2_normalize", {1: 0})]


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
    """Each bad argument returns its code before anything is launched and leaves every buffer untouched."""
    assert _call_with(ctx, fn, changes) == code


@pytest.mark.parametrize(("fn", "changes"), _NOOPS, ids=[f[0] for f in _NOOPS])
def test_zero_rows_is_a_no_op(ctx, fn, changes):
    assert _call_with(ctx, fn, changes) == 0
