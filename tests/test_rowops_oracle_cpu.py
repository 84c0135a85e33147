"""The row-kernel oracle (oracle/rowops.py) is well-posed: its dispatch is the one written in csrc/vit_kernels.cu, its sweep puts
every norm instantiation on every row boundary, its float32 models round as step-by-step arithmetic says, its exact input classes
really are exact, and its acceptance rules reject the wrong formulas a kernel could plausibly contain."""

from __future__ import annotations

from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import rowops as R

F32, F16 = np.float32, np.float16


def _rng(seed: int) -> np.random.Generator:
    return np.random.default_rng(seed)


# ------------------------------------------------------------------------------------------------ dispatch and sweep
def test_dispatch_matches_vit_kernels_cu():
    assert R.dispatch_from_source() == R.DISPATCH


@pytest.mark.parametrize("sm", [132, 114])
def test_sweep_reaches_every_instantiation_at_every_row_class(sm):
    for kernel in R.NORMS:
        pts = R.norm_sweep(kernel, sm)
        assert {p.d for p in pts} == set(R.WIDTHS)
        insts = {R.instantiation(kernel, d) for d in R.WIDTHS}
        special, generic = R.DISPATCH[kernel]
        assert insts == {*special.values(), generic}
        got = {(p.inst, p.rows) for p in pts}
        assert got == {(i, r) for i in insts for r in R.rows_classes(sm)}, kernel


def test_pool_sweep_covers_slices_and_the_shared_memory_opt_in():
    for kind in ("map", "clip"):
        pts = R.pool_sweep(kind)
        assert {hd for hd, _ in pts} == set(R.HEAD_DIMS)
        assert {t for _, t in pts} == {*R.TOKENS, R.POOL_BIG_TOKENS}
    assert [R.pool_slices(h) for h in R.HEAD_DIMS] == [4, 3, 2, 2]
    assert [R.pool_slices(h) * h for h in R.HEAD_DIMS] == [256, 216, 176, 256]
    assert (R.POOL_BIG_TOKENS + 256) * 4 > 48 * 1024 >= (max(R.TOKENS) + 256) * 4


# ------------------------------------------------------------------------------------------------ float32 arithmetic
def _fma_exact(a, b, c) -> F32:
    """Rational a * b + c rounded to float32 (ties to even) - the definition of fma."""
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    lo = F32(float(x))  # float(x) is the nearest double; search the float32 neighbours around it exactly
    cands = [np.nextafter(lo, F32(-np.inf)), lo, np.nextafter(lo, F32(np.inf))]
    best = min(cands, key=lambda f: (abs(Fraction(float(f)) - x), int(np.array(f).view(np.int32)) & 1))
    return best


def test_fma_is_correctly_rounded():
    r = _rng(1)
    a = (r.standard_normal(3000) * 2.0 ** r.integers(-30, 30, 3000)).astype(F32)
    b = (r.standard_normal(3000) * 2.0 ** r.integers(-30, 30, 3000)).astype(F32)
    c = (-(a.astype(np.float64) * b) * (1 + r.standard_normal(3000) * 2.0**-20)).astype(F32)  # heavy cancellation
    c[::3] = (r.standard_normal(1000) * 1e-30).astype(F32)  # a tiny addend: the double-rounding case
    # products that land exactly half a float32 ulp away from a representable value, with a tiny addend deciding the direction
    a[:200] = F32(1 + 2.0**-12)
    b[:200] = F32(1 + 2.0**-12)  # a * b = 1 + 2^-11 + 2^-24: a float32 tie
    c[:200] = np.where(np.arange(200) % 2, F32(2.0**-60), F32(-(2.0**-60)))
    got = R.fma(a, b, c)
    want = np.array([_fma_exact(x, y, z) for x, y, z in zip(a, b, c)], F32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def _ln_scalar(x: np.ndarray, eps: float):
    """ln_row restated one lane and one step at a time, float64 operations rounded to float32 after each step."""
    d = len(x)
    f = lambda v: F32(v)  # noqa: E731
    lane_s = []
    for lane in range(32):
        s = F32(0)
        for i in range(d // 128):
            e = x[(i * 32 + lane) * 4 : (i * 32 + lane) * 4 + 4]
            s = f(float(s) + float(f(f(float(e[0]) + float(e[1])) + float(f(float(e[2]) + float(e[3]))))))
        lane_s.append(s)

    def butterfly(v):
        v = list(v)
        for o in (16, 8, 4, 2, 1):
            v = [f(float(v[i]) + float(v[i ^ o])) for i in range(32)]
        assert len(set(np.array(v).view(np.int32).tolist())) == 1
        return v[0]

    mean = f(float(butterfly(lane_s)) / d)
    lane_q = []
    for lane in range(32):
        q = F32(0)
        for i in range(d // 128):
            c = [f(float(v) - float(mean)) for v in x[(i * 32 + lane) * 4 : (i * 32 + lane) * 4 + 4]]
            q = f(float(q) + float(f(float(_fma_exact(c[0], c[0], f(float(c[1]) * float(c[1])))) + float(_fma_exact(c[2], c[2], f(float(c[3]) * float(c[3])))))))
        lane_q.append(q)
    return mean, f(float(f(float(butterfly(lane_q)) / d)) + float(F32(eps)))


def test_layernorm_model_is_the_stepwise_float32_arithmetic():
    r = _rng(2)
    x = (r.standard_normal((3, 256)) * 3 + 1).astype(F32)
    mean, arg = R.ln_stats(x, 1e-5)
    for i in range(3):
        m, a = _ln_scalar(x[i], 1e-5)
        assert mean[i] == m and arg[i] == a


def test_block_and_warp_sums_are_the_butterfly():
    r = _rng(3)
    v = r.standard_normal((4, 256)).astype(F32)
    w = [R.warp_sum(v[:, 32 * k : 32 * k + 32]) for k in range(8)]
    assert np.array_equal(R.block_sum(v), R.warp_sum(np.concatenate([np.stack(w, 1), np.zeros((4, 24), F32)], 1)))
    assert np.allclose(R.block_sum(v), v.astype(np.float64).sum(1), rtol=1e-5)


def test_rstd_candidates_bracket_the_true_rsqrt():
    x = np.array([1e-5, 0.7, 1.0, 3.9, 1e6], F32)
    c = dict(R.rstd_candidates(x))
    assert np.array_equal(c[0], R.rsqrt_rn(x))
    for k in (-2, -1, 1, 2):
        assert np.all((c[k] > c[0]) == (k > 0))


# ------------------------------------------------------------------------------------------------ exact input classes
@pytest.mark.parametrize("hd", R.HEAD_DIMS)
@pytest.mark.parametrize("t", [1, 257, 2049])
def test_pool_uniform_class_is_exact(hd, t):
    k, v, q = R.pool_uniform_inputs(2, t, hd, seed=t + hd)
    s = R.pool_scores_f32(k, q)
    assert np.all(s == s[:, :1]), "every key's score must be the same float32"
    sums = v.astype(np.float64).sum(1)
    assert np.array_equal(sums.astype(F32).astype(np.float64), sums), "V's sums must be exact in fp32"
    # __expf(0) = ex2(0) = 1 exactly: the model with the kernel's expf argument reproduces itself with any expf that maps 0 -> 1
    got = R.pool_f32(k, v, q, expf=lambda x: np.where(x == 0, F32(1), F32(np.nan)))
    assert np.array_equal(got.view(np.int16), R.pool_f32(k, v, q).view(np.int16))


@pytest.mark.parametrize("hd", R.HEAD_DIMS)
@pytest.mark.parametrize("t", [1, 2, 729, R.POOL_BIG_TOKENS])
def test_pool_onehot_class_is_exact(hd, t):
    for scale in (1.0, hd**-0.5):
        k, v, q, j = R.pool_onehot_inputs(2, t, hd, seed=t * 7 + hd, scale=scale)
        qh = (q * F32(scale)).astype(F32)
        s = R.pool_scores_f32(k, qh)
        x = s - s.max(1, keepdims=True)
        others = np.ones_like(x, bool)
        others[np.arange(2), j] = False
        assert np.all(x[others] <= -120), "every other key must trail by >= 120 nats"
        assert np.all(x[~others] == 0)
        # any __expf within its documented error maps x <= -120 to 0: 2^(-120 log2 e) < 2^-173, far below 2^-149
        got = R.pool_f32(k, v, qh, expf=lambda y: np.where(y == 0, F32(1), np.where(y <= -120, F32(0), F32(np.nan))))
        assert np.array_equal(got, v[np.arange(2), j])


def test_pool_bound_holds_for_an_expf_at_its_documented_error():
    r = _rng(5)
    for hd, t in ((64, 729), (88, 1025), (72, 257), (128, 2)):
        k = (r.standard_normal((2, t, hd)) * 1.5).astype(F16)
        v = r.standard_normal((2, t, hd)).astype(F16)
        q = (r.standard_normal((2, hd)) * hd**-0.5).astype(F32)

        def bad_expf(x):  # the correctly rounded value pushed the documented number of ulps, alternating direction
            e = np.exp(x.astype(np.float64)).astype(F32)
            n = (2 + np.floor(1.173 * np.abs(x.astype(np.float64)))).astype(np.int64)
            up = (np.arange(x.size).reshape(x.shape) % 2) == 0
            out = e.copy()
            for step in range(int(n.max(initial=0))):
                m = step < n
                out = np.where(m & up, np.nextafter(out, F32(np.inf)), np.where(m & ~up, np.nextafter(out, F32(0)), out))
            return out

        got = R.pool_f32(k, v, q, expf=bad_expf).astype(np.float64)
        assert np.all(np.abs(got - R.pool_ref(k, v, q)) <= R.pool_bound(k, v, q))


# ------------------------------------------------------------------------------------------------ the rules reject wrong kernels
def _ln_inputs(rows: int, d: int, seed: int, mean: float = 1.0):
    r = _rng(seed)
    x = (r.standard_normal((rows, d)) * 3 + mean).astype(F32)
    gamma = (r.random(d) * 1.45 + 0.05).astype(F32)
    beta = r.standard_normal(d).astype(F32)
    return x, gamma, beta


def _unmatched_ln(got16: np.ndarray, x, gamma, beta, eps=1e-5) -> int:
    mean, arg = R.ln_stats(x, eps)
    off, _ = R.match_rows(got16, arg, lambda r: R.ln_apply(x, mean, r, gamma, beta).astype(F16))
    return int((off == 99).sum())


def _wrong_ln(x, gamma, beta, variant, eps=1e-5, d_eps=None):
    """A LayerNorm kernel with a wrong formula, rounded exactly as the real one (correctly rounded rstd)."""
    mean, arg = R.ln_stats(x, d_eps if d_eps is not None else eps, "kernel" if variant == "eps" else variant)
    r = R.rsqrt_rn(arg)
    if variant == "eps_outside":  # 1 / (sqrt(var) + eps)
        r = (F32(1) / (np.sqrt(arg) + F32(eps))).astype(F32)
    return R.ln_apply(x, mean, r, gamma, beta).astype(F16)


@pytest.mark.parametrize("d", [256, 1024, 1536])
def test_acceptance_accepts_the_kernel_formula(d):
    x, gamma, beta = _ln_inputs(64, d, d)
    mean, arg = R.ln_stats(x, 1e-5)
    for k, r in R.rstd_candidates(arg):
        assert _unmatched_ln(R.ln_apply(x, mean, r, gamma, beta).astype(F16), x, gamma, beta) == 0, k


@pytest.mark.parametrize(("variant", "mean", "d_eps"), [("unbiased", 1.0, None), ("eps_outside", 1.0, None), ("eps", 1.0, 1e-6),
                                                        ("one_pass", 1e3, None)])  # fmt: skip
@pytest.mark.parametrize("d", [768, 1024, 1152])
def test_acceptance_rejects_wrong_layernorms(variant, mean, d_eps, d):
    x, gamma, beta = _ln_inputs(64, d, d + 1, mean)
    if variant == "eps":  # eps only shows on rows whose variance is near it: the GPU tests' small-row class
        x[::2] = (x[::2] - x[::2].mean(1, keepdims=True)) * F32(1e-3)
    got = _wrong_ln(x, gamma, beta, variant, d_eps=d_eps)
    assert _unmatched_ln(got, x, gamma, beta) > 0


def test_acceptance_rejects_gamma_and_beta_swapped():
    x, gamma, beta = _ln_inputs(32, 1024, 9)
    mean, arg = R.ln_stats(x, 1e-5)
    got = R.ln_apply(x, mean, R.rsqrt_rn(arg), beta, gamma).astype(F16)
    assert _unmatched_ln(got, x, gamma, beta) == 32


def test_acceptance_rejects_rmsnorm_with_mean_subtraction():
    r = _rng(11)
    x = (r.standard_normal((32, 1408)) + 0.5).astype(F32)
    w = (r.random(1408) + 0.5).astype(F32)
    wrong = R.rms_apply(x, R.rsqrt_rn(R.rms_stats(x, 1e-6, "centred")), w).astype(F16)
    off, _ = R.match_rows(wrong, R.rms_stats(x, 1e-6), lambda rr: R.rms_apply(x, rr, w).astype(F16))
    assert (off == 99).all()


@pytest.mark.parametrize("mistake", ["no_scale", "scale_twice"])
def test_pool_bound_rejects_clip_pool_scale_mistakes(mistake):
    r = _rng(13)
    hd, t = 88, 1025
    k = (r.standard_normal((2, t, hd)) * 1.5).astype(F16)
    v = r.standard_normal((2, t, hd)).astype(F16)
    q = r.standard_normal((2, hd)).astype(F32)
    scale = F32(1) / np.sqrt(F32(hd))
    qh = (q * scale).astype(F32)
    wrong_q = q if mistake == "no_scale" else (qh * scale).astype(F32)
    got = R.pool_f32(k, v, wrong_q).astype(np.float64)
    assert np.any(np.abs(got - R.pool_ref(k, v, qh)) > R.pool_bound(k, v, qh))


def test_token_mean_rejects_dividing_by_t_minus_1():
    h = _rng(17).standard_normal((2, 257, 256)).astype(F32)
    assert not np.array_equal(R.token_mean_f32(h, -1), R.token_mean_f32(h))
    assert np.allclose(R.token_mean_f32(h), h.astype(np.float64).mean(1), atol=1e-6)


@pytest.mark.parametrize("order", ["cxy", "yxc"])
def test_tube_patches_rejects_other_k_orders(order):
    tubes = _rng(19).standard_normal((2, 3, 28, 28)).astype(F32)
    want = R.tube_patches_f32(tubes, 14, 592)
    assert want[0, 1, 5] == F16(tubes[0, 0, 0, 14 + 5])  # patch (0, 1), k = (c 0, y 0, x 5)
    assert not np.array_equal(R.tube_patches_f32(tubes, 14, 592, order), want)


def test_assemble_rejects_pos_shifted_by_one():
    r = _rng(23)
    n, g2, d = 2, 49, 256
    patch, cls, pos = (r.standard_normal(s).astype(F32) for s in ((n * g2, d), (d,), (g2 + 1, d)))
    good, _ = R.assemble_f32(patch, cls, pos, None, None, None, 1e-5, n, g2 + 1, g2)
    bad, _ = R.assemble_f32(patch, cls, pos, None, None, None, 1e-5, n, g2 + 1, g2, pos_shift=-1)
    assert not np.array_equal(good, bad)


def test_old_layernorm_tolerance_accepts_four_wrong_layernorms():
    """test_gpu_ops.py::test_layernorm compares with rtol = atol = 2e-3 on randn * 3 + 1 rows.  These wrong LayerNorms, rounded to
    fp16 as the kernel's output is, put at most one element in ten thousand outside that tolerance at d = 1024, 768 and 1152 (on the
    GPU test's own inputs, none at all), so whether the old test notices them is down to its seed.  The same four formulas rounded as
    the kernel would round them are rejected by the exact rule (one-pass variance on rows whose mean dominates, where it goes wrong),
    which accepts the kernel's own formula on the same rows."""
    g = torch.Generator().manual_seed(4)
    for rows, d in ((1000, 1024), (77, 768), (513, 1152)):
        x = torch.randn(rows, d, generator=g) * 3 + 1
        gamma, beta = torch.randn(d, generator=g), torch.randn(d, generator=g)
        want = torch.nn.functional.layer_norm(x, (d,), gamma, beta, 1e-5)
        xd, mu = x.double(), x.double().mean(1, keepdim=True)
        wrong = {
            "unbiased": (xd - mu) / (xd.var(1, unbiased=True, keepdim=True) + 1e-5).sqrt(),
            "no_eps": (xd - mu) / xd.var(1, unbiased=False, keepdim=True).sqrt(),
            "eps_1e-3": (xd - mu) / (xd.var(1, unbiased=False, keepdim=True) + 1e-3).sqrt(),
            "one_pass": (xd - mu) / ((x**2).mean(1, keepdim=True) - x.mean(1, keepdim=True) ** 2 + 1e-5).double().sqrt(),
        }
        for name, y in wrong.items():
            got = (y * gamma.double() + beta.double()).half().float()
            outside = ((got - want).abs() > 2e-3 + 2e-3 * want.abs()).sum().item()
            assert outside <= got.numel() // 10000, f"{name} at d={d}: {outside} elements outside the old tolerance"
        x32, g32, b32 = x.numpy(), gamma.numpy(), beta.numpy()
        mean, arg = R.ln_stats(x32, 1e-5)
        assert _unmatched_ln(R.ln_apply(x32, mean, R.rsqrt_rn(arg), g32, b32).astype(F16), x32, g32, b32) == 0, f"control at d={d}"
        kernel_rounded = {"unbiased": ("unbiased", None), "no_eps": ("eps", 0.0), "eps_1e-3": ("eps", 1e-3), "one_pass": ("one_pass", None)}
        for name, (variant, d_eps) in kernel_rounded.items():
            # one-pass variance in float32 only drifts past the rsqrtf window when the mean dominates: rows shifted by 1e3, as in the
            # GPU test's mean >> sigma class
            xv = (x32 + np.float32(1e3)).astype(F32) if variant == "one_pass" else x32
            assert _unmatched_ln(_wrong_ln(xv, g32, b32, variant, d_eps=d_eps), xv, g32, b32) > 0, f"{name} at d={d}: the exact rule accepted it"
