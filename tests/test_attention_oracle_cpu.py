"""The attention oracle (oracle/attention.py) is well-posed: the float64 reference is softmax attention, the structured inputs have
the exact answers the GPU tests assert bit for bit, the error bound holds with room to spare for a model of the kernels' rounding,
and the dispatch table says what cb_attention_f16's rules say."""

from __future__ import annotations

import pytest
import torch

from oracle import attention as A

SWEEP_T, SWEEP_HD = A.SWEEP_T, A.SWEEP_HD


def test_reference_matches_sdpa_in_float64():
    qkv = A.random_inputs(2, 37, 3, 24, seed=1)
    ref, s_abs = A.reference(qkv, 3)
    q, k, v = (x.double() for x in A.split_heads(qkv, 3))
    want = A.merge_heads(torch.nn.functional.scaled_dot_product_attention(q, k, v))
    torch.testing.assert_close(ref, want, rtol=1e-13, atol=1e-13)
    assert (s_abs >= ref.abs() - 1e-12).all()


def _p_max(qkv, heads):
    q, k, _ = (x.double() for x in A.split_heads(qkv, heads))
    return torch.softmax(q @ k.transpose(-1, -2) / q.shape[-1] ** 0.5, dim=-1).amax(dim=-1)


@pytest.mark.parametrize("t", SWEEP_T)
def test_selection_is_one_hot(t):
    for hd in SWEEP_HD:
        qkv, pi = A.selection_inputs(2, t, 2, hd, seed=t + hd)
        assert _p_max(qkv, 2).min().item() >= 1 - 1e-8, hd
        ref, _ = A.reference(qkv, 2)
        _, _, v = A.split_heads(qkv, 2)
        want = A.merge_heads(torch.gather(v, 2, pi[..., None].expand(-1, -1, -1, hd)))
        assert torch.equal(torch.from_numpy(A.emulate(qkv.numpy(), 2)), want), hd  # the kernels' rounding gives V[pi(i)] exactly
        torch.testing.assert_close(ref, want.double(), rtol=1e-7, atol=1e-7)
    bnd = A.boundary_tokens(t)
    assert set(pi[0, 0, bnd].tolist()) == set(bnd)
    assert t < 3 or not torch.equal(pi[0, 0], pi[1, 1])


@pytest.mark.parametrize(("t", "hd"), [(1030, 80), (257, 64), (129, 16), (353, 72), (1, 40), (560, 48)])
def test_uniform_gives_the_constant_exactly(t, hd):
    qkv, c = A.uniform_inputs(3, t, 2, hd, seed=t)
    want = A.merge_heads(c[:, :, None, :].expand(3, 2, t, hd)).half()
    assert torch.equal(torch.from_numpy(A.emulate(qkv.numpy(), 2)), want)
    ref, _ = A.reference(qkv, 2)
    torch.testing.assert_close(ref, want.double(), rtol=1e-12, atol=0)  # float64 softmax: 1/T is rounded
    assert len(set(c[:, 0, 0].tolist())) == 3  # a different constant per image


@pytest.mark.parametrize("kind", ["normal", "sharp", "large", "ties"])
def test_emulated_kernel_within_the_bound_with_margin(kind):
    worst = 0.0
    for i, t in enumerate(SWEEP_T):
        for hd in SWEEP_HD:
            qkv = A.random_inputs(1, t, 2, hd, seed=1000 * i + hd, kind=kind)
            ref, s_abs = A.reference(qkv, 2)
            err = (torch.from_numpy(A.emulate(qkv.numpy(), 2)).double() - ref).abs()
            worst = max(worst, (err / A.bound(ref, s_abs, qkv, 2)).max().item())
    print(f"{kind}: worst err/bound of the emulated kernel {worst:.3f}")
    # not 0.5: the fp16 rounding of the output and of P are each attained, and in rows carried by one or two keys both can be near
    # their worst at once (0.56 at T = 32, head_dim 16, normal inputs).  The margin left covers the tensor-core and ex2 roundings the
    # model does not reproduce, whose own terms are in the bound as well.
    assert worst <= 0.7


def test_bound_is_not_vacuous():
    """Dropping one key of 257, or counting one twice, breaks the bound for most elements when the softmax is flat (small logits)."""
    t, hd = 257, 64
    qkv = A.random_inputs(1, t, 4, hd, seed=3)
    qkv[..., : 4 * hd] *= 0.1  # Q
    ref, s_abs = A.reference(qkv, 4)
    bnd = A.bound(ref, s_abs, qkv, 4)
    q, k, v = (x.double() for x in A.split_heads(qkv, 4))
    for w_last in (0.0, 2.0):
        s = q @ k.transpose(-1, -2) / hd**0.5
        e = torch.exp(s - s.amax(dim=-1, keepdim=True))
        e[..., -1] *= w_last
        bad = A.merge_heads((e / e.sum(dim=-1, keepdim=True)) @ v)
        assert ((bad - ref).abs() > bnd).double().mean().item() > 0.5, w_last


def test_dispatch_table_matches_the_rules():
    for t in list(range(1, 1100)) + [2048]:
        for hd in range(0, 100):
            for force in (False, True):
                assert A.table_path(t, hd, force) == A.path_of(t, hd, force), (t, hd, force)
    assert A.path_of(352, 64, True) == "mma64_resident" and A.path_of(353, 64, True) == "mma64_stream"
    assert A.path_of(288, 72) == "mma80_resident" and A.path_of(289, 80) == "mma80_stream"
    assert A.path_of(128, 64) == "mma64_resident" and A.path_of(258, 64) == "mma64_resident"
    for hd in (8, 12, 88):
        assert A.path_of(100, hd) is None


def test_sweep_reaches_every_path():
    hit = {A.path_of(t, hd, force) for t in SWEEP_T for hd in SWEEP_HD for force in (False, True)}
    assert hit == {p.name for p in A.PATHS}
