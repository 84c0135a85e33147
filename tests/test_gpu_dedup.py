"""GPU: fused cosine arg-max kernel, per-cluster semantic dedup and k-means against the numpy oracle."""

from __future__ import annotations

import os

import numpy as np
import pytest
import torch

from gpu_helpers import ctx  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize(("na", "nb", "d", "upper", "clip", "bias"), [(300, 300, 64, True, True, False), (1000, 77, 48, False, False, True),
                                                                      (129, 513, 16, False, True, False), (2500, 2500, 768, True, True, False),
                                                                      (5, 1000, 32, False, False, True), (1, 1, 16, True, True, False)])
def test_rowdot_argmax(ctx, na, nb, d, upper, clip, bias):  # noqa: F811
    from cosmos_curate_b200 import dedup

    g = torch.Generator(device="cuda").manual_seed(na * 3 + nb)
    a = torch.randn(na, d, device="cuda", generator=g)
    a /= a.norm(dim=1, keepdim=True)
    if na > 40:
        a[37] = a[11]  # exact ties: the first index must win
    b = a if upper else torch.randn(nb, d, device="cuda", generator=g)
    bv = torch.randn(na, device="cuda", generator=g) * 0.1 if bias else None
    val, idx = dedup.rowdot_argmax(a, b, bias=bv, upper=upper, clip=clip, init_val=-1.0 if upper else float("-inf"), ctx=ctx)
    s = a.double() @ b.double().T
    if bv is not None:
        s += bv.double()[:, None]
    if clip:
        s = s.clamp(-1, 1)
    if upper:
        s = torch.where(torch.arange(na, device="cuda")[:, None] < torch.arange(nb, device="cuda")[None, :], s, torch.full_like(s, -np.inf))
    want_v, want_i = s.max(dim=0)
    has = torch.isfinite(want_v) & (want_v > (-1.0 if upper else -np.inf))
    assert torch.equal(idx[~has], torch.full_like(idx[~has], -1))
    np.testing.assert_allclose(val[has].cpu().numpy(), want_v[has].cpu().numpy(), atol=3e-6)
    # index: equal, or a near-tie (the value at the returned index is within fp32 noise of the maximum), and never a LATER equal
    if has.any():
        got_at = s[idx[has].long(), torch.arange(nb, device="cuda")[has]]
        assert (want_v[has] - got_at).abs().max().item() <= 3e-6
    if na > 40 and not bias:
        cols = (want_i == 11) | (want_i == 37)
        assert not (idx[cols & has] == 37).any()  # rows 11 and 37 are bitwise equal: the kernel must report 11


def test_semdedup_cluster_matches_oracle(ctx):  # noqa: F811
    from cosmos_curate_b200 import dedup
    from oracle import dedup as od

    rng = np.random.default_rng(5)
    m, d = 3000, 768
    centers = rng.standard_normal((40, d)).astype(np.float32)
    emb = centers[rng.integers(0, 40, m)] + 0.15 * rng.standard_normal((m, d)).astype(np.float32)  # tight groups: many near-duplicates
    emb[100] = emb[7]
    emb[2000] = 2.5 * emb[7]
    ids = np.array([f"{i:08x}" for i in range(m)])
    dist = rng.random(m).astype(np.float32)
    for eps in (0.01, 0.05):
        got = dedup.semdedup_cluster(ids, emb, dist, eps, ctx=ctx)
        want = od.pairwise_max(ids, emb, dist, eps)
        assert list(got["id"]) == list(want["id"])
        np.testing.assert_allclose(got["cosine_sim_score"], want["cosine_sim_score"], atol=3e-6)
        diff = got["max_id"] != want["max_id"]
        assert diff.mean() < 0.01  # fp32 near-ties only
        thr = np.float32(1 - eps)
        decisive = np.abs(want["cosine_sim_score"] - thr) > 1e-5
        assert np.array_equal((got["cosine_sim_score"] <= thr)[decisive], (want["cosine_sim_score"] <= thr)[decisive])
        assert abs(got["kept"] - want["kept"]) <= int((~decisive).sum()) and got["total"] == m
        assert 0 < got["kept"] < m
    # the exact duplicate and the scaled duplicate point at the earliest of their group with similarity 1
    pos = {v: k for k, v in enumerate(got["id"])}
    later = max(pos[ids[7]], pos[ids[100]], pos[ids[2000]])
    assert got["cosine_sim_score"][later] > 0.999999


def test_kmeans_properties_and_determinism(ctx):  # noqa: F811
    from cosmos_curate_b200 import dedup
    from oracle import dedup as od

    rng = np.random.default_rng(8)
    k, d, n = 12, 80, 5000  # d = 80 is a multiple of 16: no padding (test_gpu_dedup_exact.py runs the pad-to-16 path at d = 72)
    centers = rng.standard_normal((k, d)).astype(np.float32)
    x = centers[rng.integers(0, k, n)] + 0.3 * rng.standard_normal((n, d)).astype(np.float32)
    r1 = dedup.spherical_kmeans(x, k, max_iter=50, seed=4, ctx=ctx)
    r2 = dedup.spherical_kmeans(x, k, max_iter=50, seed=4, ctx=ctx)
    assert torch.equal(r1["centroids"], r2["centroids"]) and torch.equal(r1["labels"], r2["labels"])  # bit-reproducible
    cent = r1["centroids"].cpu().numpy()
    xu = od.l2_normalize(x)
    labels, cd = od.assign(xu, cent)
    got_l = r1["labels"].cpu().numpy()
    assert (labels == got_l).mean() > 0.999
    np.testing.assert_allclose(r1["cosine_dist_to_cent"].cpu().numpy()[labels == got_l], cd[labels == got_l], atol=2e-6)
    if r1["n_iter"] < 50:  # converged: centroids are the means of their members
        for c in range(k):
            if (got_l == c).sum() > 0:
                np.testing.assert_allclose(cent[c], xu[got_l == c].mean(0), atol=2e-3)
    assert len(np.unique(got_l)) >= k - 4  # plain Lloyd from a random subset may leave a few clusters merged or empty


def _rank_main(rank, world, port, x, k, out):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cosmos_curate_b200 import dedup

    shard = x[rank::world] if rank else x[0::world]
    r = dedup.spherical_kmeans(shard, k, max_iter=15, seed=1, tol=0.0, group=dist.group.WORLD)
    if rank == 0:
        np.save(out, r["centroids"].cpu().numpy())
    dist.destroy_process_group()


def test_kmeans_two_ranks_match_one_rank(ctx):  # noqa: F811
    """Two processes (gloo all_reduce of the centroid sums) on shards == one process on the union with the same initial centroids."""
    import socket

    import torch.multiprocessing as mp

    from cosmos_curate_b200 import dedup

    rng = np.random.default_rng(2)
    k, d, n = 6, 32, 1200
    centers = rng.standard_normal((k, d)).astype(np.float32)
    x = centers[rng.integers(0, k, n)] + 0.2 * rng.standard_normal((n, d)).astype(np.float32)
    # rank 0 seeds the centroids from ITS shard: give the single-process run the same rows first
    x_union = np.concatenate([x[0::2], x[1::2]])
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    import tempfile

    out = os.path.join(tempfile.mkdtemp(), "centroids.npy")  # no mp.Manager: it would fork() this multi-threaded CUDA process
    mp.spawn(_rank_main, args=(2, port, x, k, out), nprocs=2, join=True)
    # single process: same init (seeded permutation over rank 0's shard size) is reproduced by running on rank 0's shard
    # for the init and on the union for the iterations
    n0 = len(x[0::2])
    perm = torch.randperm(n0, generator=torch.Generator().manual_seed(1))[:k]
    xu = torch.from_numpy(x_union).cuda()
    dedup.l2_normalize_rows_(xu, ctx)
    cent = xu[:n0][perm.cuda()].clone()
    for _ in range(15):
        bias = (-0.5 * (cent * cent).sum(1)).contiguous()
        _, labels = dedup.rowdot_argmax(cent, xu, bias=bias, ctx=ctx)
        sums = torch.zeros_like(cent).index_add_(0, labels.long(), xu)
        cnt = torch.bincount(labels.long(), minlength=k).float()
        cent = torch.where(cnt[:, None] > 0, sums / cnt.clamp(min=1)[:, None], cent)
    np.testing.assert_allclose(np.load(out), cent.cpu().numpy(), atol=1e-5)


@pytest.mark.parametrize("name", ["multi_tile", "default_tile", "tiny"])
def test_semdedup_cluster_vs_reference_executed_golden(ctx, name):  # noqa: F811
    """The CUDA path against outputs of the REFERENCE's own dedup array code (dedup_actor.py:404-466 executed from its source with
    numpy standing in for cupy - tests/golden/dedup_ref.npz, oracle/ref_import.dedup_core)."""
    from conftest import load_golden
    from cosmos_curate_b200 import dedup
    from oracle import dedup as od

    g = load_golden("dedup_ref.npz")
    emb, dist = g[name + "_emb"], g[name + "_dist"]
    ids = np.arange(len(emb))
    r = dedup.semdedup_cluster(ids, emb, dist, eps=0.01, ctx=ctx)
    order = np.argsort(-dist, kind="stable")
    assert np.array_equal(r["id"], ids[order])
    np.testing.assert_allclose(r["cosine_sim_score"], g[name + "_maxv"], rtol=0, atol=3e-6)
    pos = {int(i): k for k, i in enumerate(order)}
    got = np.array([pos[int(i)] for i in r["max_id"]])
    want = np.where(g[name + "_argi"] < 0, 0, g[name + "_argi"])
    e = od.l2_normalize(emb[order])
    differ = np.flatnonzero(got != want)
    for j in differ:
        assert got[j] < j and abs(float(e[got[j]] @ e[j]) - float(e[want[j]] @ e[j])) < 3e-6
    assert len(differ) <= max(1, len(want) // 200)
    thr = np.float32(0.99)
    safe = np.abs(g[name + "_maxv"] - thr) > 1e-5
    assert int((r["cosine_sim_score"][safe] <= thr).sum()) == int((g[name + "_maxv"][safe] <= thr).sum())
