"""CPU: the semantic-dedup oracle against brute force (the reference's CuPy/cuML arithmetic cannot run here: parity with the
reference itself is unpinned, see oracle/dedup.py), and the host-side surface of the product module."""

from __future__ import annotations

import numpy as np
import pytest

from oracle import dedup as od


def _brute(ids, emb, dist, eps):
    order = sorted(range(len(ids)), key=lambda i: (-np.float32(dist[i]), i))
    e = np.asarray(emb, np.float32)[order]
    e = e / np.maximum(np.linalg.norm(e, axis=1, keepdims=True), 1e-12).astype(np.float32)
    m = len(order)
    maxv, arg = np.full(m, -1.0, np.float32), np.full(m, -1, np.int64)
    for j in range(m):
        for i in range(j):
            s = np.float32(min(1.0, max(-1.0, float(np.dot(e[i], e[j])))))
            if s > maxv[j]:
                maxv[j], arg[j] = s, i
    if m:
        maxv[0], arg[0] = 0.0, 0
    arg = np.where(arg < 0, 0, arg)
    sid = np.asarray(ids)[order]
    return sid, sid[arg], maxv, int((maxv <= np.float32(1 - eps)).sum())


@pytest.mark.parametrize("m", [1, 2, 7, 130])
def test_pairwise_max_matches_brute_force(m):
    rng = np.random.default_rng(m)
    emb = rng.standard_normal((m, 32)).astype(np.float32)
    if m > 5:
        emb[5] = emb[1]  # exact duplicate
        emb[6] = 3.0 * emb[1]  # duplicate up to scale
    dist = rng.random(m).astype(np.float32)
    if m > 3:
        dist[3] = dist[2]  # tie in the sort key: stable order
    ids = np.array([f"clip-{i}" for i in range(m)])
    r = od.pairwise_max(ids, emb, dist, eps=0.05)
    sid, mid, mv, kept = _brute(ids, emb, dist, 0.05)
    assert list(r["id"]) == list(sid)
    np.testing.assert_allclose(r["cosine_sim_score"], mv, atol=2e-6)
    # where the chosen neighbour differs it must be an fp32 near-tie (matmul vs dot summation order), e.g. among duplicates
    e = r["sim_matrix_unit"]
    pos = {v: k for k, v in enumerate(r["id"])}
    for j in np.flatnonzero(r["max_id"] != mid):
        assert abs(float(e[pos[r["max_id"][j]]] @ e[j]) - float(e[pos[mid[j]]] @ e[j])) < 2e-6
    assert r["total"] == m and abs(r["kept"] - kept) <= 1


def test_pairwise_duplicates_are_pruned_and_first_index_wins():
    base = np.eye(16, dtype=np.float32)[:4]
    emb = np.concatenate([base, base[[2]], base[[2]]])  # rows 4 and 5 duplicate row 2
    dist = np.array([0.9, 0.8, 0.7, 0.6, 0.5, 0.4], np.float32)  # already descending
    r = od.pairwise_max(np.arange(6), emb, dist, eps=0.01)
    assert list(r["max_id"][4:]) == [2, 2]  # not 4: the first of the equal maxima
    np.testing.assert_allclose(r["cosine_sim_score"][4:], 1.0)
    assert r["kept"] == 4 and r["total"] == 6
    assert r["cosine_sim_score"][0] == 0.0 and r["max_id"][0] == 0
    # orthogonal rows: similarity 0 > -1 -> index of the first earlier row
    assert list(r["max_id"][1:4]) == [0, 0, 0]


def test_assign_is_nearest_centroid():
    rng = np.random.default_rng(3)
    x = od.l2_normalize(rng.standard_normal((500, 24)))
    c = rng.standard_normal((9, 24)).astype(np.float32) * 0.7
    labels, cd = od.assign(x, c)
    d2 = ((x[:, None, :] - c[None]) ** 2).sum(-1)
    assert np.array_equal(labels, d2.argmin(1))
    cu = c / np.linalg.norm(c, axis=1, keepdims=True)
    np.testing.assert_allclose(cd, 1 - (x * cu[labels]).sum(1), atol=1e-6)


def test_product_module_imports_without_a_gpu():
    import cosmos_curate_b200.dedup as pd

    assert callable(pd.semdedup_cluster) and callable(pd.spherical_kmeans) and callable(pd.rowdot_argmax)


def _check_against_reference_golden(name, g, got_maxv, got_arg_pos):
    """got_* in the sorted order the reference works in; arg-max compared where the decision is not a float near-tie."""
    maxv, argi = g[name + "_maxv"], g[name + "_argi"]
    np.testing.assert_allclose(got_maxv, maxv, rtol=0, atol=3e-6)
    e = od.l2_normalize(g[name + "_emb"][np.argsort(-g[name + "_dist"], kind="stable")])
    argi0 = np.where(argi < 0, 0, argi)
    differ = np.flatnonzero(got_arg_pos != argi0)
    for j in differ:  # a different row may only be chosen if it is an equally good (within fp32 summation noise) earlier row
        assert got_arg_pos[j] < j and abs(float(e[got_arg_pos[j]] @ e[j]) - float(e[argi0[j]] @ e[j])) < 3e-6, j
    assert len(differ) <= max(1, len(maxv) // 200)


@pytest.mark.parametrize("name", ["multi_tile", "default_tile", "tiny"])
def test_oracle_pinned_to_reference_executed_dedup(name):
    """oracle/dedup.pairwise_max against the reference's OWN dedup array code (dedup_actor.py:404-466, run from its source with
    numpy standing in for cupy, oracle/ref_import.dedup_core -> tests/golden/dedup_ref.npz): start values, strict `>` across
    tiles, first arg-max inside a tile, the tril mask of the diagonal tile, clip, the legacy row-0 convention."""
    from conftest import load_golden

    g = load_golden("dedup_ref.npz")
    emb, dist = g[name + "_emb"], g[name + "_dist"]
    ids = np.arange(len(emb))
    r = od.pairwise_max(ids, emb, dist, eps=0.01)
    order = np.argsort(-dist, kind="stable")
    pos = {int(i): k for k, i in enumerate(order)}
    got_arg = np.array([pos[int(i)] for i in r["max_id"]])
    assert np.array_equal(r["id"], ids[order])
    _check_against_reference_golden(name, g, r["cosine_sim_score"], got_arg)
    thr = np.float32(0.99)
    safe = np.abs(g[name + "_maxv"] - thr) > 1e-5
    assert np.array_equal((r["cosine_sim_score"] <= thr)[safe], (g[name + "_maxv"] <= thr)[safe])


# ------------------------------------------------------------------------------------------------ the exact oracle of csrc/dedup.cu
def _fp32_chain(a, b, bias, rev: bool) -> np.ndarray:
    """a_i . b_j (+ bias_i) as an fp32 loop over k, every step rounded to fp32 (forward, or backward)."""
    acc = np.zeros((len(a), len(b)), np.float32)
    for k in range(a.shape[1])[:: -1 if rev else 1]:
        acc = (acc + a[:, k, None] * b[None, :, k]).astype(np.float32)
    return acc if bias is None else (acc + bias[:, None]).astype(np.float32)


@pytest.mark.parametrize(("na", "nb", "d"), [(130, 40, 16), (70, 33, 48), (9, 7, 1024), (4, 5, 4096)])
def test_dyadic_scores_are_exact_in_fp32(na, nb, d):
    """On dyadic inputs the float64 reference equals fp32 arithmetic bit for bit in any summation order: what lets the GPU suite
    compare the kernel's values and indices with rowdot_reference exactly."""
    rng = np.random.default_rng(d + na)
    a, b, bias = od.dyadic_rows(na, d, rng), od.dyadic_rows(nb, d, rng), od.dyadic_bias(na, rng)
    if d == 4096:
        a[0], b[0] = 1.0, -1.0  # the largest partial sums the generator allows
    for bv in (None, bias):
        s64 = od.rowdot_scores(a, b, bv)
        for rev in (False, True):
            s32 = _fp32_chain(a, b, bv, rev)
            assert np.array_equal(s32.astype(np.float64), s64)
    # brute-force first arg-max over the fp32 scores (strict '>' from init_val, rows in ascending order)
    for clip, init in ((False, -np.inf), (True, -1.0), (True, 0.0)):
        s32 = _fp32_chain(a, b, bias, False)
        if clip:
            s32 = np.clip(s32, -1, 1)
        want_v, want_i = od.rowdot_reference(a, b, bias, clip=clip, init_val=init)
        for j in range(nb):
            bv_, bi_ = init, -1
            for i in range(na):
                if s32[i, j] > bv_:
                    bv_, bi_ = s32[i, j], i
            assert (want_v[j], want_i[j]) == (bv_, bi_), j


def test_rowdot_reference_edges():
    a = np.array([[1, 0], [-1, 0], [1, 0], [2, 0]], np.float64)
    v, i = od.rowdot_reference(a, a, upper=True, clip=True, init_val=-1.0)
    assert list(i) == [-1, -1, 0, 0] and list(v) == [-1.0, -1.0, 1.0, 1.0]  # column 0 has no candidate; antipodal -1 is not > -1
    v, i = od.rowdot_reference(a, a, upper=True, init_val=-np.inf)
    assert list(i) == [-1, 0, 0, 0] and v[0] == -np.inf and list(v[1:]) == [-1.0, 1.0, 2.0]
    v, i = od.rowdot_reference(np.zeros((0, 2)), a, init_val=0.5)
    assert list(i) == [-1] * 4 and list(v) == [0.5] * 4


@pytest.mark.parametrize("name", ["multi_tile", "default_tile", "tiny"])
def test_rowdot_reference_is_pairwise_max_on_the_goldens(name):
    """rowdot_reference(UPPER, CLIP, init -1) on the normalised, sorted rows is pairwise_max's column loop: the scores within the fp32
    bound of pairwise_max's float32 matmul, the index equal wherever the decision is not inside that bound."""
    from conftest import load_golden

    g = load_golden("dedup_ref.npz")
    emb, dist = g[name + "_emb"], g[name + "_dist"]
    r = od.pairwise_max(np.arange(len(emb)), emb, dist, eps=0.01)
    e = r["sim_matrix_unit"]
    v, i = od.rowdot_reference(e, e, upper=True, clip=True, init_val=-1.0)
    v[0], i[0] = 0.0, 0
    i = np.where(i < 0, 0, i)
    bnd = od.rowdot_bound(e, e)
    cols = np.arange(len(e))
    assert np.all(np.abs(v - r["cosine_sim_score"]) <= bnd[i, cols] + bnd.max(0))
    got = np.array([{int(x): k for k, x in enumerate(r["id"])}[int(x)] for x in r["max_id"]])
    s = od.rowdot_scores(e, e, upper=True, clip=True)
    for j in np.flatnonzero(got != i):
        assert abs(s[got[j], j] - s[i[j], j]) <= bnd[got[j], j] + bnd[i[j], j], j
    assert (got != i).mean() <= 0.005


@pytest.mark.parametrize("m", [8, 130, 700])
def test_rowdot_reference_is_pairwise_max_on_unit_exact_rows(m):
    rng = np.random.default_rng(m)
    emb = od.unit_exact_rows(m, 72, rng)
    dist = (rng.integers(0, 5, m) / 4).astype(np.float32)  # sort-key ties
    r = od.pairwise_max(np.arange(m), emb, dist, eps=0.25)
    e = r["sim_matrix_unit"]
    assert np.array_equal(np.abs(e[e != 0]) * 16 % 4, np.zeros(np.count_nonzero(e)))  # +-1/2 or +-1/4 exactly
    v, i = od.rowdot_reference(e, e, upper=True, clip=True, init_val=-1.0)
    v[0], i[0] = 0.0, 0
    assert np.array_equal(v.astype(np.float32), r["cosine_sim_score"])
    assert np.array_equal(r["id"][np.where(i < 0, 0, i)], r["max_id"])
    if m > 100:
        assert np.any(r["cosine_sim_score"] == np.float32(0.75)) and np.any(r["cosine_sim_score"] == 1.0)


@pytest.mark.parametrize("n", [1, 64, 65, 129, 301, 1000])
def test_planted_ties_are_where_they_are_claimed(n):
    rng = np.random.default_rng(n)
    d, nb = 48, 257
    a, bias, b, planted = od.plant_ties(od.dyadic_rows(n, d, rng), od.dyadic_bias(n, rng), od.dyadic_rows(nb, d, rng), rng)
    names = {name for name, _, _ in planted}
    want = {name for name, pos in od.TIE_GROUPS if sum(p < n for p in pos) >= 2}
    assert names == want
    slots = {name: [od.tile_slot(p) for p in pos] for name, pos, _ in planted}
    if "same_thread" in slots:
        (t0, ty0, r0), (t1, ty1, r1) = slots["same_thread"]
        assert t0 == t1 and ty0 == ty1 and r1 == r0 + 4
    if "ty_groups" in slots:
        (t0, ty0, _), (t1, ty1, _) = slots["ty_groups"]
        assert t0 == t1 and ty0 > ty1  # the first copy sits in the later reduction slot
    if "halves" in slots:
        assert [r >> 2 for _, _, r in slots["halves"]] == [0, 1]
    if "row_tiles" in slots:
        assert len({t for t, _, _ in slots["row_tiles"]}) == len(slots["row_tiles"])
    v, i = od.rowdot_reference(a, b, bias)
    s = od.rowdot_scores(a, b, bias)
    for g, (_name, pos, cols) in enumerate(planted):
        assert cols == od.tie_columns(g, nb) and {c >= 64 for c in cols} == {False, True}  # both tx halves of a column tile
        for j in cols:
            assert np.all(s[list(pos), j] == v[j]) and i[j] == pos[0] and np.count_nonzero(s[:, j] == v[j]) == len(pos)
    assert not planted or max(c for _, _, cols in planted for c in cols) == nb - 1  # the partial last column tile
    if n > 300:  # under UPPER (b = a), each later copy's column ties on every earlier copy
        _, iu = od.rowdot_reference(a, a, bias, upper=True)
        for _, pos, _ in planted:
            assert all(iu[p] == pos[0] for p in pos[1:])


def test_cluster_sums_sequential_is_a_left_to_right_fp32_sum():
    rng = np.random.default_rng(4)
    x = (rng.standard_normal((60, 5)) * 10 ** rng.uniform(-3, 3, (60, 1))).astype(np.float32)
    order = rng.permutation(60)
    seg = np.array([0, 7, 7, 30, 31, 55])
    sums0 = rng.standard_normal((5, 5)).astype(np.float32)
    got = od.cluster_sums_sequential(x, order, seg, sums0)
    for c in range(5):
        rows = np.concatenate([np.zeros((1, 5), np.float32), x[order[seg[c] : seg[c + 1]]]])
        assert np.array_equal(got[c], sums0[c] + np.add.accumulate(rows, axis=0, dtype=np.float32)[-1])
    assert np.array_equal(got[1], sums0[1])  # empty
    assert not np.array_equal(got[2], (sums0[2] + x[order[7:30]].sum(0, dtype=np.float64)).astype(np.float32))  # the order is observable
