"""CPU: the shot network's kernel oracle (oracle/transnet_kernels.py) - its dispatch against transnet.cu, the sweep's coverage, the exact
classes, cb_transnet_finalize's packing and BatchNorm fold against the reference's own conv3d + batch_norm, and that the bitwise
acceptance rule rejects near-miss formulas while accepting the kernel's."""

from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import transnet_kernels as K
from oracle import transnetv2 as tn

F32 = np.float32


def _bits(a):
    return np.ascontiguousarray(a, dtype=F32).view(np.int32)


# ------------------------------------------------------------------------------------------------ dispatch and schedule
def test_dispatch_read_from_source_equals_oracle():
    src = K.dispatch_from_source()
    assert K.instantiations_in_source() == set(K.INSTS)
    for cin in range(1, 300):
        for n in range(1, 1100):
            assert src(cin, n) == K.conv_inst(cin, n), (cin, n)


# (stack, block) -> instantiation of the spatial and the temporal conv, and the two Linear layers
EXPECTED = {"s0b0.spatial": (16, 8, 4), "s0b1.spatial": (16, 8, 16), "s1b0.spatial": (16, 8, 16), "s1b1.spatial": (16, 8, 16),
            "s2b0.spatial": (16, 8, 16), "s2b1.spatial": (16, 8, 16), "s0b0.temporal": (4, 4, 8), "s0b1.temporal": (4, 4, 8),
            "s1b0.temporal": (8, 4, 16), "s1b1.temporal": (8, 4, 16), "s2b0.temporal": (8, 8, 16), "s2b1.temporal": (8, 8, 16),
            "proj": (16, 8, 16), "fc1": (16, 8, 16)}  # fmt: skip


@pytest.mark.parametrize("B,T", [(1, 1), (1, 7), (4, 100), (16, 45)])
def test_schedule_launches_map_to_the_expected_instantiations(B, T):
    L = K.schedule(B, T)
    convs = {l["name"]: l for l in L if l["kind"] == "conv"}
    assert {n: K.conv_inst(l["cin"], l["N"]) for n, l in convs.items()} == EXPECTED
    assert set(EXPECTED.values()) == set(K.INSTS)
    assert [l["kind"] for l in L].count("conv") == 14 and len(L) == 25  # one mark_launch per kernel: 25 per batch of windows
    for l in convs.values():
        hw = l["H"] * l["W"]
        assert l["M"] % (hw * (l["T"] if l["mode"] == 2 else 1)) == 0
        assert all(l[k] % 4 == 0 for k in ("in_ld", "in_coff", "out_ld", "out_coff", "w_ld", "z_in_coff", "z_out_coff", "z_w"))
    # the concat row: colour 0..127, similarity 128..255, trunk (stack 2 pooled in place at stride 4864) 256..4863
    pool2 = [l for l in L if l["kind"] == "pool"][2]
    assert (pool2["out"], pool2["out_off"], pool2["out_frame_stride"]) == ("concat", 256, 4864)
    assert 256 + 3 * 6 * 256 == 4864
    sims = [l for l in L if l["kind"] == "simfc"]
    assert [(s["x"], s["out_coff"]) for s in sims] == [("proj", 128), ("hist", 0)]
    assert [l["coff"] for l in L if l["kind"] == "mean"] == [0, 64, 192]


# ------------------------------------------------------------------------------------------------ the sweep's coverage
def test_sweep_reaches_every_instantiation_at_every_boundary_class():
    pts = K.conv_sweep()
    assert {p.inst for p in pts} == set(K.INSTS)
    for inst in K.INSTS:
        mine = [p for p in pts if p.inst == inst]
        bm, bn = K.tile(inst)
        assert {p.M % bm for p in mine} >= set(K.m_classes(inst)), inst
        # the fewest k chunks per tap the dispatch admits (cin 16, or 4 for <16,8,4>: one chunk, two for <4,4,8>) and more
        chunks = {p.cin // inst[2] for p in mine}
        assert min(chunks) == (4 if inst == (16, 8, 4) else 16) // inst[2] and max(chunks) > min(chunks), inst
        assert {p.N % bn for p in mine} >= {0, 4}, inst  # a full last column tile and the narrowest tail
        assert {p.z for p in mine} >= {1, 4} and {p.mode for p in mine} >= {0, 1, 2}, inst
    # both sides of every dispatch boundary
    ns = {(p.cin % 16 == 0, p.N) for p in pts}
    for lo, hi in ((28, 32), (60, 64), (124, 128)):
        assert (True, lo) in ns and (True, hi) in ns
    assert any(p.cin % 16 and p.N >= 128 for p in pts) and any(p.cin % 16 == 0 and p.N >= 128 for p in pts)
    # spatial borders including one-row and one-column frames
    m1 = [p for p in pts if p.mode == 1]
    assert any(p.H == 1 and p.W > 1 for p in m1) and any(p.W == 1 and p.H > 1 for p in m1) and any(p.H == 27 and p.W == 48 for p in m1)
    # every T class, each dilation with taps inside the window and outside it
    m2 = [p for p in pts if p.mode == 2 and p.z == 4]
    assert {p.T for p in m2} >= set(K.T_CLASSES)
    for d in (1, 2, 4, 8):
        assert any(p.T > 2 * d for p in m2) and any(p.T <= d for p in m2), d
    assert {(p.epi, p.relu) for p in pts} >= {("scale", 0), ("scale", 1), ("shift", 0), ("shift", 1), ("none", 0)}  # every epilogue


def test_predict_window_plan_and_stitch_cover_every_frame_once():
    for n in (1, 24, 25, 26, 49, 50, 51, 74, 75, 76, 99, 100, 101, 150, 151, 4 * 50 - 1, 4 * 50 + 49, 1030):
        for mw in (1, 4):
            batches = K.predict_batches(n, mw)
            plan = tn.window_plan(n)
            assert sum(b for _, b, _ in batches) == len(plan)
            dst = []
            for w0, B, T in batches:
                assert all(plan[w0 + b][1] + plan[w0 + b][2] == T for b in range(B)) and B <= mw
                dst += list(K.stitch_targets(B, T, w0, n).values())
            assert sorted(dst) == list(range(n)), n


# ------------------------------------------------------------------------------------------------ exactness and bounds
def _small_points():
    """One small point per (instantiation, mode) of the sweep, so the float32 model runs on every row in about a second each."""
    seen, out = set(), []
    for p in sorted(K.conv_sweep(), key=lambda p: p.M * p.N * p.cin * p.z):
        if (p.inst, p.mode) not in seen and p.M <= 700:
            seen.add((p.inst, p.mode))
            out.append(p)
    return out


def _run(p, kind, seed=0, **kw):
    a = p.args()
    rng = np.random.default_rng(seed)
    inp, w, scale, shift, w_ref = K.conv_inputs(kind, p, a, rng)
    rows = np.arange(p.M)
    got = K.conv_f32(inp, w, scale, shift, a, rows, **kw)
    x = inp.reshape(p.M, a["in_ld"])
    refs, bounds = [], []
    for z in range(p.z):
        c0 = a["in_coff"] + z * a["z_in_coff"]
        acc = K.conv_ref(x[:, c0 : c0 + p.cin], w_ref[z], p.mode, p.T, p.H, p.W, dil=1 << z if a["z_dil_shift"] else 1)
        c = a["out_coff"] + z * a["z_out_coff"] + np.arange(p.N)
        y = K.epilogue_ref(acc, None if scale is None else scale[c], None if shift is None else shift[c], bool(p.relu)).numpy()
        refs.append(y)
        sabs = np.abs(scale[c]) if scale is not None else 1.0
        kk = {0: 1, 1: 9, 2: 3}[p.mode] * p.cin
        bounds.append(K.conv_bound(K.conv_abs_f32(inp, w, a, rows)[:, z], y, sabs, kk))
    return got, np.stack(refs, 1), np.stack(bounds, 1)


@pytest.mark.parametrize("p", _small_points(), ids=lambda p: p.name)
def test_conv_model_exact_class_is_exact_and_random_class_within_bound(p):
    got, ref, _ = _run(p, "exact")
    assert np.array_equal(_bits(got), _bits(ref.astype(F32))), p.name
    assert np.array_equal(got.astype(np.float64), ref)
    got, ref, bound = _run(p, "random")
    err = np.abs(got - ref)
    assert (err <= bound).all(), (p.name, (err / bound).max())


def test_packing_and_bn_fold_equal_conv3d_and_batch_norm():
    """pack() + bn_fold() through a float64 gather-GEMM equal F.conv3d + F.batch_norm on the state dict, within the fold's fp32 rounding."""
    sd = tn.random_state_dict(4)
    P = K.pack(sd)
    rng = np.random.default_rng(1)
    T = 5
    hws = {0: (27, 48), 1: (13, 24), 2: (6, 12)}
    L = {l["name"]: l for l in K.schedule(1, T) if l["kind"] == "conv"}
    for s, b, cin, cin_pad, f, relu in K.blocks():
        H, W = hws[s]
        M = T * H * W
        x = rng.standard_normal((M, cin_pad))
        x[:, cin:] = 0
        sp, tp = dict(L[f"s{s}b{b}.spatial"], M=M, in_ld=cin_pad), L[f"s{s}b{b}.temporal"]
        A = K.conv_gather(x.reshape(-1), sp, 0, np.arange(M))
        mid = A @ P[f"s{s}b{b}.w1"].astype(np.float64)
        w2 = P[f"s{s}b{b}.w2"].reshape(4, 6 * f, f).astype(np.float64)
        y = np.concatenate([K.conv_gather(mid.reshape(-1), dict(tp, M=M), z, np.arange(M)) @ w2[z] for z in range(4)], 1)
        y = y * P[f"s{s}b{b}.scale"] + P[f"s{s}b{b}.shift"]
        # the reference: four (1,3,3) -> (3,1,1) branches, concat, batch_norm
        p = f"SDDCNN.{s}.DDCNN.{b}"
        v = torch.from_numpy(x[:, :cin]).reshape(1, T, H, W, cin).permute(0, 4, 1, 2, 3)
        br = []
        for d in tn.DILATIONS:
            u = F.conv3d(v, torch.from_numpy(sd[f"{p}.Conv3D_{d}.layers.0.weight"]).double(), padding=(0, 1, 1))
            br.append(F.conv3d(u, torch.from_numpy(sd[f"{p}.Conv3D_{d}.layers.1.weight"]).double(), padding=(d, 0, 0), dilation=(d, 1, 1)))
        acc = torch.cat(br, 1)
        g = {k: torch.from_numpy(sd[f"{p}.bn.{k}"]).double() for k in ("running_mean", "running_var", "weight", "bias")}
        ref = F.batch_norm(acc, g["running_mean"], g["running_var"], g["weight"], g["bias"], training=False, eps=1e-3)
        ref = ref.permute(0, 2, 3, 4, 1).reshape(M, 4 * f).numpy()
        accn = acc.permute(0, 2, 3, 4, 1).reshape(M, 4 * f).numpy()
        sc64, sh64 = K.bn_fold(sd, p)[0].astype(np.float64), K.bn_fold(sd, p)[1].astype(np.float64)
        bound = 2 * K.U * (np.abs(sc64 * accn) + np.abs(sh64) + 1) + 1e-9 * (1 + np.abs(ref))
        assert (np.abs(y - ref) <= bound).all(), (p, np.abs(y - ref).max())
    # the Linear layers: [out][in] -> [in][out]
    xin = rng.standard_normal((3, 448))
    np.testing.assert_allclose(xin @ P["proj_wt"], F.linear(torch.from_numpy(xin), torch.from_numpy(sd["frame_sim_layer.projection.weight"]).double()).numpy(), rtol=1e-12, atol=1e-12)
    assert P["fc1_wt"].shape == (4864, 1024) and np.array_equal(P["fc1_wt"], sd["fc1.weight"].T)
    assert P["sim_fc_wt"].shape == (101, 128) and np.array_equal(P["hist_fc_wt"], sd["color_hist_layer.fc.weight"].T)


def test_row_kernel_models_against_float64_references():
    rng = np.random.default_rng(3)
    # window_gather: x0 is the correctly rounded r / 255; the histogram within two roundings (sqrt, division) of float64
    frames = rng.integers(0, 256, (12, 27, 48, 3), dtype=np.uint8)
    frames[3] = 255
    frames[4] = 0
    x0, hist = K.window_gather_f32(frames, [0, 5], [2, 0], 7)
    x0r, histr = K.window_gather_ref(frames, [0, 5], [2, 0], 7)
    assert np.array_equal(x0[..., :3], x0r.astype(F32)) and not x0[..., 3].any()
    assert (np.abs(hist - histr) <= 3 * K.U * histr + 1e-45).all()
    # shortcut_pool and spatial_mean: exact class exact, random class within the bound
    for kind in ("exact", "random"):
        x2, x1 = ((rng.integers(-6, 7, (3, 7, 9, 8)) if kind == "exact" else rng.standard_normal((3, 7, 9, 8))).astype(F32) for _ in range(2))
        got, ref = K.shortcut_pool_f32(x2, x1), K.shortcut_pool_ref(x2, x1)
        if kind == "exact":
            assert np.array_equal(got.astype(np.float64), ref)
        absum = K.shortcut_pool_ref(np.abs(x2), np.abs(x1))
        assert (np.abs(got - ref) <= K.sum_bound(absum, 8, ref)).all()
        x = ((rng.integers(-20, 21, (4, 312, 16)) if kind == "exact" else rng.standard_normal((4, 312, 16))).astype(F32))
        got, ref = K.spatial_mean_f32(x), K.spatial_mean_ref(x)
        if kind == "exact":
            assert np.array_equal(got, ref.astype(F32))
        assert (np.abs(got - ref) <= K.sum_bound(K.spatial_mean_ref(np.abs(x)), 312, ref)).all()
    # l2_normalize_rows, window_similarity_fc, head
    x = rng.standard_normal((18, 128)).astype(F32)
    ref = K.l2_normalize_ref(x)
    assert (np.abs(K.l2_normalize_f32(x) - ref) <= 4 * K.U * np.abs(ref) + 130 * K.U * np.abs(ref)).all()
    xn = K.l2_normalize_f32(x)
    wt = (rng.standard_normal((101, 128)) / 10).astype(F32)
    bias = (rng.standard_normal(128) * 0.05).astype(F32)
    got = K.window_similarity_fc_f32(xn, 9, wt, bias)
    ref, terms = K.window_similarity_fc_ref(xn, 9, wt, bias)
    assert (np.abs(got - ref) <= K.window_similarity_fc_bound(terms, 128, ref, bias)).all()
    h = np.maximum(rng.standard_normal((40, 1024)), 0).astype(F32)
    w = (rng.standard_normal(1024) * 0.06).astype(F32)
    cands = dict(K.head_candidates(h, w, F32(-4.75)))
    ref = K.head_ref(h, w, -4.75)
    terms = np.abs(h.astype(np.float64)) @ np.abs(w.astype(np.float64))
    assert (np.abs(cands[0] - ref) <= ref * (1 - ref) * (1100 * K.U * terms + 8 * K.U) + 4 * K.U * ref).all()
    assert (K.head_match(cands[0], list(cands.items())) == 0).all()
    m = K.head_match(cands[1], list(cands.items()))  # candidates may coincide after 1 + e rounds: the nearest offset that fits is named
    assert ((m == 0) | (m == 1)).all() and (m == 1).any()


# ------------------------------------------------------------------------------------------------ the acceptance rule's power
def test_acceptance_rule_rejects_wrong_formulas_and_accepts_the_kernels():
    rng = np.random.default_rng(11)
    # BN epilogue: mul + add rounded twice instead of fmaf
    p = K.ConvPoint(32, 16, 3 * 9 * 6, 2, T=9, H=2, W=3, z=4, epi="scale")
    a = p.args()
    inp, w, sc, sh, _ = K.conv_inputs("random", p, a, rng)
    rows = np.arange(p.M)
    good = K.conv_f32(inp, w, sc, sh, a, rows)
    assert not np.array_equal(_bits(K.conv_f32(inp, w, sc, sh, a, rows, epilogue="muladd")), _bits(good))
    # a temporal tap bounded by the launch's frames instead of the window
    assert not np.array_equal(_bits(K.conv_f32(inp, w, sc, sh, a, rows, tap_bound="frames")), _bits(good))
    # the pool: dx-major order, relu(a) and b added to s separately
    x2, x1 = (rng.standard_normal((4, 6, 8, 16)).astype(F32) for _ in range(2))
    good = K.shortcut_pool_f32(x2, x1)
    for v in ("dxdy", "split"):
        assert not np.array_equal(_bits(K.shortcut_pool_f32(x2, x1, v)), _bits(good)), v
    # (relu(a) + b) * 0.25 per element: * 0.25 is exact for normal numbers, so it differs only where a partial sum is subnormal
    assert np.array_equal(_bits(K.shortcut_pool_f32(x2, x1, "quarter_each")), _bits(good))
    t2, t1 = (x * F32(2.0**-126) for x in (x2, x1))
    assert not np.array_equal(_bits(K.shortcut_pool_f32(t2, t1, "quarter_each")), _bits(K.shortcut_pool_f32(t2, t1)))
    # spatial_mean: * (1 / npos)
    x = rng.standard_normal((6, 312, 32)).astype(F32)
    assert not np.array_equal(_bits(K.spatial_mean_f32(x, "recip")), _bits(K.spatial_mean_f32(x)))
    # the kernel's own formulas pass the float64 bound, so the bitwise rule is the only thing the wrong ones fail
    got, ref, bound = _run(p, "random", seed=5)
    assert (np.abs(got - ref) <= bound).all()
