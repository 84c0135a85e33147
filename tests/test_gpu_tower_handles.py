"""Lifecycle of the tower handles through the C ABI (cb_vit_* for CLIP and SigLIP, cb_iv2_*, cb_iv2_text_*) on small seeded
configurations: set_tensor's name and size checks, finalize's completeness check, forward before finalize, a set_tensor after finalize
(forward refused until the next finalize, which gives a fresh handle's output bit for bit, including SigLIP's folded pooling query), and a
second finalize with another capacity (calls larger than the capacity, so they run in chunks)."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from gpu_helpers import ctx  # noqa: F401
from oracle import vit

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = -2, -6
N = 5  # items per forward: more than either capacity below


def _err(ctx) -> str:
    msg = ctx.lib.cb_last_error(ctx.h)
    return msg.decode() if msg else ""


class _Tower:
    """One handle driven through its C entry points; `prefix` is "vit", "iv2" or "iv2_text"."""

    prefix = ""

    def __init__(self, ctx, weights: dict):
        self.ctx, self.lib, self.h = ctx, ctx.lib, C.c_void_p()
        rc = getattr(self.lib, f"cb_{self.prefix}_create")(ctx.h, C.byref(self.cfg_struct()), C.byref(self.h))
        assert rc == 0, _err(ctx)
        for name, a in weights.items():
            assert self.set(name, a) == 0, _err(ctx)

    def close(self):
        getattr(self.lib, f"cb_{self.prefix}_destroy")(self.h)

    def set(self, name: str, arr: np.ndarray) -> int:
        a = np.ascontiguousarray(arr, dtype=np.float32)
        return getattr(self.lib, f"cb_{self.prefix}_set_tensor")(self.h, name.encode(), a.ctypes.data_as(C.POINTER(C.c_float)), a.size)

    def finalize(self, cap: int) -> int:
        return getattr(self.lib, f"cb_{self.prefix}_finalize")(self.h, cap)


class _Vit(_Tower):
    prefix = "vit"

    def __init__(self, ctx, cfg: vit.VitConfig, weights: dict):
        self.vcfg = cfg
        super().__init__(ctx, weights)
        self.k_pad = int(self.lib.cb_vit_k_pad(self.h))

    def cfg_struct(self):
        from cosmos_curate_b200 import _lib

        c = self.vcfg
        return _lib.VitCfg(c.image_size, c.patch, c.hidden, c.layers, c.heads, c.mlp, c.proj_dim,
                           _lib.ACT_QUICK_GELU if c.act == "quick_gelu" else _lib.ACT_GELU_TANH,
                           _lib.ARCH_CLIP if c.arch == "clip" else _lib.ARCH_SIGLIP, c.ln_eps)  # fmt: skip

    def inputs(self):
        g2, kp = (self.vcfg.image_size // self.vcfg.patch) ** 2, 3 * self.vcfg.patch**2
        p = torch.zeros(N, g2, self.k_pad, dtype=torch.float16)
        p[:, :, :kp] = torch.randn(N, g2, kp, generator=torch.Generator().manual_seed(7)).half()
        return p.cuda()

    def forward(self, x):
        from cosmos_curate_b200.runtime import _stream_ptr

        out_dim = self.vcfg.proj_dim or self.vcfg.hidden
        emb = torch.full((N, out_dim), float("nan"), device="cuda")
        feat = torch.full((N, out_dim), float("nan"), device="cuda")
        rc = self.lib.cb_vit_forward(self.h, x.data_ptr(), N, emb.data_ptr(), feat.data_ptr(), None, _stream_ptr())
        torch.cuda.synchronize()
        return rc, torch.cat([emb, feat], 1).cpu()


class _Iv2(_Tower):
    prefix = "iv2"
    CFG = {"image_size": 224, "patch": 14, "frames": 1, "hidden": 1408, "layers": 1, "heads": 16, "mlp": 512, "clip_dim": 256,
           "embed_dim": 128, "rms_eps": 1e-6, "ln_eps": 1e-5}  # fmt: skip

    def cfg_struct(self):
        from cosmos_curate_b200 import _lib
        from cosmos_curate_b200.runtime import Iv2Tower

        return _lib.Iv2Cfg(*[self.CFG[k] for k in Iv2Tower.FIELDS])

    def inputs(self):
        c = self.CFG
        return torch.randn(N, c["frames"], 3, c["image_size"], c["image_size"], generator=torch.Generator().manual_seed(7)).cuda()

    def forward(self, x):
        from cosmos_curate_b200.runtime import _stream_ptr

        emb = torch.full((N, self.CFG["embed_dim"]), float("nan"), device="cuda")
        rc = self.lib.cb_iv2_forward(self.h, x.data_ptr(), N, emb.data_ptr(), _stream_ptr())
        torch.cuda.synchronize()
        return rc, emb.cpu()


class _Text(_Tower):
    prefix = "iv2_text"
    CFG = {"hidden": 1024, "layers": 1, "heads": 16, "mlp": 512, "vocab": 64, "max_pos": 16, "embed_dim": 128, "ln_eps": 1e-12}
    L = 8

    def cfg_struct(self):
        from cosmos_curate_b200 import _lib
        from cosmos_curate_b200.runtime import Iv2TextTower

        return _lib.Iv2TextCfg(*[self.CFG[k] for k in Iv2TextTower.FIELDS])

    def finalize(self, cap: int) -> int:
        return self.lib.cb_iv2_text_finalize(self.h, cap, self.L)

    def inputs(self):
        rng = np.random.default_rng(7)
        return rng.integers(0, self.CFG["vocab"], (N, self.L), dtype=np.int32), np.array([8, 1, 5, 8, 3], dtype=np.int32)

    def forward(self, x):
        from cosmos_curate_b200.runtime import _stream_ptr

        ids, lengths = x
        emb = torch.full((N, self.CFG["embed_dim"]), float("nan"), device="cuda")
        rc = self.lib.cb_iv2_text_forward(self.h, ids.ctypes.data_as(C.POINTER(C.c_int32)), lengths.ctypes.data_as(C.POINTER(C.c_int32)), N,
                                          self.L, emb.data_ptr(), _stream_ptr())  # fmt: skip
        torch.cuda.synchronize()
        return rc, emb.cpu()


SIGLIP_TINY = vit.VitConfig(image_size=64, patch=16, hidden=128, layers=1, heads=2, mlp=256, proj_dim=0, act="gelu_tanh", ln_eps=1e-6,
                            arch="siglip")  # fmt: skip


# the tensor the set-after-finalize test replaces (SigLIP's: the query folded at finalize is projected by it) and the finalize test omits
SWAP = {"clip": "L1.fc1_w", "siglip": "map_in_w", "iv2": "L0.qkv_w", "text": "L0.fc2_w"}


def _make(kind: str, ctx, skip: str | None = None, replace: dict | None = None):
    """(handle with every seeded tensor set but `skip`, overridden by `replace`; the full weights)."""
    from cosmos_curate_b200.models import internvideo2 as M

    if kind == "clip":
        w, make = vit.random_weights(vit.CLIP_TINY, seed=0), lambda c, w: _Vit(c, vit.CLIP_TINY, w)
    elif kind == "siglip":
        w, make = vit.random_weights(SIGLIP_TINY, seed=0), lambda c, w: _Vit(c, SIGLIP_TINY, w)
    elif kind == "iv2":
        w, make = M.seeded_weights(_Iv2.CFG, seed=0), _Iv2
    else:
        w, make = M.seeded_text_weights(_Text.CFG, seed=0), _Text
    w = {**w, **(replace or {})}
    return make(ctx, {k: v for k, v in w.items() if k != skip}), w


KINDS = ["clip", "siglip", "iv2", "text"]


@pytest.mark.parametrize("kind", KINDS)
def test_set_tensor_rejects_unknown_names_and_wrong_sizes(ctx, kind):
    t, w = _make(kind, ctx)
    try:
        assert t.set("L0.no_such_leaf", np.zeros(4, np.float32)) == ERR_ARG
        assert "unknown tensor" in _err(ctx)
        assert t.set("L99.fc1_w", np.zeros(4, np.float32)) == ERR_ARG  # a layer past the configured depth
        assert "unknown tensor" in _err(ctx)
        name = next(iter(w))
        assert t.set(name, np.zeros(w[name].size + 1, np.float32)) == ERR_ARG
        assert "expected" in _err(ctx)
    finally:
        t.close()


@pytest.mark.parametrize("kind", KINDS)
def test_finalize_needs_every_tensor_and_forward_needs_finalize(ctx, kind):
    swap = SWAP[kind]
    t, w = _make(kind, ctx, skip=swap)
    try:
        x = t.inputs()
        assert t.forward(x)[0] == ERR_STATE
        assert t.finalize(2) == ERR_STATE
        assert "never set" in _err(ctx) and swap in _err(ctx)
        assert t.forward(x)[0] == ERR_STATE
        assert t.set(swap, w[swap]) == 0
        assert t.finalize(2) == 0
        rc, out = t.forward(x)
        assert rc == 0 and torch.isfinite(out).all()
    finally:
        t.close()


@pytest.mark.parametrize("kind", KINDS)
def test_set_tensor_after_finalize_takes_effect_at_the_next_finalize(ctx, kind):
    swap = SWAP[kind]
    t, w = _make(kind, ctx)
    new = {swap: (np.random.default_rng(11).standard_normal(w[swap].shape) * w[swap].std()).astype(np.float32)}
    fresh, _ = _make(kind, ctx, replace=new)
    try:
        x = t.inputs()
        assert t.finalize(2) == 0
        rc, before = t.forward(x)
        assert rc == 0
        assert t.set(swap, new[swap]) == 0
        assert t.forward(x)[0] == ERR_STATE
        assert t.finalize(2) == 0
        assert fresh.finalize(2) == 0
        rc, got = t.forward(x)
        rc_f, want = fresh.forward(x)
        assert rc == 0 and rc_f == 0
        assert torch.isfinite(want).all() and not torch.equal(want, before)
        assert torch.equal(got, want)
    finally:
        t.close(), fresh.close()


@pytest.mark.parametrize("kind", KINDS)
def test_second_finalize_with_another_capacity(ctx, kind):
    t, _ = _make(kind, ctx)
    fresh, _ = _make(kind, ctx)
    try:
        x = t.inputs()
        assert t.finalize(2) == 0
        assert t.forward(x)[0] == 0
        assert t.finalize(3) == 0
        assert fresh.finalize(3) == 0
        rc, got = t.forward(x)
        rc_f, want = fresh.forward(x)
        assert rc == 0 and rc_f == 0 and torch.isfinite(want).all()
        assert torch.equal(got, want)
    finally:
        t.close(), fresh.close()

