"""Oracle for the shot network's kernels (csrc/transnet.cu): the conv gather-GEMM and its dispatch, window_gather, shortcut_pool,
spatial_mean, l2_normalize_rows, window_similarity_fc and head, plus the network's launch schedule and cb_transnet_finalize's packing.

Every kernel has two models here:

* a float64 reference built from the reference model's own formulation (`F.conv3d` with the state dict's weight layout, padding
  and dilation, `F.batch_norm`, `F.avg_pool3d`, `transnetv2._windowed` of the cosine matrix), never from the gather-GEMM, so a
  packing or tap-indexing error shared by a kernel and its float32 model still shows;
* a float32 model (`*_f32`) that rounds exactly as the kernel does.  The contractions it assumes were read from `cuobjdump -sass` of
  the library built for sm_90a with the project's flags (no fast-math, -fmad on):
    - conv: `acc = fmaf(a, b, acc)` is one FFMA per k, k tap-major then channel, from +0; epilogue FFMA(acc, scale, shift) with a scale,
      else FADD(acc, shift); relu is FMNMX(y, 0), which turns NaN into 0;
    - window_gather: `(float)r / 255.0f` is the IEEE division (MUFU.RCP + FFMA fix-up + slow path): correctly rounded; the histogram's
      sum of squared counts is exact; `sqrtf` and `/ denom` are IEEE;
    - shortcut_pool: FMNMX(a, 0), FADD(b, .), FADD(s, .) per tap in dy, dx order, then FMUL by 0.25;
    - spatial_mean: FADDs in position order, then the IEEE division by (float)npos;
    - l2_normalize_rows: `ss += r * r` is an FFMA chain per thread (stride 128), SHFL.BFLY + FADD butterfly, then
      ((red0 + red1) + red2) + red3, IEEE sqrtf and division;
    - window_similarity_fc: explicit fmaf chains (lane stride 32), butterfly, then the 101-term fmaf chain from bias[o];
    - head: fmaf chain per lane (stride 32), butterfly, FADD(s, bias); `1.0f + expf(-x)` is FFMA(2^i, ex2(f), 1), a single rounding of
      1 + expf(-x); `1.0f / .` is the IEEE division.  CUDA's expf is within 2 ulp, so head gives a candidate per ulp offset.

Input classes: "exact" (small integers and dyadic scale/shift: every partial sum is exact below 2^24, so kernel, model and float64
reference agree bit for bit at any size) and "random" (network magnitudes: the kernel equals the model bit for bit and the model is
within gamma_K sum|a w| of the float64 reference).

Test infrastructure only (see oracle/__init__.py).
"""

from __future__ import annotations

import re
from dataclasses import dataclass
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

from oracle import transnetv2 as tn
from oracle.rowops import fma, ulp_step, warp_sum

TRANSNET_CU = Path(__file__).resolve().parent.parent / "cosmos_curate_b200" / "csrc" / "transnet.cu"
F32 = np.float32
U = 2.0**-24
EXPF_ULP = 2  # CUDA Math API: expf max error 2 ulp
FRAME_H, FRAME_W, LOOKUP, SIM, HIST, FC_IN, FC_OUT, TRUNK_OFF = 27, 48, 101, 128, 512, 4864, 1024, 256

# ------------------------------------------------------------------------------------------------ dispatch
INSTS = ((16, 8, 16), (8, 8, 16), (8, 4, 16), (4, 4, 8), (16, 8, 4))  # (CT, TN, BKC) of every conv_gemm_kernel instantiation


def tile(inst) -> tuple[int, int]:
    """(BM, BN) of an instantiation: 256 threads as (256 / CT) x CT, each owning 8 rows x TN columns."""
    ct, tn_, _ = inst
    return 8 * 256 // ct, ct * tn_


def conv_inst(cin: int, n: int):
    """conv_dispatch restated: the (CT, TN, BKC) that runs (cin, N), or None where it returns CB_ERR_UNSUPPORTED."""
    if n % 4:
        return None
    if cin % 16 == 0:
        if n >= 128:
            return (16, 8, 16)
        if n >= 64:
            return (8, 8, 16)
        if n >= 32:
            return (8, 4, 16)
        return (4, 4, 8)
    if cin % 4 == 0 and n >= 128:
        return (16, 8, 4)
    return None


def dispatch_from_source(text: str | None = None):
    """conv_dispatch as transnet.cu writes it, as a function (cin, N) -> inst | None."""
    text = TRANSNET_CU.read_text() if text is None else text
    body = re.search(r"\nstatic int conv_dispatch\(.*?\n}\n", text, re.S)
    assert body, "transnet.cu has no conv_dispatch"
    b = body.group(0)
    n_mod = int(re.search(r"if \(a\.N % (\d+)\) return fail", b).group(1))
    rules = []  # (cin_mod, n_min, inst) in source order
    blk = re.search(r"if \(a\.cin % (\d+) == 0\) \{(.*?)\n  \}", b, re.S)
    for nmin, *inst in re.findall(r"(?:if \(a\.N >= (\d+)\) )?return launch_conv<(\d+), (\d+), (\d+)>", blk.group(2)):
        rules.append((int(blk.group(1)), int(nmin or 0), tuple(map(int, inst))))
    for cm, nmin, *inst in re.findall(r"if \(a\.cin % (\d+) == 0 && a\.N >= (\d+)\) return launch_conv<(\d+), (\d+), (\d+)>", b[blk.end():]):
        rules.append((int(cm), int(nmin), tuple(map(int, inst))))

    def dispatch(cin: int, n: int):
        if n % n_mod:
            return None
        for cm, nmin, inst in rules:  # the cin % 16 block ends with an unconditional launch, so its first match is final
            if cin % cm == 0 and n >= nmin:
                return inst
        return None

    dispatch.rules = rules
    return dispatch


def instantiations_in_source(text: str | None = None) -> set:
    text = TRANSNET_CU.read_text() if text is None else text
    return {tuple(map(int, m)) for m in re.findall(r"launch_conv<(\d+), (\d+), (\d+)>\(ctx", text)}


# ------------------------------------------------------------------------------------------------ the network's schedule
def blocks():
    """(stack, block, cin, cin_pad, filters, relu) in execution order (cb_transnet_finalize)."""
    for lp in tn.layer_plan():
        cin = lp["in"]
        yield lp["stack"], lp["block"], cin, (cin + 3) & ~3, lp["filters"], lp["relu"]


def conv_launch(name, inp, w, out, M, N, cin, in_ld, w_ld, out_ld, T, H, W, mode, *, scale=None, shift=None, in_off=0, out_off=0, in_coff=0,
                out_coff=0, dil=1, relu=0, z=1, z_in_coff=0, z_out_coff=0, z_dil_shift=0, z_w=0) -> dict:
    return dict(kind="conv", name=name, inp=inp, in_off=in_off, w=w, out=out, out_off=out_off, scale=scale, shift=shift, M=M, N=N, cin=cin,
                in_ld=in_ld, in_coff=in_coff, w_ld=w_ld, out_ld=out_ld, out_coff=out_coff, T=T, H=H, W=W, mode=mode, dil=dil, relu=relu, z=z,
                z_in_coff=z_in_coff, z_out_coff=z_out_coff, z_dil_shift=z_dil_shift, z_w=z_w)  # fmt: skip


def schedule(B: int, T: int) -> list[dict]:
    """run_windows' launches for B windows of T frames, in order.  Buffers are named as in cb_transnet (x0, mid, b1, b2, p0, p1,
    hist, feats, proj, concat, fc1, prob); `*_off` are float offsets into them; weights are named by `pack`'s keys."""
    fr = B * T
    L = [dict(kind="gather", B=B, T=T, x0="x0", hist="hist")]
    H, W, x, x_off, x_ld, feat_off = FRAME_H, FRAME_W, "x0", 0, 4, 0
    for s in range(3):
        f = 16 << s
        C, M = 4 * f, fr * H * W
        for _, b, _, cin_pad, _, relu in (bl for bl in blocks() if bl[0] == s):
            p = f"s{s}b{b}"
            L.append(conv_launch(f"{p}.spatial", x, f"{p}.w1", "mid", M, 8 * f, cin_pad, x_ld, 8 * f, 8 * f, T, H, W, 1, in_off=x_off))
            L.append(conv_launch(f"{p}.temporal", "mid", f"{p}.w2", ("b1", "b2")[b], M, f, 2 * f, 8 * f, f, C, T, H, W, 2, scale=f"{p}.scale",
                                 shift=f"{p}.shift", relu=int(relu), z=4, z_in_coff=2 * f, z_out_coff=f, z_dil_shift=1, z_w=6 * f * f))  # fmt: skip
            x, x_off, x_ld = ("b1", "b2")[b], 0, C
        hp, wp = H // 2, W // 2
        pooled, p_off = (("p0", 0), ("p1", 0), ("concat", TRUNK_OFF))[s]
        fstride = FC_IN if s == 2 else hp * wp * C
        L.append(dict(kind="pool", x2="b2", x1="b1", out=pooled, out_off=p_off, frames=fr, H=H, W=W, C=C, out_frame_stride=fstride))
        L.append(dict(kind="mean", x=pooled, x_off=p_off, frame_stride=fstride, frames=fr, npos=hp * wp, C=C, feats="feats", feats_ld=448, coff=feat_off))
        feat_off += C
        x, x_off, x_ld, H, W = pooled, p_off, C, hp, wp
    L.append(conv_launch("proj", "feats", "proj_wt", "proj", fr, SIM, 448, 448, SIM, SIM, T, 1, 1, 0, shift="proj_b"))
    L.append(dict(kind="l2", x="proj", rows=fr, D=SIM))
    L.append(dict(kind="simfc", x="proj", rows=fr, D=SIM, T=T, wt="sim_fc_wt", bias="sim_fc_b", out="concat", out_ld=FC_IN, out_coff=SIM))
    L.append(dict(kind="simfc", x="hist", rows=fr, D=HIST, T=T, wt="hist_fc_wt", bias="hist_fc_b", out="concat", out_ld=FC_IN, out_coff=0))
    L.append(conv_launch("fc1", "concat", "fc1_wt", "fc1", fr, FC_OUT, FC_IN, FC_IN, FC_OUT, FC_OUT, T, 1, 1, 0, shift="fc1_b", relu=1))
    L.append(dict(kind="head", h="fc1", w="cls_w", bias="cls_b", rows=fr, T=T))
    return L


def workspace_floats(frames: int) -> dict[str, int]:
    """Floats each workspace buffer needs for `frames` frames (the sizes cb_transnet_finalize allocates per frame)."""
    pos0 = FRAME_H * FRAME_W
    per = dict(x0=pos0 * 4, mid=pos0 * 128, b1=pos0 * 64, b2=pos0 * 64, p0=13 * 24 * 64, p1=6 * 12 * 128, hist=HIST, feats=448, proj=SIM,
               concat=FC_IN, fc1=FC_OUT)  # fmt: skip
    return {k: v * frames for k, v in per.items()}


# ------------------------------------------------------------------------------------------------ packing (cb_transnet_finalize)
def pack_spatial(w: np.ndarray, cin_pad: int) -> np.ndarray:
    """(1,3,3) conv weight [N][cin][1][3][3] -> Wt[tap * cin_pad + ci][n], tap = 3 kh + kw, rows cin..cin_pad-1 zero."""
    n, cin = w.shape[:2]
    out = np.zeros((9, cin_pad, n), F32)
    out[:, :cin] = np.asarray(w, F32).reshape(n, cin, 9).transpose(2, 1, 0)
    return out.reshape(9 * cin_pad, n)


def pack_temporal(w: np.ndarray) -> np.ndarray:
    """(3,1,1) conv weight [N][cin][3][1][1] -> Wt[kt * cin + c][n]."""
    n, cin = w.shape[:2]
    return np.ascontiguousarray(np.asarray(w, F32).reshape(n, cin, 3).transpose(2, 1, 0).reshape(3 * cin, n))


def bn_fold(sd: dict, p: str) -> tuple[np.ndarray, np.ndarray]:
    """BatchNorm3d(eps=1e-3, eval) as scale/shift, folded in double and rounded to fp32 as cb_transnet_finalize does."""
    g, be, mu, var = (np.asarray(sd[f"{p}.bn.{k}"], np.float64) for k in ("weight", "bias", "running_mean", "running_var"))
    inv = 1.0 / np.sqrt(var + 1e-3)
    return (g * inv).astype(F32), (be - mu * g * inv).astype(F32)


def pack(sd: dict) -> dict[str, np.ndarray]:
    """The device tensors cb_transnet_finalize uploads, by the names `schedule` uses (cls_b is a 1-element array)."""
    out = {}
    for s, b, cin, cin_pad, f, _ in blocks():
        p = f"SDDCNN.{s}.DDCNN.{b}"
        w1 = np.zeros((9 * cin_pad, 8 * f), F32)
        w2 = np.zeros((4, 3 * 2 * f, f), F32)
        for br, d in enumerate(tn.DILATIONS):
            w1[:, br * 2 * f : (br + 1) * 2 * f] = pack_spatial(sd[f"{p}.Conv3D_{d}.layers.0.weight"], cin_pad)
            w2[br] = pack_temporal(sd[f"{p}.Conv3D_{d}.layers.1.weight"])
        out[f"s{s}b{b}.w1"], out[f"s{s}b{b}.w2"] = w1, w2.reshape(-1)
        out[f"s{s}b{b}.scale"], out[f"s{s}b{b}.shift"] = bn_fold(sd, p)
    t = lambda k: np.ascontiguousarray(np.asarray(sd[k], F32).T)  # noqa: E731  [out][in] Linear weight -> [in][out]
    out["proj_wt"], out["proj_b"] = t("frame_sim_layer.projection.weight"), np.asarray(sd["frame_sim_layer.projection.bias"], F32)
    out["sim_fc_wt"], out["sim_fc_b"] = t("frame_sim_layer.fc.weight"), np.asarray(sd["frame_sim_layer.fc.bias"], F32)
    out["hist_fc_wt"], out["hist_fc_b"] = t("color_hist_layer.fc.weight"), np.asarray(sd["color_hist_layer.fc.bias"], F32)
    out["fc1_wt"], out["fc1_b"] = t("fc1.weight"), np.asarray(sd["fc1.bias"], F32)
    out["cls_w"], out["cls_b"] = np.asarray(sd["cls_layer1.weight"], F32).reshape(-1), np.asarray(sd["cls_layer1.bias"], F32).reshape(1)
    return out


# ------------------------------------------------------------------------------------------------ conv: float32 model
def conv_gather(inp: np.ndarray, a: dict, z: int, rows: np.ndarray, tap_bound: str = "window") -> np.ndarray:
    """A[rows][taps * cin] of branch z as the kernel gathers it from the flat buffer `inp` (zero outside the frame / window).
    tap_bound="frames" restates the wrong rule that bounds a temporal tap by all the launch's frames instead of the window."""
    hw = a["H"] * a["W"]
    m = np.asarray(rows, np.int64)
    fr, pos = m // hw, m % hw
    t, h, w = fr % a["T"], pos // a["W"], pos % a["W"]
    taps = {0: 1, 1: 9, 2: 3}[a["mode"]]
    dil = a["dil"] << (z if a["z_dil_shift"] else 0)
    cols = a["in_coff"] + z * a["z_in_coff"] + np.arange(a["cin"])
    out = np.zeros((len(m), taps, a["cin"]), inp.dtype)
    for tap in range(taps):
        if a["mode"] == 1:
            dh, dw = tap // 3 - 1, tap % 3 - 1
            ok, src = (h + dh >= 0) & (h + dh < a["H"]) & (w + dw >= 0) & (w + dw < a["W"]), m + dh * a["W"] + dw
        elif a["mode"] == 2:
            dt = (tap - 1) * dil
            ok = ((t + dt >= 0) & (t + dt < a["T"])) if tap_bound == "window" else ((fr + dt >= 0) & (fr + dt < a["M"] // hw))
            src = m + dt * hw
        else:
            ok, src = np.ones(len(m), bool), m
        idx = np.where(ok, src, 0)[:, None] * a["in_ld"] + cols[None, :]
        out[:, tap] = np.where(ok[:, None], inp[idx], 0)
    return out.reshape(len(m), taps * a["cin"])


def conv_f32(inp, w, scale, shift, a: dict, rows, epilogue: str = "fma", tap_bound: str = "window") -> np.ndarray:
    """The kernel's output at `rows` for every branch: [len(rows)][z][N].  The k sum is one fmaf chain from +0 in tap-major order;
    epilogue "fma" is the kernel's fmaf(acc, scale, shift), "muladd" the wrong acc * scale + shift rounded twice."""
    out = np.empty((len(rows), a["z"], a["N"]), F32)
    for z in range(a["z"]):
        A = conv_gather(inp, a, z, rows, tap_bound)
        wz = w[z * a["z_w"] :][: A.shape[1] * a["w_ld"]].reshape(A.shape[1], a["w_ld"])[:, : a["N"]]
        acc = np.zeros((len(rows), a["N"]), F32)
        for k in range(A.shape[1]):
            acc = fma(A[:, k, None], wz[k][None, :], acc)
        c = a["out_coff"] + z * a["z_out_coff"] + np.arange(a["N"])
        sh = shift[c] if shift is not None else np.zeros(a["N"], F32)
        if scale is not None:
            y = fma(acc, scale[c][None, :], sh[None, :]) if epilogue == "fma" else (acc * scale[c][None, :]).astype(F32) + sh[None, :]
        else:
            y = acc + sh[None, :]
        out[:, z] = relu_f32(y) if a["relu"] else y
    return out


def relu_f32(y: np.ndarray) -> np.ndarray:
    """fmaxf(y, 0): NaN -> 0."""
    return np.where(y > 0, y, F32(0)).astype(F32)


def conv_abs_f32(inp, w, a: dict, rows) -> np.ndarray:
    """sum_k |A w| per output in float64 ([len(rows)][z][N]), for the gamma_K bound."""
    out = np.empty((len(rows), a["z"], a["N"]))
    for z in range(a["z"]):
        A = np.abs(conv_gather(inp, a, z, rows).astype(np.float64))
        wz = w[z * a["z_w"] :][: A.shape[1] * a["w_ld"]].reshape(A.shape[1], a["w_ld"])[:, : a["N"]]
        out[:, z] = A @ np.abs(wz.astype(np.float64))
    return out


def conv_bound(abs_sum: np.ndarray, y_ref: np.ndarray, scale_abs: np.ndarray, K: int) -> np.ndarray:
    """|fp32 result - float64 reference| bound: the fmaf chain's gamma_K sum|a w|, carried through |scale|, plus one rounding of the
    epilogue (relu is 1-Lipschitz)."""
    g = K * U / (1 - K * U)
    e = scale_abs * g * abs_sum
    return e + U * (np.abs(y_ref) + e) + 1e-45


# ------------------------------------------------------------------------------------------------ conv: float64 reference
def conv_ref(x: np.ndarray, w_ref: np.ndarray, mode: int, T: int, H: int, W: int, dil: int = 1, device="cpu") -> torch.Tensor:
    """The reference's formulation in float64.  x [M][cin] (rows as the kernel sees them), w_ref in the state dict's layout:
    mode 1 [N][cin][1][3][3] (padding (0, 1, 1)), mode 2 [N][cin][3][1][1] (padding (dil, 0, 0), dilation (dil, 1, 1)), mode 0 [N][cin]
    (F.linear).  Returns [M][N] float64 before the epilogue."""
    xt = torch.as_tensor(x, device=device).to(torch.float64)
    wt = torch.as_tensor(w_ref, device=device).to(torch.float64)
    if mode == 0:
        return F.linear(xt, wt)
    cin, hw = xt.shape[1], H * W
    frames = xt.shape[0] // hw
    if mode == 1:
        v = xt.reshape(1, frames, H, W, cin).permute(0, 4, 1, 2, 3)
        y = F.conv3d(v, wt, padding=(0, 1, 1))
    else:
        v = xt.reshape(frames // T, T, H, W, cin).permute(0, 4, 1, 2, 3)
        y = F.conv3d(v, wt, padding=(dil, 0, 0), dilation=(dil, 1, 1))
    return y.permute(0, 2, 3, 4, 1).reshape(xt.shape[0], -1)


def epilogue_ref(acc: torch.Tensor, scale, shift, relu: bool) -> torch.Tensor:
    y = acc
    if scale is not None:
        y = y * torch.as_tensor(scale, device=acc.device).to(torch.float64)
    if shift is not None:
        y = y + torch.as_tensor(shift, device=acc.device).to(torch.float64)
    return torch.relu(y) if relu else y


# ------------------------------------------------------------------------------------------------ conv: sweep
@dataclass(frozen=True)
class ConvPoint:
    cin: int
    N: int
    M: int
    mode: int
    T: int = 1
    H: int = 1
    W: int = 1
    z: int = 1
    epi: str = "scale"  # "scale" (BN: scale + shift), "shift" (bias), "none"
    relu: int = 0
    note: str = ""

    @property
    def inst(self):
        return conv_inst(self.cin, self.N)

    @property
    def name(self) -> str:
        ct, tn_, bkc = self.inst
        return f"c{ct}x{tn_}x{bkc}-m{self.mode}-cin{self.cin}-N{self.N}-M{self.M}-T{self.T}-{self.H}x{self.W}-z{self.z}-{self.epi}{'-relu' if self.relu else ''}"

    def args(self, ld_pad: int = 4) -> dict:
        """Launch arguments with strides wider than the operands (ld_pad floats more) and a column offset, so a stride / offset mix-up
        shows.  Each branch z reads its own cin-channel slice and writes its own N-column slice."""
        z_in, z_out = (self.cin + 4 if self.z > 1 else 0), (self.N + 4 if self.z > 1 else 0)
        in_coff, out_coff = 4, 8
        k = {0: 1, 1: 9, 2: 3}[self.mode] * self.cin
        w_ld = self.N + ld_pad
        return dict(M=self.M, N=self.N, cin=self.cin, in_ld=in_coff + self.z * max(z_in, self.cin) + ld_pad, in_coff=in_coff, w_ld=w_ld,
                    out_ld=out_coff + self.z * max(z_out, self.N) + ld_pad, out_coff=out_coff, T=self.T, H=self.H, W=self.W, mode=self.mode,
                    dil=1, relu=self.relu, z=self.z, z_in_coff=z_in, z_out_coff=z_out, z_dil_shift=int(self.mode == 2 and self.z > 1),
                    z_w=k * w_ld if self.z > 1 else 0)  # fmt: skip


def m_classes(inst) -> tuple[int, ...]:
    """M mod BM classes: 0, 1, HALF_M - 1, HALF_M, HALF_M + 1, BM - 1 (rows split at HALF_M in the thread mapping)."""
    bm = tile(inst)[0]
    return (0, 1, bm // 2 - 1, bm // 2, bm // 2 + 1, bm - 1)


# cin / N choices per instantiation: one and several k chunks per tap; the N tails the dispatch admits and both sides of each
# dispatch boundary (N 28/32, 60/64, 124/128; cin % 16 vs cin % 4)
INST_SHAPES = {
    (16, 8, 16): [(16, 128), (32, 132), (48, 252)],
    (8, 8, 16): [(16, 64), (32, 68), (16, 124)],
    (8, 4, 16): [(16, 32), (32, 36), (16, 60)],
    (4, 4, 8): [(16, 4), (32, 16), (16, 20), (16, 28)],
    (16, 8, 4): [(4, 128), (20, 132), (12, 256)],
}
T_CLASSES = (1, 2, 8, 9, 16, 17, 100)


def conv_sweep() -> list[ConvPoint]:
    pts: list[ConvPoint] = []
    epis = [("scale", 1), ("shift", 0), ("none", 0), ("scale", 0), ("shift", 1)]
    for inst, shapes in INST_SHAPES.items():
        bm = tile(inst)[0]
        # every M class in mode 0 (rows as they are) and in mode 2 with one-frame windows of one position
        for i, r in enumerate(m_classes(inst)):
            cin, n = shapes[i % len(shapes)]
            M = bm * (1 + i % 2) + r if r else bm * 2
            e, rl = epis[i % len(epis)]
            pts.append(ConvPoint(cin, n, M, 0, epi=e, relu=rl, note="m-class"))
        for j, (cin, n) in enumerate(shapes):
            e, rl = epis[(j + 1) % len(epis)]
            pts.append(ConvPoint(cin, n, bm + 1 + j, 2, T=1, z=4 if j % 2 == 0 else 1, epi=e, relu=rl, note="n-tail"))
        # spatial borders: a real frame, a single row, a single column, one position
        cin, n = shapes[0]
        for H, W, fr in ((27, 48, 1), (1, 7, 5), (6, 1, 3), (1, 1, 9), (5, 9, 2)):
            pts.append(ConvPoint(cin, n, H * W * fr, 1, H=H, W=W, epi="none", note="border"))
    # temporal taps at every T class, four dilation branches (1, 2, 4, 8) and one, through the instantiations the network's
    # temporal convs use
    for i, T in enumerate(T_CLASSES):
        for cin, n in ((32, 16), (64, 32), (128, 64)):
            H, W = (1, 1) if T >= 16 else (2, 3)
            nwin = 3 if T < 100 else 2
            pts.append(ConvPoint(cin, n, nwin * T * H * W, 2, T=T, H=H, W=W, z=4, epi="scale", relu=(i + cin // 32) % 2, note="temporal"))
        pts.append(ConvPoint(16, 128, 2 * T, 2, T=T, z=1, epi="shift", note="temporal-z1"))
    return pts


def select_rows(M: int, inst, T: int, H: int, W: int, rng: np.random.Generator, extra: int = 24) -> np.ndarray:
    """The rows the float32 model evaluates at large M: the first and last rows, both sides of HALF_M and BM in the first tile and
    the last one, the first and last frame of every window the first tile touches, and a few random rows."""
    bm = tile(inst)[0]
    hw = H * W
    cand = {0, 1, bm // 2 - 1, bm // 2, bm // 2 + 1, bm - 1, bm, bm + 1, M - 1, M - 2, M - bm // 2 - 1, M - bm // 2}
    last_tile = (M - 1) // bm * bm
    cand |= {last_tile, last_tile + 1, last_tile + bm // 2 - 1, last_tile + bm // 2}
    for w0 in range(0, min(M, 2 * bm), T * hw):
        cand |= {w0, w0 + hw - 1, w0 + (T - 1) * hw, w0 + T * hw - 1}
    cand |= set(rng.integers(0, M, extra).tolist())
    return np.array(sorted(c for c in cand if 0 <= c < M), np.int64)


def conv_inputs(kind: str, p: ConvPoint, a: dict, rng: np.random.Generator):
    """(inp flat [M * in_ld], w flat, scale [out_ld] | None, shift [out_ld] | None, w_ref per branch) for one sweep point; `inp`
    carries garbage in the columns the launch must not read.  w_ref is the state-dict layout conv_ref takes."""
    K1 = {0: 1, 1: 9, 2: 3}[p.mode]
    if kind == "exact":
        x = rng.integers(-3, 4, (p.M, a["in_ld"])).astype(F32)
        w_ref = rng.integers(-2, 3, (p.z, p.N, p.cin, K1)).astype(F32)
        sc = (rng.integers(1, 17, a["out_ld"]) / 8).astype(F32)
        sh = (rng.integers(-8, 9, a["out_ld"]) / 4).astype(F32)
    else:
        x = rng.standard_normal((p.M, a["in_ld"])).astype(F32)
        w_ref = (rng.standard_normal((p.z, p.N, p.cin, K1)) * np.sqrt(2.0 / (K1 * p.cin))).astype(F32)
        sc = rng.uniform(0.5, 1.5, a["out_ld"]).astype(F32)
        sh = (rng.standard_normal(a["out_ld"]) * 0.1).astype(F32)
    w = np.full((max(1, p.z) * (a["z_w"] or K1 * p.cin * a["w_ld"]),), np.nan, F32)
    for z in range(p.z):
        wz = np.full((K1 * p.cin, a["w_ld"]), np.nan, F32)
        wz[:, : p.N] = w_ref[z].reshape(p.N, p.cin, K1).transpose(2, 1, 0).reshape(K1 * p.cin, p.N)  # [(tap, c)][n]
        w[z * a["z_w"] : z * a["z_w"] + wz.size] = wz.reshape(-1)
    read = np.zeros(a["in_ld"], bool)
    for z in range(p.z):
        read[a["in_coff"] + z * a["z_in_coff"] :][: p.cin] = True
    x[:, ~read] = np.nan  # columns the launch must not read
    scale = sc if p.epi == "scale" else None
    shift = sh if p.epi in ("scale", "shift") else None
    shape = {0: lambda r: r.reshape(p.N, p.cin), 1: lambda r: r.reshape(p.N, p.cin, 1, 3, 3), 2: lambda r: r.reshape(p.N, p.cin, 3, 1, 1)}[p.mode]
    return x.reshape(-1), w, scale, shift, [shape(w_ref[z]) for z in range(p.z)]


# ------------------------------------------------------------------------------------------------ window_gather
def window_gather_f32(frames: np.ndarray, first, pad, T: int) -> tuple[np.ndarray, np.ndarray]:
    """frames uint8 [n][27][48][3] -> (x0 [B T][1296][4], hist [B T][512]): r / 255.0f, integer bin counts, counts / max(sqrtf(sum of
    squares), 1e-12) (the sum is exact: counts <= 1296)."""
    src = np.array([first[b] + max(t - pad[b], 0) for b in range(len(first)) for t in range(T)], np.int64)
    f = frames[src].reshape(len(src), -1, 3)
    x0 = np.zeros((len(src), f.shape[1], 4), F32)
    x0[..., :3] = f.astype(F32) / F32(255)
    bins = ((f[..., 0].astype(np.int64) >> 5) << 6) + ((f[..., 1].astype(np.int64) >> 5) << 3) + (f[..., 2].astype(np.int64) >> 5)
    counts = np.stack([np.bincount(b, minlength=HIST) for b in bins]).astype(F32)
    ss = (counts.astype(np.float64) ** 2).sum(1).astype(F32)
    denom = np.maximum(np.sqrt(ss), F32(1e-12))
    return x0, counts / denom[:, None]


def window_gather_ref(frames: np.ndarray, first, pad, T: int) -> tuple[np.ndarray, np.ndarray]:
    """float64: frames / 255 and transnetv2.color_histograms' normalised counts."""
    src = np.array([first[b] + max(t - pad[b], 0) for b in range(len(first)) for t in range(T)], np.int64)
    f = frames[src]
    x0 = f.reshape(len(src), -1, 3).astype(np.float64) / 255.0
    b = torch.as_tensor(f).to(torch.int64).view(len(src), -1, 3)
    idx = ((b[..., 0] >> 5) << 6) + ((b[..., 1] >> 5) << 3) + (b[..., 2] >> 5)
    h = torch.zeros(len(src), HIST, dtype=torch.float64).scatter_add_(1, idx, torch.ones_like(idx, dtype=torch.float64))
    return x0, F.normalize(h, p=2, dim=1).numpy()


# ------------------------------------------------------------------------------------------------ shortcut_pool / spatial_mean
def shortcut_pool_f32(x2: np.ndarray, x1: np.ndarray, variant: str = "kernel") -> np.ndarray:
    """x2, x1 [frames][H][W][C] -> [frames][H/2][W/2][C]: s += relu(x2) + x1 over (dy, dx) in row-major order, then s * 0.25.
    Wrong variants: "dxdy" (dx outer), "split" (s = (s + relu(a)) + b), "quarter_each" (s += (relu(a) + b) * 0.25, no final scale:
    equal to the kernel wherever no partial sum is subnormal, since * 0.25 is exact there)."""
    hp, wp = x2.shape[1] // 2, x2.shape[2] // 2
    order = [(0, 0), (0, 1), (1, 0), (1, 1)] if variant != "dxdy" else [(0, 0), (1, 0), (0, 1), (1, 1)]
    s = np.zeros((x2.shape[0], hp, wp, x2.shape[3]), F32)
    for dy, dx in order:
        a = x2[:, dy : 2 * hp : 2, dx : 2 * wp : 2].astype(F32)
        b = x1[:, dy : 2 * hp : 2, dx : 2 * wp : 2].astype(F32)
        if variant == "split":
            s = (s + relu_f32(a)) + b
        elif variant == "quarter_each":
            s = s + (relu_f32(a) + b) * F32(0.25)
        else:
            s = s + (relu_f32(a) + b)
    return s if variant == "quarter_each" else s * F32(0.25)


def shortcut_pool_ref(x2: np.ndarray, x1: np.ndarray) -> np.ndarray:
    """float64 F.avg_pool3d((1, 2, 2)) of relu(x2) + x1 (transnetv2.py:204-221)."""
    v = torch.relu(torch.as_tensor(x2, dtype=torch.float64)) + torch.as_tensor(x1, dtype=torch.float64)
    y = F.avg_pool3d(v.permute(3, 0, 1, 2)[None], kernel_size=(1, 2, 2))
    return y[0].permute(1, 2, 3, 0).numpy()


def spatial_mean_f32(x: np.ndarray, variant: str = "kernel") -> np.ndarray:
    """x [frames][npos][C] -> sum over positions in order, / (float)npos ("recip": * (1.0f / npos), wrong)."""
    s = np.zeros((x.shape[0], x.shape[2]), F32)
    for p in range(x.shape[1]):
        s = s + x[:, p].astype(F32)
    n = F32(x.shape[1])
    return s * (F32(1) / n) if variant == "recip" else s / n


def spatial_mean_ref(x: np.ndarray) -> np.ndarray:
    return torch.mean(torch.as_tensor(x, dtype=torch.float64), dim=1).numpy()


def sum_bound(abs_sum: np.ndarray, n: int, ref: np.ndarray, extra_roundings: int = 1) -> np.ndarray:
    """gamma_n sum|terms| plus `extra_roundings` roundings of the result."""
    g = n * U / (1 - n * U)
    return g * abs_sum + extra_roundings * U * (np.abs(ref) + g * abs_sum) + 1e-45


# ------------------------------------------------------------------------------------------------ l2_normalize_rows
def _lane_chain(x: np.ndarray, y: np.ndarray, threads: int) -> np.ndarray:
    """Per-thread fmaf(x[i], y[i], s) over i = tid, tid + threads, ... from +0: [..., threads]."""
    d = x.shape[-1]
    pad = (-d) % threads
    xp = np.concatenate([x, np.zeros((*x.shape[:-1], pad), F32)], -1).reshape(*x.shape[:-1], -1, threads)
    yp = np.concatenate([y, np.zeros((*y.shape[:-1], pad), F32)], -1).reshape(*y.shape[:-1], -1, threads)
    s = np.zeros((*np.broadcast_shapes(xp.shape, yp.shape)[:-2], threads), F32)
    for k in range(xp.shape[-2]):
        s = fma(xp[..., k, :], yp[..., k, :], s)
    return s


def l2_normalize_f32(x: np.ndarray) -> np.ndarray:
    """x [rows][D] -> rows / max(sqrtf(((r0 + r1) + r2) + r3), 1e-12), r_w = butterfly of warp w's fmaf chains (stride 128)."""
    x = x.astype(F32)
    ss = _lane_chain(x, x, 128)
    r = warp_sum(ss.reshape(x.shape[0], 4, 32))
    tot = ((r[:, 0] + r[:, 1]) + r[:, 2]) + r[:, 3]
    return x / np.maximum(np.sqrt(tot), F32(1e-12))[:, None]


def l2_normalize_ref(x: np.ndarray) -> np.ndarray:
    return F.normalize(torch.as_tensor(x, dtype=torch.float64), p=2, dim=1).numpy()


# ------------------------------------------------------------------------------------------------ window_similarity_fc
def similarities_f32(x: np.ndarray, T: int, rows: np.ndarray) -> np.ndarray:
    """sims [len(rows)][101]: per-lane fmaf chains of x[r] . x[r + j - 50] (lane stride 32) and the butterfly; 0 outside the window."""
    rows = np.asarray(rows, np.int64)
    t = rows % T
    j = np.arange(LOOKUP)
    t2 = t[:, None] + j[None, :] - (LOOKUP - 1) // 2
    ok = (t2 >= 0) & (t2 < T)
    nb = np.where(ok, rows[:, None] - t[:, None] + t2, 0)
    s = warp_sum(_lane_chain(x[rows][:, None, :].astype(F32), x[nb].astype(F32), 32))
    return np.where(ok, s, F32(0)).astype(F32)


def window_similarity_fc_f32(x: np.ndarray, T: int, wt: np.ndarray, bias: np.ndarray, rows=None) -> np.ndarray:
    """[len(rows)][128]: relu of the 101-term fmaf chain bias[o] + sum_j sims[j] wt[j][o], j in order."""
    rows = np.arange(x.shape[0]) if rows is None else np.asarray(rows)
    sims = similarities_f32(x, T, rows)
    acc = np.broadcast_to(bias.astype(F32), (len(rows), SIM)).copy()
    for j in range(LOOKUP):
        acc = fma(sims[:, j, None], wt[j][None, :].astype(F32), acc)
    return relu_f32(acc)


def window_similarity_fc_ref(x: np.ndarray, T: int, wt: np.ndarray, bias: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """float64: transnetv2._windowed of the per-window Gram matrix, Linear, relu (transnetv2.py:393-418).  Returns (out, the bound's
    sum |terms| per output)."""
    xt = torch.as_tensor(x, dtype=torch.float64).reshape(-1, T, x.shape[1])
    sim = tn._windowed(torch.bmm(xt, xt.transpose(1, 2))).reshape(-1, LOOKUP)
    asim = tn._windowed(torch.bmm(xt.abs(), xt.abs().transpose(1, 2))).reshape(-1, LOOKUP)
    w64 = torch.as_tensor(wt, dtype=torch.float64)
    out = torch.relu(sim @ w64 + torch.as_tensor(bias, dtype=torch.float64))
    return out.numpy(), (asim @ w64.abs()).numpy()


def window_similarity_fc_bound(abs_terms: np.ndarray, D: int, ref: np.ndarray, bias: np.ndarray) -> np.ndarray:
    """The dot products' gamma_D (carried through |wt|) plus the fc chain's gamma_102 over |bias| + sum |sim w| and the output's rounding."""
    gd, gf = D * U / (1 - D * U), (LOOKUP + 1) * U / (1 - (LOOKUP + 1) * U)
    t = abs_terms + np.abs(bias)[None, :]
    return gd * abs_terms + gf * (1 + gd) * t + U * np.abs(ref) + 1e-45


# ------------------------------------------------------------------------------------------------ head
def head_logit_f32(h: np.ndarray, w: np.ndarray, bias: np.float32) -> np.ndarray:
    """s + bias: per-lane fmaf chains over i = lane + 32 k, the butterfly, then one FADD."""
    s = warp_sum(_lane_chain(h.astype(F32), np.broadcast_to(w.astype(F32), h.shape), 32))
    return s + F32(bias)


def head_candidates(h: np.ndarray, w: np.ndarray, bias) -> list[tuple[int, np.ndarray]]:
    """[(ulp offset k, p [rows])]: 1.0f / (1.0f + e_k), e_k = the correctly rounded exp(-(s + bias)) moved k ulps, |k| <= 2."""
    x = -head_logit_f32(h, w, bias)
    e = np.exp(x.astype(np.float64)).astype(F32)
    return [(k, F32(1) / (F32(1) + ulp_step(e, k))) for k in range(-EXPF_ULP, EXPF_ULP + 1)]


def head_match(got: np.ndarray, cands) -> np.ndarray:
    """Per row the offset of the first candidate, nearest the correctly rounded exp first, equal bit for bit to `got`; 99 if none."""
    off = np.full(got.shape, 99, np.int64)
    for k, p in sorted(cands, key=lambda kv: (abs(kv[0]), kv[0])):
        off = np.where((off == 99) & (p.view(np.int32) == got.astype(F32).view(np.int32)), k, off)
    return off


def head_ref(h: np.ndarray, w: np.ndarray, bias) -> np.ndarray:
    return torch.sigmoid(torch.as_tensor(h, dtype=torch.float64) @ torch.as_tensor(w, dtype=torch.float64) + float(bias)).numpy()


def stitch_targets(B: int, T: int, w0: int, n_total: int, lo: int = 25, hi: int = 75) -> dict[int, int]:
    """head's stitch mode: {row: prob index} for frames lo..hi-1 of window w0 + b that land below n_total."""
    out = {}
    for b in range(B):
        for t in range(lo, min(hi, T)):
            dst = 50 * (w0 + b) + t - 25
            if dst < n_total:
                out[b * T + t] = dst
    return out


# ------------------------------------------------------------------------------------------------ predict's window plan
def predict_batches(n: int, max_windows: int) -> list[tuple[int, int, int]]:
    """cb_transnet_predict's batches: (first window, windows, T) with every window of a batch the same length."""
    plan = tn.window_plan(n)
    lens = [cnt + pad for _, cnt, pad in plan]
    out, w = [], 0
    while w < len(plan):
        B = 1
        while w + B < len(plan) and B < max_windows and lens[w + B] == lens[w]:
            B += 1
        out.append((w, B, lens[w]))
        w += B
    return out


def len_class(n: int, i: int) -> str:
    """Which terms of len_of decide window i's length: front padding, a cut end, both or neither."""
    return ("pad" if 50 * i < 25 else "") + ("cut" if 50 * i + 75 > n else "") or "full"

