"""ORACLE (test infrastructure, NOT product code) -- the plain-fp16 precision of the tensor-core networks
(OSB_PRECISION_FP16, csrc/conv_umma.cu with FP16 = true).

In plain fp16 a layer reads only the hi planes: activations fp16(16 x), weights fp16(1024 w), one product per K step into
an fp32 accumulator.  That is oracle.split_model.conv_model with both lo planes zero, which `fp16_conv_model` states.
Since fp16 x fp16 products are exact in fp32, the float64 bound TAU * (sum |x| |w| + |b|) of the split layers holds on the
dequantised hi operands; a stored plane adds its own fp16 rounding.

`superpoint_net_fp16` / `netvlad_net_fp16` emulate the whole networks: weights rounded to fp16(1024 w) / 1024 and every
activation the device stores as a plane rounded to fp16(16 x) / 16 at that point; everything else (conv1a, NetVLAD's
conv0 and block 0, the depthwise convolutions, softmax, norms, the VLAD head) in fp32 as on the device.  `accum` selects
float64 or float32 convolutions: the difference between the two is what a different accumulation order costs once it
flips an fp16 rounding, and the GPU tests derive their network tolerance from it (NET_TOL_FACTOR x that difference).
`mutant` switches in one defect per network so that a CPU test can show the tolerance separates it:
  tap_missing   tap 0 of conv2a (SuperPoint) / of no layer in NetVLAD (1x1 only): the first input channel slab of the
                projection instead
  slab_missing  the first 64-channel input slab of conv3b / of block 3's pointwise layer is never accumulated
  lo_read       every tensor-core layer reads the unrounded (hi + lo) activations, as a kernel that reads a nonzero lo
                plane by mistake would (the kernel is shared by all layers)
"""
from __future__ import annotations

import numpy as np

from . import split_model as sm

SA, SW = 16.0, 1024.0
NET_MUTANTS = ("tap_missing", "slab_missing", "lo_read")
# the network tolerance of the GPU tests is this multiple of |emulation(float64) - emulation(float32)|
NET_TOL_FACTOR = 4.0


def fp16_conv_model(x_hi, w_hi, bias, ks: int, act_scale: float, w_scale: float, relu: int = 0, pool: int = 0,
                    rounding: str = "rz", mutant: str | None = None) -> np.ndarray:
    """the plain-fp16 layer: split_model.conv_model with zero lo planes (only mutants that touch the hi planes apply)"""
    return sm.conv_model(x_hi, np.zeros_like(x_hi), w_hi, np.zeros_like(w_hi), bias, ks, act_scale, w_scale, relu, pool,
                         rounding, mutant)


def round_plane(x, scale: float = SA):
    """the value of a stored fp16 plane: fp16(scale * x) / scale (x a torch tensor, any float dtype)"""
    import torch
    return (x.float() * scale).half().to(x.dtype) / scale


def _w16(w):
    import torch
    return (torch.from_numpy(np.asarray(w, np.float32)) * SW).half().float() / SW


def superpoint_net_fp16(img_u8: np.ndarray, w: dict, accum: str = "f64", mutant: str | None = None):
    """img_u8 [H,W] uint8 -> (semi [H,W], desc [256,H/8,W/8]) of the plain-fp16 network, float64 arrays"""
    import torch
    import torch.nn.functional as F
    assert accum in ("f64", "f32") and (mutant is None or mutant in NET_MUTANTS)
    dt = torch.float64 if accum == "f64" else torch.float32
    rp = (lambda v: v) if mutant == "lo_read" else round_plane

    def conv(x, n, pad):
        wt, bt = _w16(w[n + ".weight"]), torch.from_numpy(np.asarray(w[n + ".bias"], np.float32))
        if mutant == "tap_missing" and n == "conv2a":
            wt = wt.clone(); wt[:, :, 0, 0] = 0
        if mutant == "slab_missing" and n == "conv3b":
            wt = wt.clone(); wt[:, :64] = 0
        return F.conv2d(x.to(dt), wt.to(dt), bt.to(dt), padding=pad)

    with torch.no_grad():
        x = torch.from_numpy(img_u8.astype(np.float32) * np.float32(1.0 / 255.0))[None, None]
        a = F.relu(F.conv2d(x, torch.from_numpy(w["conv1a.weight"]), torch.from_numpy(w["conv1a.bias"]), padding=1))
        x = rp(a)                                                   # conv1a (fp32) -> planes
        x = rp(F.max_pool2d(F.relu(conv(x, "conv1b", 1)), 2, 2))
        x = rp(F.relu(conv(x, "conv2a", 1)))
        x = rp(F.max_pool2d(F.relu(conv(x, "conv2b", 1)), 2, 2))
        x = rp(F.relu(conv(x, "conv3a", 1)))
        x = rp(F.max_pool2d(F.relu(conv(x, "conv3b", 1)), 2, 2))
        x = rp(F.relu(conv(x, "conv4a", 1)))
        x = rp(F.relu(conv(x, "conv4b", 1)))
        cpa = rp(F.relu(conv(x, "convPa", 1)))
        semi = conv(cpa, "convPb", 0).float()                       # fp32 logits -> fp32 softmax
        cda = rp(F.relu(conv(x, "convDa", 1)))
        desc = conv(cda, "convDb", 0).float()
        desc = desc / torch.norm(desc, p=2, dim=1, keepdim=True)
        semi = torch.softmax(semi, 1)[:, :64].permute(0, 2, 3, 1)
        Hc, Wc = semi.shape[1], semi.shape[2]
        semi = semi.reshape(-1, Hc, Wc, 8, 8).permute(0, 1, 3, 2, 4).reshape(-1, Hc * 8, Wc * 8)
    return semi[0].double().numpy(), desc[0].double().numpy()


def netvlad_net_fp16(img_u8: np.ndarray, w: dict, accum: str = "f64", mutant: str | None = None) -> np.ndarray:
    """img_u8 [H,W] uint8 -> the 4096-vector of the plain-fp16 network (float64 array)"""
    import torch
    import torch.nn.functional as F
    from omniswarm_b200 import synth
    assert accum in ("f64", "f32") and (mutant is None or mutant in NET_MUTANTS)
    dt = torch.float64 if accum == "f64" else torch.float32
    t = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in w.items()}
    relu6 = lambda v: torch.clamp(v, 0.0, 6.0)
    rp = (lambda v: v) if mutant == "lo_read" else round_plane

    def pointwise(x, n):
        wt = _w16(w[n + ".weight"])
        if mutant == "slab_missing" and n == "b3.pw":
            wt = wt.clone(); wt[:, :64] = 0
        if mutant == "tap_missing" and n == "proj":
            wt = wt.clone(); wt[:, :64] = 0
        return F.conv2d(x.to(dt), wt.to(dt), t[n + ".bias"].to(dt)).float()

    with torch.no_grad():
        x = torch.from_numpy(img_u8.astype(np.float32))[None, None] * np.float32(synth.NV_INPUT_SCALE)
        x = relu6(F.conv2d(x, t["conv0.weight"], t["conv0.bias"], stride=2, padding=1))
        for i, (ci, co, s) in enumerate(synth.NV_BLOCKS):
            d = relu6(F.conv2d(x, t[f"b{i}.dw.weight"], t[f"b{i}.dw.bias"], stride=s, padding=1, groups=ci))
            if i == 0:                                              # block 0: fused fp32 kernel, no planes
                x = relu6(F.conv2d(d, t["b0.pw.weight"], t["b0.pw.bias"]))
            else:
                x = relu6(pointwise(rp(d), f"b{i}.pw"))
        x = pointwise(rp(x), "proj")                       # block 6 output -> planes -> projection (fp32 out)
        x = x - x.mean(dim=(2, 3), keepdim=True)
        x = x / torch.clamp(torch.norm(x, dim=1, keepdim=True), min=1e-12)
        a = torch.softmax(F.conv2d(x, t["assign.weight"], t["assign.bias"]), 1)
        D, K = x.shape[1], a.shape[1]
        vlad = a.reshape(K, -1) @ x.reshape(D, -1).t() - a.reshape(K, -1).sum(1, keepdim=True) * t["centroids"]
        vlad = vlad / torch.clamp(torch.norm(vlad, dim=1, keepdim=True), min=1e-12)
        v = vlad.reshape(-1)
        v = v / torch.clamp(torch.norm(v), min=1e-12)
    return v.double().numpy()


def rel(a, b) -> float:
    """|a - b| / |b| (L2 over the whole array)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def network_tolerances(images, wsp: dict, wnv: dict) -> dict:
    """{semi, desc, vlad}: NET_TOL_FACTOR x the largest relative L2 difference, over `images`, between the float64 and
    the float32-accumulated emulation"""
    d = {"semi": 0.0, "desc": 0.0, "vlad": 0.0}
    for img in images:
        s64, d64 = superpoint_net_fp16(img, wsp, "f64")
        s32, d32 = superpoint_net_fp16(img, wsp, "f32")
        d["semi"] = max(d["semi"], rel(s32, s64))
        d["desc"] = max(d["desc"], rel(d32, d64))
        d["vlad"] = max(d["vlad"], rel(netvlad_net_fp16(img, wnv, "f32"), netvlad_net_fp16(img, wnv, "f64")))
    return {k: NET_TOL_FACTOR * v for k, v in d.items()}
