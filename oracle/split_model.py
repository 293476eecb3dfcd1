"""ORACLE (test infrastructure, NOT product code) -- numpy model of the split-fp16 tensor-core convolution
(omni-swarm_b200/csrc/conv_umma.cu).

Every fp32 operand x is carried as two fp16 planes hi = fp16(s*x), lo = fp16(s*x - hi) (s a power of two); each 16-wide
K step of the kernel issues three MMAs: hi*hi into a MAIN accumulator, hi*lo and then lo*hi into a CROSS accumulator,
both fp32.  The model forms the exact products of each step (float64), adds them to the accumulator and rounds the sum
to fp32, to nearest or toward zero; the K steps run in the kernel's order (horizontal tap kx, 64-channel slab, vertical
tap ky, 16 channels).  The epilogue is the kernel's fmaf((main + cross), 1 / (s_a * s_w), bias), then the activation and
the 2x2 max-pool.

`mutant` switches in one defect of the kind an indexing or descriptor error produces, so that a test can show a
tolerance separates correct from wrong arithmetic:
  drop_hilo / drop_lohi   one cross product never issued
  act_lo_slab / w_lo_slab the lo plane of one 64-channel slab of one tap (tap 0, the last slab) read as zero
  tap_missing             tap 0 skipped
  kx_shift                the box of horizontal tap 0 fetched one column to the right
  halo_off                every box fetched one row low (vertical halo off by one)
  nsplit_rows             the second 128-channel work item of a layer wider than 128 reads the first item's weight rows
"""
from __future__ import annotations

import numpy as np

FP16_MAX_FINITE_SPLIT = 65520.0      # fp16 rounds |v| >= 65520 to inf
# The bound of the GPU layer tests: |y - y64| <= TAU * (sum |x| |w| + |b|) per output element, y64 the float64 convolution
# of the dequantised operands.  tests/test_split_model.py shows that the faithful model stays below TAU / 4 and every
# mutant exceeds TAU; DESIGN.md section 4 lists what an H100 measures against it.
TAU = 6e-6
KC = 64                              # channels per slab (one 128-byte swizzle row of fp16)
KSTEP = 16                           # K of one wgmma

MUTANTS = ("drop_hilo", "drop_lohi", "act_lo_slab", "w_lo_slab", "tap_missing", "kx_shift", "halo_off", "nsplit_rows")


def split(x, scale: float):
    """fp32 -> (hi, lo) fp16 planes of scale * x, as the kernels split (round to nearest even, like __float2half_rn)."""
    s = np.asarray(x, np.float32) * np.float32(scale)
    with np.errstate(over="ignore", invalid="ignore"):
        hi = s.astype(np.float16)
        lo = (s - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def dequant(hi, lo, scale: float) -> np.ndarray:
    """the value the planes represent, float64"""
    return (np.asarray(hi, np.float64) + np.asarray(lo, np.float64)) / scale


def split_weights(w_oihw, w_scale: float):
    """OIHW fp32 -> (hi, lo) [taps][cout][cin] (the layout umma_layer_upload writes, without the row padding)"""
    w = np.asarray(w_oihw, np.float32)
    co, ci, kh, kw = w.shape
    t = np.ascontiguousarray(w.reshape(co, ci, kh * kw).transpose(2, 0, 1))
    return split(t, w_scale)


def round_f32(v: np.ndarray, mode: str) -> np.ndarray:
    """float64 -> the nearest fp32 ("rn") or the fp32 next toward zero ("rz"), returned as float64"""
    r = v.astype(np.float32)
    if mode == "rz":
        over = np.abs(r.astype(np.float64)) > np.abs(v)
        r = np.where(over, np.nextafter(r, np.float32(0)), r)
    return r.astype(np.float64)


def conv_model(x_hi, x_lo, w_hi, w_lo, bias, ks: int, act_scale: float, w_scale: float, relu: int = 0, pool: int = 0,
               rounding: str = "rz", mutant: str | None = None) -> np.ndarray:
    """x planes [B,H,W,Cin], weight planes [taps][Cout][Cin] -> fp32 output [B,Ho,Wo,Cout] (float64 array of fp32 values)."""
    assert mutant is None or mutant in MUTANTS
    xh, xl = np.asarray(x_hi, np.float64), np.asarray(x_lo, np.float64)
    wh, wl = np.asarray(w_hi, np.float64).copy(), np.asarray(w_lo, np.float64).copy()
    B, H, W, cin = xh.shape
    taps, cout, _ = wh.shape
    assert taps == ks * ks and cin % KC == 0
    halo = ks // 2
    slabs = cin // KC
    if mutant == "nsplit_rows":
        assert cout >= 256, "nsplit_rows needs a layer of more than 128 output channels"
        wh[:, 128:256], wl[:, 128:256] = wh[:, :128], wl[:, :128]
    pad = halo + 1                                     # one extra so that the shifted mutants stay in the padded frame
    xph = np.zeros((B, H + 2 * pad, W + 2 * pad, cin)); xph[:, pad:pad + H, pad:pad + W] = xh
    xpl = np.zeros_like(xph); xpl[:, pad:pad + H, pad:pad + W] = xl
    main = np.zeros((B, H, W, cout))
    cross = np.zeros((B, H, W, cout))
    for kx in range(ks):
        dx = kx - halo + (1 if mutant == "kx_shift" and kx == 0 else 0)
        for cs in range(slabs):
            for ky in range(ks):
                t = ky * ks + kx
                if mutant == "tap_missing" and t == 0:
                    continue
                dy = ky - halo + (1 if mutant == "halo_off" else 0)
                ah = xph[:, pad + dy:pad + dy + H, pad + dx:pad + dx + W]
                al = xpl[:, pad + dy:pad + dy + H, pad + dx:pad + dx + W]
                lo_gone = t == 0 and cs == slabs - 1
                for k in range(KC // KSTEP):
                    c = slice(cs * KC + k * KSTEP, cs * KC + (k + 1) * KSTEP)
                    a_h, a_l, b_h, b_l = ah[..., c], al[..., c], wh[t, :, c], wl[t, :, c]
                    if mutant == "act_lo_slab" and lo_gone:
                        a_l = np.zeros_like(a_l)
                    if mutant == "w_lo_slab" and lo_gone:
                        b_l = np.zeros_like(b_l)
                    main = round_f32(main + a_h @ b_h.T, rounding)
                    if mutant != "drop_hilo":
                        cross = round_f32(cross + a_h @ b_l.T, rounding)
                    if mutant != "drop_lohi":
                        cross = round_f32(cross + a_l @ b_h.T, rounding)
    inv = 1.0 / (act_scale * w_scale)                  # a power of two: the product is exact
    y = round_f32(round_f32(main + cross, "rn") * inv + np.asarray(bias, np.float32).astype(np.float64), "rn")
    if relu:
        y = np.maximum(y, 0.0)
    if relu == 2:
        y = np.minimum(y, 6.0)
    if pool:
        y = y.reshape(B, H // 2, 2, W // 2, 2, cout).max(axis=(2, 4))
    return y


REGIMES = ("relu_gauss", "signed", "ramp", "sparse_w", "bias_dominant")
ACT_LIMIT = FP16_MAX_FINITE_SPLIT / 16.0             # 4095: activations at the networks' x16 plane scale


def make_case(regime: str, B: int, H: int, W: int, cin: int, cout: int, ks: int, seed: int = 0):
    """seeded layer operands (x [B,H,W,cin], w [cout,cin,ks,ks], bias [cout], all fp32) in one of the value regimes:
      relu_gauss     ReLU'd Gaussian activations, Gaussian weights of the synthetic networks' size
      signed         signed Gaussian activations
      ramp           activation magnitude growing geometrically with the channel, from 2^-12 to just below the plane
                     limit (the last slab dominates every sum); weights scaled so that the outputs stay below it too
      sparse_w       a third of the weights exactly zero and a tenth of magnitude 1e-6
      bias_dominant  a bias 30 times the size of the sum (at most 1000, below the plane limit)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, H, W, cin))
    w = rng.standard_normal((cout, cin, ks, ks)) * (1.5 / np.sqrt(cin * ks * ks))
    b = rng.standard_normal(cout) * 0.05
    if regime in ("relu_gauss", "sparse_w", "bias_dominant"):
        x = np.maximum(x, 0.0)
    if regime == "ramp":
        mag = 2.0 ** (-12.0 + 23.9 * np.arange(cin) / max(cin - 1, 1))
        x = mag * rng.uniform(0.5, 1.0, (B, H, W, cin))
        worst = (np.abs(w) * mag[None, :, None, None]).sum(axis=(1, 2, 3)).max()
        w *= min(1.0, 2000.0 / worst)
    if regime == "sparse_w":
        u = rng.uniform(size=w.shape)
        w[u < 0.33] = 0.0
        w[(u >= 0.33) & (u < 0.43)] = 1e-6 * np.sign(w[(u >= 0.33) & (u < 0.43)])
    if regime == "bias_dominant":
        b = np.sign(b) * np.minimum(30.0 * np.abs(x).mean() * np.abs(w).sum(axis=(1, 2, 3)), 1000.0)
    return x.astype(np.float32), w.astype(np.float32), b.astype(np.float32)


def conv_f64(x, w_oihw, bias, ks: int) -> tuple[np.ndarray, np.ndarray]:
    """(y, d): the exact convolution of x [B,H,W,Cin] with w (both float64, zero padding ks // 2) plus bias, and the
    scale of its rounding error d = sum |x| |w| + |b| per output element; both [B,H,W,Cout]"""
    import torch
    import torch.nn.functional as F
    xt = torch.from_numpy(np.ascontiguousarray(np.asarray(x, np.float64).transpose(0, 3, 1, 2)))
    wt = torch.from_numpy(np.asarray(w_oihw, np.float64))
    bt = torch.from_numpy(np.asarray(bias, np.float64))
    y = F.conv2d(xt, wt, bt, padding=ks // 2)
    d = F.conv2d(xt.abs(), wt.abs(), bt.abs(), padding=ks // 2)
    return y.numpy().transpose(0, 2, 3, 1), d.numpy().transpose(0, 2, 3, 1)
