"""The embedder's fused InstanceNorm (+ residual) (+ ReLU) kernels against an fp64 norm of their OWN fp32 input, element by
element, on planes shaped like slide tiles.

`test_zz_embedder_gpu.py` compares the kernels with fp32 `F.instance_norm` on i.i.d. random planes, where no pixel sits
far from its plane's mean.  Slide tiles are different: most of a tile is flat background, and the corner pixel, which
sees the most zero padding in every convolution, is an outlier of its plane.  Here each plane is normalised in fp64
(mean mu, biased variance var, r = 1/sqrt(var + eps), y64 = [relu]((x - mu) r [+ res])) and every output must satisfy
(u = 2^-24)

    |y - y64| <= r e_mu + |x - mu| r e_v / (2 (var + eps)) + 4 u (|y64| + |res|),
    e_mu = C_BAR L u mean|x|,   e_v = C_BAR L u var + e_mu^2,

where L is the longest fp32 addition chain of the kernel that runs the plane (mirrored below from embed_kernels.cuh):
k_instnorm_plane ceil(HW / 256) + 8 (its strided per-thread chain and block_sum_256), k_instnorm_warp 32 + 5 (32
registers, 5 shuffles), k_instnorm_nhwc ceil(HW / 16) + 16 (the per-thread chain and the 16-partial merge).  The bar is
relative to var itself, never to a pixel's distance from the mean; ReLU is 1-Lipschitz, so the same bar covers it.

CPU part: fp32 restatements of each kernel's reduction order stay 4x under every bar on the synthetic planes; the
one-pass statistics shifted by the first pixel (S2 - S1^2/HW, what k_instnorm_nhwc computed before it switched to
Welford + Chan) break the variance bar by more than 20x on first-pixel-outlier planes; and dropping or doubling any
probe pixel (pixel 0, the last pixel, the last pixel of every thread's / warp's strided chain, the .w of every
thread's last float4, register 31 of the warp kernel, the last warp's partial of the NHWC merge) moves an output by more
than 20x its bar.

GPU part: the planes every InstanceNorm2d of a seeded ResNet-18 sees on slide-like patches, synthetic planes at the
route edges, the probe planes, the fused network against its fp64 twin, and the embedding loop from JPEG files to the
'%.4f' CSV.  Measured maxima (error over bar) are in DESIGN §3.
"""
from __future__ import annotations

import copy
import math
import os
import re

import numpy as np
import pytest
import torch

U = 2.0 ** -24
EPS = 1e-5
C_BAR = 2.0                  # bar constant: the CPU part shows the fp32 restatements stay 4x under it
SENSITIVITY = 20.0
# mirrored from csrc/embed_kernels.cuh (checked below)
K_PLANE_THREADS, K_WARP_MAX_HW, K_NHWC_WARPS, K_NHWC_CHUNK, K_IN_PLANE_MAX = 256, 1024, 16, 8, 16384
SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dsmil_wsi_b200", "csrc",
                   "embed_kernels.cuh")

ROUTE_EDGES = (1, 2, 31, 32, 33, 1023, 1024, 1025, 1028, 12544, 16383, 16384)
NHWC_HWS = (1, 15, 16, 17, 12544, 50176)


def ceil_div(a, b):
    return -(-a // b)


def route(HW, nhwc, aligned=True):
    """Which kernel runs a plane of HW elements (launch_instnorm / dsmil_instnorm_act_nhwc)."""
    if nhwc:
        return "nhwc"
    if HW <= K_WARP_MAX_HW:
        return "warp"
    return "vec" if HW % 4 == 0 and aligned else "plane"


def chain_len(rt, HW):
    if rt == "nhwc":
        return ceil_div(HW, K_NHWC_WARPS) + K_NHWC_WARPS
    if rt == "warp":
        return 32 + 5
    # the variance pass is scalar-strided on both plane forms; the float4 sum chain (ceil(HW / 1024) + 2) is shorter
    return ceil_div(HW, K_PLANE_THREADS) + 8


# ------------------------------------------------------------------------------------------- fp64 norm and bars
def norm64(x, res, relu, eps=EPS, weight=None):
    """x [P, HW] (fp32, any device) -> (y64, mu, var, r) in fp64.  `weight` [P, HW] scales each pixel's share of the
    statistics (a pixel dropped or counted twice); the sums are still divided by HW."""
    xd = x.double()
    w = torch.ones_like(xd) if weight is None else weight.double()
    HW = x.shape[1]
    mu = (w * xd).sum(1, keepdim=True) / HW
    var = (w * (xd - mu).square()).sum(1, keepdim=True) / HW
    r = (var + eps).rsqrt()
    y = (xd - mu) * r
    if res is not None:
        y = y + res.double()
    if relu:
        y = y.clamp_min(0.0)
    return y, mu, var, r


def bars(x, res, y64, mu, var, r, L, eps=EPS):
    xd = x.double()
    e_mu = C_BAR * L * U * xd.abs().mean(1, keepdim=True)
    e_v = C_BAR * L * U * var + e_mu.square()
    b = r * e_mu + (xd - mu).abs() * r * e_v / (2.0 * (var + eps)) + 4.0 * U * y64.abs()
    if res is not None:
        b = b + 4.0 * U * res.double().abs()
    return b, e_v


def ratio(x, res, relu, y, L, eps=EPS):
    """max over the elements of |y - y64| / bar (0 where y == y64 exactly)."""
    y64, mu, var, r = norm64(x, res, relu, eps)
    b, _ = bars(x, res, y64, mu, var, r, L, eps)
    err = (y.double() - y64).abs()
    q = torch.where(err == 0, torch.zeros_like(err), err / b)
    return float(q.max())


# ------------------------------------------------------------------------------------------- synthetic planes
def synthetic(HW, seed=0):
    """{name: fp32 plane [HW]}: outliers at the first and last pixel, |mu| / sigma = 1e3, var ~ eps and 1e-3 eps,
    constant planes, and a plain normal plane."""
    g = np.random.default_rng(seed + HW)
    n = g.standard_normal(HW)
    out = {}
    bg = 0.3 + 1e-3 * n
    a = bg.copy(); a[0] = -2.0
    out["first_outlier"] = a
    a = bg.copy(); a[-1] = -2.0
    out["last_outlier"] = a
    a = bg.copy(); a[0] = 4.0; a[-1] = -3.0
    out["both_outliers"] = a
    out["mean_1e3_sigma"] = 1000.0 + n
    out["var_eps"] = 0.5 + math.sqrt(EPS) * n
    out["var_1e-3_eps"] = -0.25 + math.sqrt(1e-3 * EPS) * n
    out["constant"] = np.full(HW, 0.3)
    out["constant_neg"] = np.full(HW, -7.25)
    out["normal"] = 1.5 + 3.0 * n
    return {k: v.astype(np.float32) for k, v in out.items()}


def probes(rt, HW):
    """[(pixel, what)] of the probe pixels of route rt at HW; each asserts the chain boundary it sits on."""
    out = [(0, "pixel 0"), (HW - 1, "last pixel")]
    if rt == "plane":
        for t in range(min(K_PLANE_THREADS, HW)):
            p = t + K_PLANE_THREADS * (ceil_div(HW - t, K_PLANE_THREADS) - 1)
            assert p % K_PLANE_THREADS == t and p < HW <= p + K_PLANE_THREADS
            out.append((p, f"last pixel of thread {t}"))
    elif rt == "vec":
        n4 = HW // 4
        for t in range(min(K_PLANE_THREADS, n4)):
            i = t + K_PLANE_THREADS * (ceil_div(n4 - t, K_PLANE_THREADS) - 1)
            assert i % K_PLANE_THREADS == t and i < n4 <= i + K_PLANE_THREADS
            out.append((4 * i + 3, f".w of thread {t}'s last float4"))
    elif rt == "warp":
        for lane in range(min(32, HW)):
            p = lane + 32 * (ceil_div(HW - lane, 32) - 1)
            assert p % 32 == lane and p < HW <= p + 32
            out.append((p, f"last register of lane {lane}" + (" (register 31)" if p // 32 == 31 else "")))
    else:
        for w in range(min(K_NHWC_WARPS, HW)):
            p = w + K_NHWC_WARPS * (ceil_div(HW - w, K_NHWC_WARPS) - 1)
            assert p % K_NHWC_WARPS == w and p < HW <= p + K_NHWC_WARPS
            out.append((p, f"last pixel of warp {w}" + (" (the last partial merged)" if w == K_NHWC_WARPS - 1 else "")))
    return out


PROBE_SETS = [("warp", 33), ("warp", 1023), ("warp", 1024), ("plane", 1025), ("plane", 12544), ("plane", 16383),
              ("vec", 1028), ("vec", 12544), ("vec", 16384), ("nhwc", 17), ("nhwc", 12544), ("nhwc", 50176)]


def probe_planes(rt, HW, seed=1):
    """One plane per probe pixel: flat background with the probe pixel alone far from it."""
    ps = probes(rt, HW)
    g = np.random.default_rng(seed + HW)
    x = (0.3 + 1e-3 * g.standard_normal((len(ps), HW))).astype(np.float32)
    for k, (p, _) in enumerate(ps):
        x[k, p] = -2.0
    if rt == "warp":
        assert HW != 1024 or any("register 31" in w for _, w in ps)
    if rt == "nhwc":
        assert any("last partial merged" in w for _, w in ps) == (HW >= K_NHWC_WARPS)
    return ps, x


# ------------------------------------------------------------------------------------------- fp32 restatements
def f32(a):
    return np.asarray(a, dtype=np.float32)


def fma32(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def rsqrt32(v):
    return f32(1.0 / np.sqrt(np.asarray(v, np.float64)))


def warp_sum32(v):
    """common.cuh warp_sum over the last axis (32 lanes): xor butterfly, every lane ends with lanes 0..o-1's value."""
    for o in (16, 8, 4, 2, 1):
        v = v[..., :o] + v[..., o:2 * o]
    return v[..., 0]


def block_sum32(v):
    """block_sum_256 over the last axis (256 threads)."""
    s = warp_sum32(v.reshape(v.shape[:-1] + (8, 32)))
    return ((s[..., 0] + s[..., 1]) + (s[..., 2] + s[..., 3])) + ((s[..., 4] + s[..., 5]) + (s[..., 6] + s[..., 7]))


def _finish(x, res, relu, mean, rstd):
    y = (x - mean[:, None]) * rstd[:, None]
    if res is not None:
        y = y + res
    return np.maximum(y, f32(0.0)) if relu else y


def emu_plane(x, res, relu, vec, eps=EPS):
    P, HW = x.shape
    T = K_PLANE_THREADS
    acc = np.zeros((P, T), np.float32)
    if vec:
        n4 = HW // 4
        it = ceil_div(n4, T)
        xp = np.zeros((P, it * T * 4), np.float32); xp[:, :HW] = x
        xp = xp.reshape(P, it, T, 4)
        for k in range(it):
            v = xp[:, k]
            acc = acc + ((v[..., 0] + v[..., 1]) + (v[..., 2] + v[..., 3]))
    it = ceil_div(HW, T)
    xs = np.zeros((P, it * T), np.float32); xs[:, :HW] = x
    xs = xs.reshape(P, it, T)
    valid = (np.arange(it * T) < HW).reshape(it, T)
    if not vec:
        for k in range(it):
            acc = acc + xs[:, k]
    mean = block_sum32(acc) / f32(HW)
    sq = np.zeros((P, T), np.float32)
    for k in range(it):
        d = np.where(valid[k], xs[:, k] - mean[:, None], f32(0.0))
        sq = fma32(d, d, sq)
    var = block_sum32(sq) / f32(HW)
    return _finish(x, res, relu, mean, rsqrt32(var + f32(eps))), var


def emu_warp(x, res, relu, eps=EPS):
    P, HW = x.shape
    xp = np.zeros((P, 32 * 32), np.float32); xp[:, :HW] = x
    xp = xp.reshape(P, 32, 32)                                   # [plane, register j, lane]
    valid = (np.arange(1024) < HW).reshape(32, 32)
    acc = np.zeros((P, 32), np.float32)
    for j in range(32):
        acc = acc + xp[:, j]
    mean = warp_sum32(acc) / f32(HW)
    sq = np.zeros((P, 32), np.float32)
    for j in range(32):
        d = np.where(valid[j], xp[:, j] - mean[:, None], f32(0.0))
        sq = fma32(d, d, sq)
    var = warp_sum32(sq) / f32(HW)
    return _finish(x, res, relu, mean, rsqrt32(var + f32(eps))), var


def emu_nhwc(x, res, relu, shifted=False, eps=EPS):
    """k_instnorm_nhwc's statistics: per thread, Welford over pixels w, w + 16, ... in chunks of up to 8, and Chan's formula over the 16 partials in warp order (shifted=True: the replaced one-pass sums shifted by the
    first pixel)."""
    P, HW = x.shape
    W_ = K_NHWC_WARPS
    it = ceil_div(HW, W_)
    xp = np.zeros((P, it * W_), np.float32); xp[:, :HW] = x
    xp = xp.reshape(P, it, W_)
    valid = (np.arange(it * W_) < HW).reshape(it, W_)
    a = np.zeros((P, W_), np.float32)
    b = np.zeros((P, W_), np.float32)
    if shifted:
        x0 = x[:, :1]
        for k in range(it):
            d = xp[:, k] - x0
            a = np.where(valid[k], a + d, a)
            b = np.where(valid[k], fma32(d, d, b), b)
        s1 = np.zeros(P, np.float32); s2 = np.zeros(P, np.float32)
        for w in range(W_):
            s1 = s1 + a[:, w]; s2 = s2 + b[:, w]
        inv = f32(1.0) / f32(HW)
        dm = s1 * inv
        mean = x0[:, 0] + dm
        var = np.maximum(fma32(-dm, s1, s2) * inv, f32(0.0))
    else:
        for w in range(min(W_, HW)):
            vals = x[:, w::W_]
            mean_w = np.zeros(P, np.float32); m2_w = np.zeros(P, np.float32)
            cnt, n = 0, vals.shape[1]
            while cnt < n:
                t = min(K_NHWC_CHUNK, n - cnt)
                v = np.zeros((P, K_NHWC_CHUNK), np.float32)
                v[:, :t] = vals[:, cnt:cnt + t]
                mc = (((v[:, 0] + v[:, 1]) + (v[:, 2] + v[:, 3])) + ((v[:, 4] + v[:, 5]) + (v[:, 6] + v[:, 7]))) / f32(t)
                q = np.zeros(P, np.float32)
                for k in range(t):
                    d = v[:, k] - mc
                    q = fma32(d, d, q)
                f = f32(t) / f32(cnt + t)
                d = mc - mean_w
                mean_w = fma32(d, f, mean_w)
                m2_w = fma32(d * d, f32(cnt) * f, m2_w + q)
                cnt += t
            a[:, w], b[:, w] = mean_w, m2_w
        nw = [f32(ceil_div(HW - w, W_)) if w < HW else f32(0.0) for w in range(W_)]
        s = np.zeros(P, np.float32)
        for w in range(W_):
            s = fma32(nw[w], a[:, w], s)
        mean = s / f32(HW)
        m2 = np.zeros(P, np.float32)
        for w in range(W_):
            d = a[:, w] - mean
            m2 = m2 + fma32(nw[w] * d, d, b[:, w])
        var = m2 / f32(HW)
    return _finish(x, res, relu, mean, rsqrt32(var + f32(eps))), var


def emulate(rt, x, res, relu):
    if rt == "nhwc":
        return emu_nhwc(x, res, relu)
    if rt == "warp":
        return emu_warp(x, res, relu)
    return emu_plane(x, res, relu, vec=(rt == "vec"))


# ===================================================================================================== CPU part
def test_mirrored_constants_match_the_sources():
    s = open(SRC).read()
    assert re.search(rf"kNhwcChunk\s*=\s*{K_NHWC_CHUNK};", s)
    assert re.search(rf"kNhwcWarps\s*=\s*{K_NHWC_WARPS};", s) and re.search(rf"kInPlaneMax\s*=\s*{K_IN_PLANE_MAX};", s)
    assert "if (HW <= 1024)" in s and s.count("__launch_bounds__(256)") == 2
    assert "float v[32];" in s and "((s_red[0] + s_red[1]) + (s_red[2] + s_red[3]))" in s
    assert "(HW % 4 == 0)" in s


def _cpu_cases():
    for HW in ROUTE_EDGES:
        rts = ["warp"] if HW <= K_WARP_MAX_HW else (["plane", "vec"] if HW % 4 == 0 else ["plane"])
        for rt in rts:
            yield rt, HW
    for HW in NHWC_HWS:
        yield "nhwc", HW


@pytest.mark.parametrize("rt,HW", list(_cpu_cases()))
def test_norm64_is_instance_norm_and_restatements_stay_under_a_quarter_of_the_bars(rt, HW):
    planes = synthetic(HW)
    x = np.stack(list(planes.values()))
    xt = torch.from_numpy(x)
    g = np.random.default_rng(HW)
    res = torch.from_numpy(g.standard_normal(x.shape).astype(np.float32))
    # the fp64 restatement is F.instance_norm in float64
    y64, mu, var, r = norm64(xt, None, False)
    # (F.instance_norm refuses one-element planes; their output is exactly 0)
    want = torch.nn.functional.instance_norm(xt.double()[None], eps=EPS)[0] if HW > 1 else torch.zeros_like(y64)
    assert torch.allclose(y64, want, rtol=1e-11, atol=1e-11)
    L = chain_len(rt, HW)
    for rs, relu in ((None, True), (res, False), (res, True)):
        y, _ = emulate(rt, x, None if rs is None else rs.numpy(), relu)
        q = ratio(xt, rs, relu, torch.from_numpy(y), L)
        assert q <= 0.25, (rt, HW, q)


@pytest.mark.parametrize("HW", [3136, 12544, 50176])
def test_first_pixel_shifted_sums_break_the_variance_bar(HW):
    """The case set catches the replaced NHWC statistics: sums shifted by the first pixel lose a factor
    1 + (x0 - mu)^2 / var, which a first-pixel outlier makes ~HW."""
    planes = synthetic(HW)
    x = np.stack([planes["first_outlier"]])
    xt = torch.from_numpy(x)
    _, v_old = emu_nhwc(x, None, True, shifted=True)
    _, v_new = emu_nhwc(x, None, True)
    y64, mu, var, r = norm64(xt, None, True)
    _, e_v = bars(xt, None, y64, mu, var, r, chain_len("nhwc", HW))
    old = (torch.from_numpy(v_old).double()[:, None] - var).abs() / e_v
    new = (torch.from_numpy(v_new).double()[:, None] - var).abs() / e_v
    assert float(old.min()) > SENSITIVITY, old
    assert float(new.max()) <= 0.25, new


@pytest.mark.parametrize("rt,HW", PROBE_SETS)
def test_probe_pixels_carry_weight(rt, HW):
    """Dropping or doubling any probe pixel's share of the statistics moves an output by > 20x its bar."""
    ps, x = probe_planes(rt, HW)
    xt = torch.from_numpy(x)
    L = chain_len(rt, HW)
    y64, mu, var, r = norm64(xt, None, False)
    b, _ = bars(xt, None, y64, mu, var, r, L)
    for wv in (0.0, 2.0):
        w = torch.ones_like(xt, dtype=torch.float64)
        w[torch.arange(len(ps)), torch.tensor([p for p, _ in ps])] = wv
        y2, *_ = norm64(xt, None, False, weight=w)
        moved = ((y2 - y64).abs() / b).amax(1)
        worst = int(moved.argmin())
        assert float(moved[worst]) > SENSITIVITY, (rt, HW, wv, ps[worst], float(moved[worst]))
    # and the restatement of the route itself stays under a quarter of the bars on these planes
    y, _ = emulate(rt, x, None, False)
    assert ratio(xt, None, False, torch.from_numpy(y), L) <= 0.25


# ===================================================================================================== GPU part
def _layout(nhwc):
    return torch.channels_last if nhwc else torch.contiguous_format


def _run(x, res, relu, nhwc, inplace=False, offset=None):
    """instnorm_act on x [N, C, H, W] (fp32 values) in the given layout; returns (y as NCHW planes, route).
    offset='x' / 'res': that operand starts one float past a 16-byte boundary (the scalar plane kernel)."""
    from dsmil_wsi_b200 import _lib
    from dsmil_wsi_b200 import functional as Fn
    from dsmil_wsi_b200.embedder import instnorm_act
    N, Cc, H, W = x.shape
    HW = H * W
    fmt = _layout(nhwc)
    xi = x.contiguous(memory_format=fmt)
    ri = None if res is None else res.contiguous(memory_format=fmt)
    if offset == "x":
        xi = torch.empty(x.numel() + 1, device=x.device)[1:].view(x.shape).copy_(x)
    if offset == "res":
        ri = torch.empty(res.numel() + 1, device=x.device)[1:].view(res.shape).copy_(res)
    aligned = offset is None
    if offset is not None:
        assert not nhwc and (xi if offset == "x" else ri).data_ptr() % 16 == 4
    rt = route(HW, nhwc, aligned)
    if nhwc and (HW == 1 or Cc == 1):
        # [N, C, 1, 1] is both layouts and instnorm_act takes it as NCHW: call the channels-last entry itself
        assert not inplace
        y = torch.empty_like(xi)
        _lib.check(_lib.load().dsmil_instnorm_act_nhwc(xi.data_ptr(), Fn._ptr(ri), y.data_ptr(), N, HW, Cc, EPS,
                                                        int(relu), Fn._stream()), "dsmil_instnorm_act_nhwc")
    elif inplace:
        xi = xi.clone(memory_format=fmt) if offset != "x" else xi
        y = instnorm_act(xi, ri, relu, out=xi)
        assert y.data_ptr() == xi.data_ptr()
    else:
        y = instnorm_act(xi, ri, relu)
    if nhwc and HW > 1:
        assert y.is_contiguous(memory_format=torch.channels_last) and not y.is_contiguous()
    return y.contiguous().view(N * Cc, HW), rt


def _check(x, res, relu, nhwc, **kw):
    y, rt = _run(x, res, relu, nhwc, **kw)
    N, Cc, H, W = x.shape
    xp = x.contiguous().view(N * Cc, H * W)
    rp = None if res is None else res.contiguous().view(N * Cc, H * W)
    return ratio(xp, rp, relu, y, chain_len(rt, H * W)), rt


# ------------------------------------------------------------------------------------------- slide-like patches
def slide_patches(hw=224):
    """uint8 [6, hw, hw, 3]: flat background, background with a tissue blob, tissue in one corner, a tissue edge
    along the diagonal, uniform noise (what the other tests feed), a near-black patch."""
    g = np.random.default_rng(7)
    yy, xx = np.mgrid[0:hw, 0:hw].astype(np.float64)
    bg = np.array([0.94, 0.92, 0.95]) * 255.0
    tissue = np.array([0.80, 0.45, 0.66]) * 255.0

    def mix(mask):
        tex = g.normal(0.0, 14.0, (hw, hw, 3))
        img = bg * (1.0 - mask[..., None]) + (tissue + tex) * mask[..., None]
        return np.clip(np.rint(img), 0, 255).astype(np.uint8)

    def disk(cy, cx, rad):
        return 1.0 / (1.0 + np.exp((np.hypot(yy - cy, xx - cx) - rad) / 4.0))
    out = [np.broadcast_to(np.rint(bg).astype(np.uint8), (hw, hw, 3)).copy(),
           mix(disk(hw * 0.55, hw * 0.45, hw * 0.2)),
           mix(disk(hw, hw, hw * 0.45)),
           mix(1.0 / (1.0 + np.exp(-(xx - yy) / 3.0))),
           g.integers(0, 256, (hw, hw, 3)).astype(np.uint8),
           np.clip(np.rint(g.normal(6.0, 2.0, (hw, hw, 3))), 0, 255).astype(np.uint8)]
    return np.stack(out)


PATCH_NAMES = ("background", "blob", "corner", "diagonal", "uniform_noise", "near_black")


def _resnet():
    import torchvision.models as models
    torch.manual_seed(0)
    m = models.resnet18(weights=None, norm_layer=torch.nn.InstanceNorm2d)
    m.fc = torch.nn.Identity()
    for p in m.parameters():
        p.requires_grad = False
    return m.eval()


class _NoTF32:
    def __enter__(self):
        self.c, self.m = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.c, self.m


def _patch_batch(u8):
    return torch.from_numpy(u8).permute(0, 3, 1, 2).float().div(255.0).contiguous()    # == VF.to_tensor per image


_REAL = {}


def _real_planes():
    """The input of every InstanceNorm2d of the seeded ResNet-18 (fp32, on the device) on the slide-like patches."""
    if "x" not in _REAL:
        m = _resnet().cuda()
        rec = []
        hooks = [mod.register_forward_pre_hook(lambda mod, inp: rec.append(inp[0].detach().clone()))
                 for mod in m.modules() if isinstance(mod, torch.nn.InstanceNorm2d)]
        with _NoTF32(), torch.no_grad():
            m(_patch_batch(slide_patches()).cuda())
        for h in hooks:
            h.remove()
        assert len(rec) == 20
        _REAL["x"] = rec
    return _REAL["x"]


@pytest.mark.gpu
@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "channels_last"])
def test_real_planes_of_slide_patches(nhwc):
    planes = _real_planes()
    assert {p.shape[2] for p in planes} == {112, 56, 28, 14, 7}
    g = torch.Generator(device="cuda").manual_seed(3)
    worst = {}
    for k, x in enumerate(planes):
        assert x.shape[1] % 32 == 0
        res = torch.randn(x.shape, generator=g, device="cuda") * x.std()
        for relu, rs, inplace in ((True, None, False), (False, res, False), (True, res, True)):
            q, rt = _check(x, rs, relu, nhwc, inplace=inplace)
            assert q <= 1.0, (k, tuple(x.shape), relu, rs is not None, inplace, rt, q)
            worst[rt] = max(worst.get(rt, 0.0), q)
    print(f"real planes {'channels_last' if nhwc else 'nchw'}: max err / bar {worst}")


def _synthetic_batch(HW, C):
    """[1, C, 1, HW]: the synthetic planes of this HW, filled up to C channels with normal planes."""
    pl = list(synthetic(HW).values())
    g = np.random.default_rng(HW + C)
    while len(pl) < C:
        pl.append((2.0 + g.standard_normal(HW)).astype(np.float32))
    return torch.from_numpy(np.stack(pl[:C]))[None, :, None, :].cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("HW", ROUTE_EDGES)
def test_synthetic_planes_nchw(HW):
    x = _synthetic_batch(HW, 9)
    res = torch.randn(x.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(HW))
    worst = 0.0
    for relu, rs, inplace in ((True, None, False), (False, None, False), (True, res, False), (False, res, True)):
        q, rt = _check(x, rs, relu, False, inplace=inplace)
        assert q <= 1.0, (HW, relu, rs is not None, inplace, rt, q)
        worst = max(worst, q)
    if HW > K_WARP_MAX_HW and HW % 4 == 0:               # one float past alignment forces the scalar plane kernel
        for off in ("x", "res"):
            q, rt = _check(x, res, True, False, offset=off)
            assert rt == "plane" and q <= 1.0, (HW, off, q)
            worst = max(worst, q)
    print(f"synthetic nchw HW={HW}: max err / bar {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("C", [32, 64, 2048])
@pytest.mark.parametrize("HW", NHWC_HWS)
def test_synthetic_planes_channels_last(HW, C):
    if HW == 50176 and C == 2048:
        pytest.skip("covered at C = 32 and 64 (a 400 MB plane set)")
    x = _synthetic_batch(HW, C)
    x = x.view(1, C, 1, HW) if HW != 50176 else x.view(1, C, 224, 224)
    res = torch.randn(x.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(HW + C))
    worst = 0.0
    for relu, rs, inplace in ((True, None, False), (False, None, False), (True, res, False), (False, res, True)):
        if HW == 1 and inplace:
            continue
        q, rt = _check(x, rs, relu, True, inplace=inplace)
        assert rt == "nhwc" and q <= 1.0, (HW, C, relu, rs is not None, inplace, q)
        worst = max(worst, q)
    print(f"synthetic channels_last HW={HW} C={C}: max err / bar {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("rt,HW", PROBE_SETS)
def test_probe_planes(rt, HW):
    ps, x = probe_planes(rt, HW)
    P = len(ps)
    nhwc = rt == "nhwc"
    C = ceil_div(P, 32) * 32 if nhwc else P
    xt = torch.from_numpy(x)
    if C > P:                                             # fill the channel groups with normal planes
        xt = torch.cat([xt, 1.0 + torch.randn(C - P, HW, generator=torch.Generator().manual_seed(HW))])
    xt = xt[None, :, None, :].cuda()
    kw = {"offset": "x"} if rt == "plane" and HW % 4 == 0 else {}
    q, got = _check(xt, None, False, nhwc, **kw)
    assert got == rt and q <= 1.0, (rt, HW, q)
    print(f"probe planes {rt} HW={HW}: max err / bar {q:.3g}")


# ------------------------------------------------------------------------------------------- whole network
def _net_bars(u8):
    """(fp32 batch on the device, fp64 features, per-patch bar): bar = max(4 x the untouched fp32 module's distance
    to fp64, 2e-6 x max |f64|) per patch."""
    m = _resnet().cuda()
    x = _patch_batch(u8).cuda()
    with _NoTF32(), torch.no_grad():
        f32_ = m(x).double()
        f64 = copy.deepcopy(m).double()(x.double())
    own = (f32_ - f64).abs().amax(1)
    bar = torch.maximum(4.0 * own, 2e-6 * f64.abs().amax(1))
    return m, x, f64, bar, own


@pytest.mark.gpu
@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "channels_last"])
def test_fused_network_against_fp64(nhwc):
    from dsmil_wsi_b200.embedder import fuse_instance_norm
    m, x, f64, bar, own = _net_bars(slide_patches())
    fused = copy.deepcopy(m)
    assert fuse_instance_norm(fused) == 20
    if nhwc:
        fused = fused.to(memory_format=torch.channels_last)
        x = x.contiguous(memory_format=torch.channels_last)
    with _NoTF32(), torch.no_grad():
        f = fused(x).double()
    err = (f - f64).abs().amax(1)
    print(f"network {'channels_last' if nhwc else 'nchw'}: err / bar per patch "
          f"{dict(zip(PATCH_NAMES, (err / bar).tolist()))}; untouched fp32 rel {(own / f64.abs().amax(1)).tolist()}")
    assert bool((err <= bar).all()), dict(zip(PATCH_NAMES, (err / bar).tolist()))


@pytest.mark.gpu
def test_embedding_loop_from_jpeg_files_against_fp64(tmp_path):
    """compute_feats with its defaults (device JPEG decode, channels-last, CUDA graph) on the patches saved as
    quality-70 JPEGs (deepzoom_tiler.py), against the fp64 module on the PIL-decoded patches; the '%.4f' CSV holds
    round(f64, 4) except where f64 lies within the bar of a rounding boundary."""
    import pandas as pd
    from PIL import Image
    import dsmil as mil
    from dsmil_wsi_b200.embed import compute_feats, list_patches
    bag = tmp_path / "WSI" / "ds" / "single" / "c0" / "slideA"
    bag.mkdir(parents=True)
    u8 = slide_patches()
    for i in range(8):                                    # 4 full batches of 2: the graph is captured
        Image.fromarray(u8[i % len(u8)]).save(bag / f"{i}_{i}.jpeg", quality=70)
    paths = list_patches(str(bag))
    dec = np.stack([np.asarray(Image.open(p).convert("RGB")) for p in paths])
    m, _, f64, bar, _ = _net_bars(dec)
    ic = mil.IClassifier(copy.deepcopy(m), 512, output_class=2).cuda().eval()
    got = {}

    class A:
        batch_size, num_workers = 2, 2
    with _NoTF32():
        compute_feats(A(), [str(bag)], ic, save_path=str(tmp_path / "out"),
                      sink=lambda d, f, c: got.update(feats=f.double().clone()))
    assert getattr(ic.feature_extractor, "_dsmil_channels_last", False)
    err = (got["feats"] - f64).abs().amax(1)
    print(f"loop: err / bar per patch {(err / bar).tolist()}")
    assert bool((err <= bar).all()), (err / bar).tolist()
    csv = pd.read_csv(tmp_path / "out" / "c0" / "slideA.csv").to_numpy()
    ref = f64.cpu().numpy()
    s = ref * 1e4
    near = np.abs(s - (np.floor(s) + 0.5)) * 1e-4 <= bar.cpu().numpy()[:, None]
    assert np.array_equal(np.rint(csv * 1e4)[~near], np.rint(s)[~near])
