"""Helpers for the -m gpu parity tests (all calls go through the C ABI via ctypes)."""
import ctypes

import numpy as np
import torch

from ivid_b200 import _lib


def rel(a, b):
    a = a.double(); b = b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def report(name, got, want):
    got = got.detach().float().cpu(); want = want.detach().float().cpu()
    d = (got - want).abs()
    r = rel(got, want)
    print(f"[parity] {name}: rel_l2={r:.3e} max_abs={float(d.max()):.3e} ref_rms={float(want.pow(2).mean().sqrt()):.3e} "
          f"nan={int(torch.isnan(got).sum())} shape={tuple(got.shape)}")
    return r


def conv2d(act_nhwc_f16, w, b, ksize, act2=None, w2=None, b2=None, residual=None, out_fp16=False):
    N, H, W, Cin = act_nhwc_f16.shape
    Cout = w.shape[0]
    out = torch.empty((N, H, W, Cout), dtype=torch.float16 if out_fp16 else torch.float32, device="cuda")
    wc = w.detach().float().cpu().contiguous(); bc = b.detach().float().cpu().contiguous()
    w2c = w2.detach().float().cpu().contiguous() if w2 is not None else None
    b2c = b2.detach().float().cpu().contiguous() if b2 is not None else None
    _lib.check(_lib.lib().ivid_op_conv2d(_lib.ptr(act_nhwc_f16), N, H, W, Cin, _lib.ptr(wc), _lib.ptr(bc), Cout, ksize,
                                         _lib.ptr(act2), act2.shape[-1] if act2 is not None else 0, _lib.ptr(w2c), _lib.ptr(b2c),
                                         _lib.ptr(residual), _lib.ptr(out), 1 if out_fp16 else 0, _lib.cur_stream()))
    return out


def group_norm(x0, x1, groups, gamma, beta, film, silu, mode):
    N, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    Ho = H * 2 if mode == 1 else (H // 2 if mode == 2 else H)
    Wo = W * 2 if mode == 1 else (W // 2 if mode == 2 else W)
    out = torch.empty((N, Ho, Wo, C0 + C1), dtype=torch.float16, device="cuda")
    g = gamma.float().cpu().contiguous(); bt = beta.float().cpu().contiguous()
    _lib.check(_lib.lib().ivid_op_group_norm(_lib.ptr(x0), C0, _lib.ptr(x1), C1, N, H, W, groups, 1e-5, _lib.ptr(g), _lib.ptr(bt),
                                             _lib.ptr(film), 1 if silu else 0, mode, _lib.ptr(out), _lib.cur_stream()))
    return out


def nan_like_buffer(shape, dtype):
    """A device buffer filled with NaN (e4m3 bytes: 0x7F, its NaN): any element a kernel leaves alone stays NaN."""
    if dtype == torch.uint8:
        return torch.full(shape, 0x7F, dtype=torch.uint8, device="cuda")
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _host(t):
    return t.detach().float().cpu().contiguous() if t is not None else None


def conv_ex(act0, w0, b0, ksize, out, out_mode=0, *, N=None, e4m3=False, act1=None, act2=None, wskip=None, bskip=None,
            residual=None, residual_up=False, out16=None, stats=None):
    """ivid_op_conv2d_ex.  act0 [N,H,W,C0] fp16 (uint8 e4m3 bytes with e4m3=True); wskip [Cout, C1 + C2] for a 1x1 skip over
    act1 [| act2].  The caller allocates out / out16 / stats (they may hold more samples than N).  Returns (status, e)."""
    N = act0.shape[0] if N is None else N
    _, H, W, C0 = act0.shape
    w0h, b0h, wsh, bsh = _host(w0), _host(b0), _host(wskip), _host(bskip)
    p = lambda t: t.data_ptr() if t is not None else None
    e = ctypes.c_int(0)
    a = _lib.OpConvT(act0_dev=act0.data_ptr(), C0=C0, ksize=ksize, w0_host=w0h.data_ptr(), b0_host=p(b0h),
                     e4m3=1 if e4m3 else 0, e_out=ctypes.pointer(e),
                     act1_dev=p(act1), C1=act1.shape[-1] if act1 is not None else 0,
                     act2_dev=p(act2), C2=act2.shape[-1] if act2 is not None else 0, wskip_host=p(wsh), bskip_host=p(bsh),
                     residual_dev=p(residual), residual_up=1 if residual_up else 0,
                     N=N, H=H, W=W, Cout=w0.shape[0], out_dev=out.data_ptr(), out_mode=out_mode, out16_dev=p(out16),
                     stats_dev=p(stats))
    rc = _lib.lib().ivid_op_conv2d_ex(ctypes.byref(a), _lib.cur_stream())
    return rc, e.value


def gn_apply(x0, x1, out, *, groups, gamma, beta, N=None, stats0=None, stats1=None, film=None, film_ld=0, film_off=0,
             film_add=False, silu=True, mode=0, out_e4m3=False, out_lo=None, out_raw16=None, out_raw32=None, eps=1e-5):
    """ivid_op_group_norm_apply over x0 [| x1] (NHWC, fp32 or fp16).  Returns the status."""
    N = x0.shape[0] if N is None else N
    _, H, W, C0 = x0.shape
    g = _host(gamma); bt = _host(beta)
    p = lambda t: t.data_ptr() if t is not None else None
    a = _lib.OpGnT(x0_dev=x0.data_ptr(), C0=C0, x1_dev=p(x1), C1=x1.shape[-1] if x1 is not None else 0,
                   x_fp16=1 if x0.dtype == torch.float16 else 0, stats0_dev=p(stats0), stats1_dev=p(stats1),
                   N=N, H=H, W=W, groups=groups, eps=eps, gamma_host=g.data_ptr(), beta_host=bt.data_ptr(),
                   film_dev=p(film), film_ld=film_ld, film_off=film_off, film_add=1 if film_add else 0,
                   silu=1 if silu else 0, mode=mode, out_dev=out.data_ptr(), out_e4m3=1 if out_e4m3 else 0,
                   out_lo_dev=p(out_lo), out_raw16_dev=p(out_raw16), out_raw32_dev=p(out_raw32))
    return _lib.lib().ivid_op_group_norm_apply(ctypes.byref(a), _lib.cur_stream())


def conv_tile(H, W):
    """(TW, TH, TN, fused_stats) of the conv kernel at an H x W layer."""
    v = [ctypes.c_int() for _ in range(4)]
    _lib.check(_lib.lib().ivid_conv_tile(H, W, *[ctypes.byref(x) for x in v]))
    return tuple(x.value for x in v)


def attention(qkv_f16, C):
    N, T, _ = qkv_f16.shape
    out = torch.empty((N, T, C), dtype=torch.float16, device="cuda")
    _lib.check(_lib.lib().ivid_op_attention(_lib.ptr(qkv_f16), N, T, C, _lib.ptr(out), _lib.cur_stream()))
    return out
