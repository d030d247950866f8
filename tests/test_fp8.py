"""CPU: the fp8 (e4m3) precision mode's host side.  The packer's e4m3 conversion against torch's float8_e4m3fn, its
power-of-two weight-scale rule at the (224, 448] boundaries, the new entry points, and the fp8 emulation of
tests/precision_model_fp8.py (finite, and further from fp32 than the fp16 plan)."""
import ctypes
import json
import math

import numpy as np
import torch

from ivid_b200 import _lib


def _quantize(x):
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.empty(x.size, dtype=np.uint8)
    _lib.check(_lib.lib().ivid_fp8_e4m3_quantize(x.ctypes.data, out.ctypes.data, x.size))
    return out


def _torch_e4m3_bytes(x):
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).clamp(-448.0, 448.0)
    return t.to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def test_quantize_matches_torch_e4m3fn():
    codes = np.arange(256, dtype=np.uint8)
    grid = torch.from_numpy(codes).view(torch.float8_e4m3fn).float().numpy()
    grid = grid[np.isfinite(grid)]
    # every representable value, the midpoints between neighbours (ties: round to even), one fp32 ulp either side of each
    # midpoint, and values that must saturate
    pos = np.unique(np.abs(grid))
    mids = ((pos[:-1].astype(np.float64) + pos[1:]) / 2).astype(np.float32)
    near = np.concatenate([np.nextafter(mids, np.float32(np.inf)), np.nextafter(mids, np.float32(0))])
    big = np.array([448, 449, 463.9, 464, 465, 480, 500, 1e4, 3.4e38, np.inf], dtype=np.float32)
    tiny = np.array([2.0 ** -10, 2.0 ** -9 * 0.5, 2.0 ** -9 * 0.75, 2.0 ** -9 * 1.5, 2.0 ** -6 - 2.0 ** -11, 1e-30, 0.0],
                    dtype=np.float32)
    rand = np.random.default_rng(0).standard_normal(100000).astype(np.float32) * np.float32(30)
    x = np.concatenate([grid, mids, near, big, tiny, rand])
    x = np.concatenate([x, -x, np.array([-0.0], dtype=np.float32)])
    got, want = _quantize(x), _torch_e4m3_bytes(x)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{bad.size} mismatches, e.g. {x[bad[:5]]} -> {got[bad[:5]]} vs {want[bad[:5]]}"
    assert _quantize(np.array([448.0, 1e9, -1e9, -np.inf], np.float32)).tolist() == [0x7E, 0x7E, 0xFE, 0xFE]
    assert _quantize(np.array([np.nan], np.float32))[0] & 0x7F == 0x7F


def _exponent(w):
    w = np.ascontiguousarray(w, dtype=np.float32)
    e = ctypes.c_int()
    _lib.check(_lib.lib().ivid_fp8_weight_exponent(w.ctypes.data, w.size, ctypes.byref(e)))
    return e.value


def test_weight_exponent_rule():
    assert _exponent(np.zeros(10)) == 0
    for m in [448.0, 224.0, float(np.nextafter(np.float32(224), np.float32(1e9))), float(np.nextafter(np.float32(448), np.float32(0))),
              float(np.nextafter(np.float32(448), np.float32(1e9))), 0.875, 0.8750001, 1.0, 3e-5, 12345.0, 2.0 ** -20, 300.0]:
        w = np.array([0.1 * m, -m, 0.5 * m], dtype=np.float32)
        e = _exponent(w)
        scaled = float(np.float32(m)) * 2.0 ** e
        assert 224.0 < scaled <= 448.0, (m, e, scaled)
    assert _exponent(np.array([224.0], np.float32)) == 1          # 224 itself is excluded: it scales to 448
    assert _exponent(np.array([448.0], np.float32)) == 0
    assert _exponent(np.array([-1.0], np.float32)) == 8            # 256


def test_fp8_entry_points_exported():
    L = _lib.lib()
    for name in ("ivid_unet_set_precision", "ivid_op_conv2d_e4m3", "ivid_op_group_norm_e4m3", "ivid_fp8_e4m3_quantize",
                 "ivid_fp8_weight_exponent"):
        assert hasattr(L, name)


def _conv_op_status(e4m3, Cin, w, w2=None, act2=False):
    """Status and message of a conv op call whose device pointers are dummies, so it is only meaningful for arguments that
    are rejected before any CUDA call."""
    L = _lib.lib()
    dev = 0x1000                                          # never dereferenced
    Cout, k = w.shape[0], w.shape[-1]
    w = np.ascontiguousarray(w, dtype=np.float32)
    b = np.zeros(Cout, dtype=np.float32)
    w2 = None if w2 is None else np.ascontiguousarray(w2, dtype=np.float32)
    Cin2 = 64 if act2 else 0
    args = (dev, 1, 16, 16, Cin, w.ctypes.data, b.ctypes.data, Cout, k, dev if act2 else None, Cin2,
            None if w2 is None else w2.ctypes.data, None, None, dev, 0)
    rc = L.ivid_op_conv2d_e4m3(*args, None, None) if e4m3 else L.ivid_op_conv2d(*args, None)
    return rc, _lib.last_error()


def test_conv_ops_reject_before_any_cuda_call():
    w = np.random.default_rng(0).standard_normal((64, 64, 3, 3)).astype(np.float32) * 0.05
    # a skip input without its weights, for both entries
    for e4m3 in (False, True):
        rc, msg = _conv_op_status(e4m3, 64, w, act2=True)
        assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "w2_host" in msg, (e4m3, msg)
    # e4m3 only where the network's fp8 mode would run the conv in e4m3
    rc, msg = _conv_op_status(True, 40, w[:, :40])
    assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "multiple of 16" in msg, msg
    rc, msg = _conv_op_status(True, 64, w * 1e-36)                     # e > 100
    assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "exponent" in msg, msg
    w_small = w / np.abs(w).max() * 1e-3                               # e = 18: a skip weight of 1 scales to 2^18
    rc, msg = _conv_op_status(True, 64, w_small, np.full((64, 64), 1.0), act2=True)
    assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "overflow" in msg, msg
    w_large = w / np.abs(w).max() * 1e3                                # e = -2: 1e-4 (a normal fp16) scales to 2.5e-5
    rc, msg = _conv_op_status(True, 64, w_large, np.full((64, 64), 1e-4), act2=True)
    assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "subnormal" in msg, msg


def test_set_precision_rejects_unknown_values():
    import pytest
    import ivid_b200.backbones as backbones
    net = backbones.AdmUnet2d(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
                              attention_resolutions=[], channel_mult=(1, 2))
    assert net.precision == "fp16"
    with pytest.raises(ValueError):
        net.set_precision("bf16")
    assert _lib.lib().ivid_unet_set_precision(net._handle, 2) == _lib.IVID_ERR_INVALID_ARGUMENT
    net.set_precision("fp8")
    assert net.precision == "fp8"


def test_fp8_plan_emulation_tiny(golden):
    import precision_model as PM
    import precision_model_fp8 as P8
    from oracle import unet_ref
    cfg = json.loads(bytes(golden["tiny_cfg"]).decode())
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=1234)
    x = torch.from_numpy(golden["tiny_x"]); t = torch.from_numpy(golden["tiny_t"]); c = torch.from_numpy(golden["tiny_classes"])
    ref = unet_ref.unet_forward(cfg, sd, x, t, c)
    e8 = P8.forward(cfg, sd, x, t, c)
    assert torch.isfinite(e8).all()
    r8, r16 = PM.rel(e8, ref), PM.rel(PM.forward(cfg, sd, x, t, c, PM.PLAN), ref)
    print(f"[fp8] tiny eps rel to fp32: fp8 emulation {r8:.3e}, PLAN {r16:.3e}")
    assert r8 > r16
    assert not math.isnan(r8)
