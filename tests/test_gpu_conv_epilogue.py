"""The conv epilogue stages its outputs in shared memory and writes them with TMA box stores; the residual arrives by TMA
into the idle operand ring.  The epilogue's arithmetic is fixed (acc + bias, then + residual, then the fp16 rounding), so
these relations hold bit for bit, through ivid_op_conv2d_ex:

- the output with a residual r is the float32 sum out(no residual) + r (under residual_up: + nearest2x(r));
- the fp16 copy is out32.half(), and an fp16 output (out_mode 1) is the fp32 output (out_mode 0) rounded;
- nothing is written past sample N (the box stores clip at the tensor's extent).

They are checked at every tile class (16x8 and 8x16 slabs, 8x8x2, a 4x4x8 tile without fused statistics, 1x1), at
BN 128 / 64 / 16, in fp16 and e4m3, with N % TN != 0 and with Cout not a multiple of 32 (a box clipped mid-box)."""
import pytest
import torch

import gpu_util as G

pytestmark = pytest.mark.gpu


def _gen(tag):
    return torch.Generator().manual_seed(sum(ord(ch) * (i + 1) for i, ch in enumerate(tag)) % 2**31)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _run(act, w, b, k, N, H, W, Cout, out_mode=0, e4m3=False, residual=None, residual_up=False, copy=False, stats=False):
    out = G.nan_like_buffer((N + 1, H, W, Cout), torch.float16 if out_mode == 1 else torch.float32)
    out16 = G.nan_like_buffer((N + 1, H, W, Cout), torch.float16) if copy else None
    st = torch.zeros(N, Cout, 2, dtype=torch.float64, device="cuda") if stats else None
    rc, _ = G.conv_ex(act, w, b, k, out, out_mode, e4m3=e4m3, residual=residual, residual_up=residual_up, out16=out16,
                      stats=st)
    assert rc == 0, f"ivid_op_conv2d_ex returned {rc}"
    torch.cuda.synchronize()
    for buf in (out, out16):
        if buf is not None:
            b_ = buf.cpu().float()
            assert bool(torch.isnan(b_[N:]).all()), "written past sample N"
            assert not bool(torch.isnan(b_[:N]).any()), "an element was not written"
    return out[:N], (out16[:N] if copy else None), st


# tag, H, W, k, N, tile class: 32x32 -> 16x8 slab; 16x8 (H x W) -> 8x16 slab; 8x8 -> 8x8x2; 4x4 -> 4x4x8, no statistics
SHAPES = [
    ("slab16x8", 32, 32, 3, 2),
    ("slab8x16", 16, 8, 3, 2),
    ("tile8x8x2", 8, 8, 3, 3),
    ("tile4x4x8", 4, 4, 3, 3),
    ("1x1", 32, 32, 1, 2),
]
# Cout -> BN: 128 -> 128, 200 -> 128 (last block clipped at 72 of 128 columns), 64 -> 64, 40 -> 16 (clipped mid-block)
COUTS = [128, 200, 64, 40]


@pytest.mark.parametrize("e4m3", [False, True], ids=["fp16", "e4m3"])
@pytest.mark.parametrize("Cout", COUTS)
@pytest.mark.parametrize("tag,H,W,k,N", SHAPES, ids=[s[0] for s in SHAPES])
def test_epilogue_bitwise(tag, H, W, k, N, Cout, e4m3):
    g = _gen(f"{tag}-{Cout}-{e4m3}")
    Cin = 64
    a = torch.randn(N, H, W, Cin, generator=g)
    act = (a.clamp(-448.0, 448.0).to(torch.float8_e4m3fn) if e4m3 else a.half()).cuda()
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    r = torch.randn(N, H, W, Cout, generator=g).cuda()
    stats = H * W >= 32 and (H >= 8 or W >= 8)
    kw = dict(e4m3=e4m3)

    base, _, _ = _run(act, w, b, k, N, H, W, Cout, stats=stats, **kw)
    got, copy, _ = _run(act, w, b, k, N, H, W, Cout, residual=r, copy=True, stats=stats, **kw)
    assert torch.equal(_bits(got), _bits(base + r)), f"{tag} Cout {Cout}: out(residual) != out + r"
    assert torch.equal(_bits(copy), _bits(got.half())), f"{tag} Cout {Cout}: fp16 copy != out.half()"
    half, _, _ = _run(act, w, b, k, N, H, W, Cout, out_mode=1, residual=r, stats=stats, **kw)
    assert torch.equal(_bits(half), _bits(got.half())), f"{tag} Cout {Cout}: out_mode 1 != out_mode 0 .half()"
    if W >= 16 and H % 2 == 0 and Cout % 8 == 0:
        r2 = torch.randn(N, H // 2, W // 2, Cout, generator=g).cuda()
        up, _, _ = _run(act, w, b, k, N, H, W, Cout, residual=r2, residual_up=True, copy=True, stats=stats, **kw)
        near = r2.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
        assert torch.equal(_bits(up), _bits(base + near)), f"{tag} Cout {Cout}: out(residual_up) != out + nearest2x(r)"
