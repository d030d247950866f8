"""CPU replica of the path selection and the rounding of the resampling layers and the fp32-source GroupNorm passes.

Which code path a layer takes is decided on the host from its shape alone:
  conv_tile / conv_can_fuse_stats   (csrc/ops.cu) the conv's pixel tile TW x TH x TN, and whether its epilogue can take the
                                    GroupNorm statistics of the output (TW * TH >= 32 pixels of one sample); otherwise the
                                    separate gn_stats pass reads the fp32 output.  Every pooling / nearest layer without a
                                    conv takes gn_stats.
  gn_prologue_fast                  (csrc/elementwise.cuh) the apply prologue's shuffle path: power-of-two group width
                                    <= 32, C % 32 == 0, C <= 1024; every other width takes the per-group loop.
  gn_stats_layout / gn_stats_run    gn_stats_kernel: cols = min(C/4, 256) float4 columns by rows = 256 / cols pixel rows,
                                    256 pixels per block; a thread sums its pixels p0 + ty, p0 + ty + rows, ... in fp32, the
                                    rows and blocks are added in fp64.

The bounds (tests/test_gpu_resample.py holds the kernels to them):
  gn_stats  |S - S64| <= gamma(m) sum|x| + fp64,  |Q - Q64| <= gamma(m) sum x^2 + fp64, m = gn_stats_run(C, HW): a thread's
            running fp32 sum passes each value through at most m roundings (the first addition to 0 is exact; the square
            is one more for Q when it is not fused into the addition).
  pool      ((a00 + a01) + (a10 + a11)) * 0.25 in fp32: three roundings of partial sums, the x0.25 exact.
gn_stats_emulate and pool_f32 repeat the kernels' summation order in numpy float32 (tests/test_resample_model.py checks
the bounds against them)."""
import math

import numpy as np

U24 = 2.0 ** -24
U53 = 2.0 ** -53
STATS_PIX_PER_BLOCK = 256


def pow2_divisor(v, cap):
    t = 1
    while t * 2 <= cap and v % (t * 2) == 0:
        t *= 2
    return t


def conv_tile(H, W):
    """(TW, TH, TN) of the conv kernel at an H x W output (ops.cu conv_tile)."""
    TW = pow2_divisor(W, 16)
    TH = pow2_divisor(H, 128 // TW)
    return TW, TH, 128 // (TW * TH)


def conv_can_fuse_stats(H, W):
    TW, TH, _ = conv_tile(H, W)
    return TW * TH >= 32


def conv_pad_k(c):
    return (c + 63) // 64 * 64


def slab(H, W):
    """Whether a 3x3 conv at an H x W output loads one slab per (chunk, dx) (ops.cu conv_launch_create)."""
    TW, _, TN = conv_tile(H, W)
    return TN == 1 and TW >= 8


def gn_prologue_fast(C, groups):
    cpg = C // groups
    return (cpg & (cpg - 1)) == 0 and cpg <= 32 and C % 32 == 0 and C <= 1024


def gn_stats_layout(C):
    """(cols, rows, rounds) of gn_stats_kernel at C channels: rounds = ceil(C/4 / cols) passes over the columns."""
    c4 = C // 4
    cols = min(c4, 256)
    return cols, 256 // cols, -(-c4 // cols)


def gn_stats_run(C, HW):
    """The longest fp32 running sum of one thread: ceil(min(HW, 256) / rows) pixels."""
    _, rows, _ = gn_stats_layout(C)
    return -(-min(HW, STATS_PIX_PER_BLOCK) // rows)


def gamma(m):
    return m * U24 / (1 - m * U24)


def gn_stats_bound(x64, C, HW):
    """Per-(sample, channel) bounds on |S - S64| and |Q - Q64| for x64 float64 [N, HW, C]."""
    m = gn_stats_run(C, HW)
    _, rows, _ = gn_stats_layout(C)
    blocks = -(-HW // STATS_PIX_PER_BLOCK)
    f64 = (rows + blocks + 2) * U53 * (1 + 1e-6)
    A = np.abs(x64).sum(1)
    Q = (x64 * x64).sum(1)
    return (gamma(m) + f64) * A, (gamma(m + 1) + f64) * Q


def gn_stats_emulate(x):
    """gn_stats_kernel's summation order on x float32 [N, HW, C]: fp32 per-thread runs, then fp64 over rows and blocks
    (the squares fused into the addition, as one rounding of x*x + q).  Returns float64 [N, C, 2]."""
    x = np.asarray(x, np.float32)
    N, HW, C = x.shape
    _, rows, _ = gn_stats_layout(C)
    out = np.zeros((N, C, 2))
    for p0 in range(0, HW, STATS_PIX_PER_BLOCK):
        blk = x[:, p0:min(p0 + STATS_PIX_PER_BLOCK, HW)]
        steps = -(-blk.shape[1] // rows)
        pad = np.zeros((N, steps * rows, C), np.float32)
        pad[:, :blk.shape[1]] = blk
        pad = pad.reshape(N, steps, rows, C)
        s = np.zeros((N, rows, C), np.float32)
        q = np.zeros((N, rows, C), np.float32)
        for j in range(steps):
            v = pad[:, j]
            s = s + v
            q = (v.astype(np.float64) * v + q).astype(np.float32)
        out[..., 0] += s.astype(np.float64).sum(1)
        out[..., 1] += q.astype(np.float64).sum(1)
    return out


def pool_f32(x):
    """resample_f32_kernel mode 2 on x float32 [N, H, W, C]: ((a00 + a01) + (a10 + a11)) * 0.25 in fp32."""
    x = np.asarray(x, np.float32)
    a00, a01, a10, a11 = x[:, 0::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 0::2], x[:, 1::2, 1::2]
    return ((a00 + a01) + (a10 + a11)) * np.float32(0.25)


def pool_bound(x64):
    """|pool_f32 - pool64| <= 2^-24 (|a00 + a01| + |a10 + a11| + |sum|) / 4 (three roundings; x0.25 is exact)."""
    a00, a01, a10, a11 = x64[:, 0::2, 0::2], x64[:, 0::2, 1::2], x64[:, 1::2, 0::2], x64[:, 1::2, 1::2]
    s0, s1 = a00 + a01, a10 + a11
    return U24 * (np.abs(s0) + np.abs(s1) + np.abs(s0 + s1)) * 0.25 * (1 + 1e-6)


def ulp32(y):
    return np.exp2(np.floor(np.log2(np.maximum(np.abs(y), 2.0 ** -126))) - 23)


# ----------------------------------------------------------------------------------------------------------------------
# The GPU cases (tests/test_gpu_resample.py) and the path each one names; tests/test_resample_model.py checks that each
# really reaches it.
# ----------------------------------------------------------------------------------------------------------------------
# a. gn_stats: (C, HW, N, k).  Every width at HW 255 / 257 and N = 3; every HW at C = 96 and 1280; N = 1 and 33; DC offsets.
STATS_WIDTHS = [8, 40, 96, 256, 1024, 1280, 1544, 2048]
STATS_HWS = [1, 16, 31, 255, 257, 4096]
STATS_CASES = sorted({(C, HW, 3, 10) for C in STATS_WIDTHS for HW in (255, 257)}
                     | {(C, HW, 3, 0) for C in (96, 1280) for HW in STATS_HWS}
                     | {(C, 4096, 1, 10) for C in (40, 2048)}
                     | {(C, 16, 33, 10) for C in (8, 1544)}
                     | {(256, 31, 33, 0), (1024, 4096, 1, 100), (1544, 255, 3, 100), (2048, 257, 3, 100),
                        (96, 4096, 3, 100), (8, 4096, 3, 100)})


def stats_case_id(c):
    C, HW, N, k = c
    cols, rows, rounds = gn_stats_layout(C)
    kind = "idle" if 256 % cols else ("ragged" if (C // 4) % cols else ("rounds" if rounds > 1 else "full"))
    return f"C{C}-HW{HW}-N{N}-k{k}-{kind}"


# b. fp32-source apply: (tag, C0, C1, groups, film ("ss", "add", None), stats supplied, mode, H, W, N) at INPUT size H x W.
APPLY_CASES = [
    ("fast ss m2 16x16", 128, 0, 32, "ss", True, 2, 16, 16, 3),
    ("fast none m1 8x8", 256, 0, 32, None, True, 1, 8, 8, 3),
    ("fast add m0 4x4 nullstats", 256, 0, 32, "add", False, 0, 4, 4, 5),
    ("fast seam m2 64x64", 72, 56, 8, "ss", True, 2, 64, 64, 2),
    ("fast seam m1 32x32 nullstats", 88, 40, 8, None, False, 1, 32, 32, 2),
    ("fast m2 128x128", 64, 0, 32, None, True, 2, 128, 128, 1),
    ("fast m1 64x64 nullstats", 64, 0, 32, "ss", False, 1, 64, 64, 1),
    ("loop C1280 m2 12x20", 1280, 0, 32, "ss", True, 2, 12, 20, 3),
    ("loop C1280 m0 6x10 nullstats", 1280, 0, 32, "add", False, 0, 6, 10, 3),
    ("loop cpg40 seam m1 6x10", 192, 128, 8, "ss", True, 1, 6, 10, 3),
    ("loop cpg40 m2 24x40 nullstats", 320, 0, 8, None, False, 2, 24, 40, 3),
    ("loop cpg3 m0 12x20", 96, 0, 32, "ss", True, 0, 12, 20, 3),
    ("loop cpg3 seam m2 24x40 nullstats", 64, 32, 32, "add", False, 2, 24, 40, 2),
    ("loop cpg3 m1 12x20 add", 96, 0, 32, "add", True, 1, 12, 20, 3),
    ("fast seam m0 2x2 nullstats", 136, 120, 16, "ss", False, 0, 2, 2, 7),
]


def apply_path(case):
    _, C0, C1, groups, *_ = case
    return "fast" if gn_prologue_fast(C0 + C1, groups) else "loop"


# c / d. resampling convs: (mode, C, N, output H, output W).
DOWN_CASES = [(2, C, N, Ho, Wo) for C, N, Ho, Wo in
              [(64, 2, 8, 8), (96, 3, 8, 8), (160, 9, 4, 4), (64, 5, 4, 4), (96, 3, 1, 1), (160, 130, 1, 1),
               (64, 3, 2, 2), (96, 3, 6, 10), (160, 2, 32, 48), (64, 2, 16, 16)]]
UP_CASES = [(1, C, N, Ho, Wo) for C, N, Ho, Wo in
            [(64, 2, 16, 16), (96, 2, 32, 48), (160, 3, 16, 16), (64, 3, 12, 20), (96, 3, 12, 20), (160, 9, 4, 4),
             (64, 5, 4, 4)]]


def conv_case_id(c):
    mode, C, N, Ho, Wo = c
    TW, TH, TN = conv_tile(Ho, Wo)
    stats = "fused" if conv_can_fuse_stats(Ho, Wo) else "gnstats"
    path = "-slab" if mode == 1 and slab(Ho, Wo) else ""
    return f"{'down' if mode == 2 else 'up'}-C{C}-N{N}-{Ho}x{Wo}-{TW}x{TH}x{TN}-{stats}{path}"


def conv_K(mode, C):
    """Accumulated columns of the conv: the 9C gathered taps padded once (down), nine padded C-chunks (up)."""
    return conv_pad_k(9 * C) if mode == 2 else 9 * conv_pad_k(C)


# e. pool / nearest: (mode, C, N, input H, input W)
PLAIN_CASES = [(2, 64, 3, 16, 16), (2, 1280, 3, 12, 20), (2, 96, 33, 2, 2), (2, 1544, 2, 8, 8), (1, 64, 3, 8, 8),
               (1, 1280, 2, 6, 10), (1, 96, 5, 1, 1), (2, 40, 2, 64, 128)]


def plain_case_id(c):
    mode, C, N, H, W = c
    return f"{'pool' if mode == 2 else 'nearest'}-C{C}-N{N}-{H}x{W}"
