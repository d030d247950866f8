"""CPU restatement of the attention kernels' online softmax, and the inputs that drive each of its paths.

attention_kernel (csrc/attention.cuh, d = 64) and attention_hd_kernel (csrc/attention_hd.cuh, d = 64k) walk the keys in
blocks of 64.  Per query row they keep a reference maximum m (log2 units) that moves only when a block's maximum logit
exceeds it by more than LAZY = 8; then alpha = 2^(m_old - m_new) rescales O and l.  Probabilities p = 2^(lambda - m)
are rounded to fp16 for P V while l sums them in fp32; keys past T in the last block are masked to -inf.  walk() repeats
that walk (fp32 logits, the kernel's fp32 scale) and reports per row what the kernels' rescale path sees.

The second half builds q / k whose logits are known, one family per path (tests/test_gpu_attention_softmax.py runs them
on the GPU; tests/test_attention_softmax_model.py checks here that each family really drives its path):
  plateau  every later block's maximum is m0 + delta (delta < 8): m never moves after block 0, p reaches 2^delta
  ramp     block j's maximum is m0 + j * delta (delta > 8): m moves on every block; at delta = 200 alpha flushes to 0
  dominant one key 12 above the rest, at a given position (first, end of block 0, start of the last full block, last key)
  diag     the dominant key is the query's own position (rows rescale at different blocks)
  onehot   one key per row at least 30 above every other: the output is that V row
  uniform  q = 0: every logit is 0, the output is the mean of v[:T]
  offset   every logit carries a common +-1000 (natural units) plus small variation
Every q and k value is a multiple of 1/4 and every row's sum_i |q_i k_i| stays below 2^19, so each partial sum of
S = q . k is a multiple of 2^-4 below 2^20: an fp32 number.  S is then exact in any summation order, and what is left of
the logit error is the fp32 scale and the exponent (see test_gpu_attention_softmax.bound).
"""
import math

import numpy as np

KV = 64
LAZY = 8.0
LOG2E = 1.4426950408889634
GRID = 0.25                 # q / k values are multiples of this
S_EXACT_LIMIT = 2.0 ** 19   # sum_i |q_i k_i| below this keeps every partial sum of S an fp32 number (2^-4 grid)


def scale_log2(d):
    """The kernels' fp32 logit scale d^-1/2 * log2(e) (attention_kernel: 0.125f * log2e; ops.cu for the others)."""
    if d == 64:
        return np.float32(np.float32(0.125) * np.float32(LOG2E))
    return np.float32(LOG2E / math.sqrt(d))


def walk(q, k, d, lazy=LAZY):
    """The kernels' block walk for query rows q [R, d] against keys k [T, d] (fp16 values, any float dtype).

    Returns a dict of per-row arrays:
      rescales   key blocks after the first in which the reference maximum moves (alpha != 1)
      alpha_zero rescales whose alpha = 2^(m_old - m_new) is below 2^-126 and flushes to 0
      p_exp_max  largest log2 p = lambda - m over the valid keys (p <= 2^8 under the lazy rule)
      subnormal  valid keys whose fp16 p is subnormal or 0 (p < 2^-14)
      flushed    valid keys whose p is below 2^-126 (ex2.approx.ftz returns 0)
      argmax     key of the largest logit
      gap        largest logit minus the second largest (inf when T = 1)
    """
    q = np.asarray(q, dtype=np.float32)
    k = np.asarray(k, dtype=np.float32)
    R, T = q.shape[0], k.shape[0]
    lam = (q @ k.T).astype(np.float32) * scale_log2(d)          # [R, T] fp32, as the kernel scales S
    nkv = (T + KV - 1) // KV
    m = np.full(R, -np.inf, dtype=np.float32)
    out = {key: np.zeros(R, dtype=np.int64) for key in ("rescales", "alpha_zero", "subnormal", "flushed")}
    p_exp_max = np.full(R, -np.inf, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        for j in range(nkv):
            blk = lam[:, j * KV:min(T, (j + 1) * KV)]            # the tail mask: keys >= T take no part
            m_cand = np.maximum(m, blk.max(axis=1))
            take = (m_cand - m) > np.float32(lazy)               # m = -inf on the first block: always taken
            if j > 0:
                out["rescales"] += take
                out["alpha_zero"] += take & ((m - m_cand) < -126)
            m = np.where(take, m_cand, m)
            x = blk - m[:, None]
            p_exp_max = np.maximum(p_exp_max, x.max(axis=1))
            out["subnormal"] += (x < -14).sum(axis=1)
            out["flushed"] += (x < -126).sum(axis=1)
    out["p_exp_max"] = p_exp_max
    out["argmax"] = lam.argmax(axis=1)
    if T > 1:
        top2 = np.partition(lam, T - 2, axis=1)[:, T - 2:]
        out["gap"] = top2[:, 1] - top2[:, 0]
    else:
        out["gap"] = np.full(R, np.inf, dtype=np.float32)
    return out


def walk_qkv(qkv, C, d):
    """walk() over every (sample, head) of qkv [N, T, 3C] in the kernels' layout (head h: channels [3dh, 3dh + 3d) =
    q | k | v).  The per-row arrays are ordered [N][heads][T]."""
    qkv = np.asarray(qkv)
    N = qkv.shape[0]
    parts = []
    for n in range(N):
        for h in range(C // d):
            base = 3 * d * h
            parts.append(walk(qkv[n, :, base:base + d], qkv[n, :, base + d:base + 2 * d], d))
    return {key: np.concatenate([p[key] for p in parts]) for key in parts[0]}


# ------------------------------------------------------------------------------------------------------------------
# input families
# ------------------------------------------------------------------------------------------------------------------
PLATEAU = [("plateau", 4.0), ("plateau", 7.9)]
RAMP = [("ramp", 8.1), ("ramp", 20.0), ("ramp", 200.0)]
DOMINANT = [("dominant", "first"), ("dominant", "end0"), ("dominant", "lastfull"), ("dominant", "last"), ("diag", None)]
ONEHOT = [("onehot", None)]
UNIFORM = [("uniform", None)]
OFFSET = [("offset", None)]
VARIANTS = PLATEAU + RAMP + DOMINANT + ONEHOT + UNIFORM + OFFSET
# "mixed" heads: the family changes every 8 rows (rows r and r + 8 of a warp differ) and between the two warpgroup halves
# of each 128-query tile; one head of a launch carries it next to whole-head families in the other heads
MIXED = ([("ramp", 20.0), ("plateau", 7.9), ("uniform", None), ("dominant", "last")],
         [("offset", None), ("ramp", 8.1), ("plateau", 4.0), ("ramp", 200.0)])
DOMINANT_GAP = 12.0
ONEHOT_GAP = 34.0
DIAG_GAP = 14.0
OFFSET_NATURAL = 1000.0
NOISE = 0.5                 # standard deviation of the free q / k channels (logit noise ~0.36 in log2 units)


def label(variant):
    name, param = variant
    return name if param is None else f"{name}:{param:g}" if isinstance(param, float) else f"{name}:{param}"


def _round_grid(x):
    return np.round(np.asarray(x, dtype=np.float64) / GRID) * GRID


def _fp16_grid(x):
    """Round to the 1/4 grid, then to fp16 (fp16 values >= 256 are multiples of 1/4 already)."""
    return _round_grid(x).astype(np.float16).astype(np.float64)


def dominant_key(param, T):
    return {"first": 0, "end0": min(KV - 1, T - 1), "lastfull": max(T // KV - 1, 0) * KV, "last": T - 1}[param]


def _key_levels(variant, T, rng):
    """Per-key logit level (log2 units, for a row multiplier of 1) on the variant's channel (NaN: channel left 0), and
    the keys that set a block's maximum (their free channels are 0, so their logits are exactly the level)."""
    name, param = variant
    nkv = (T + KV - 1) // KV
    lev = np.full(T, np.nan)
    top_keys = np.zeros(T, dtype=bool)
    if name in ("plateau", "ramp"):
        blocks = np.arange(T) // KV
        if name == "plateau":
            top = np.where(blocks == 0, 0.0, param)
        else:
            top = (blocks - (nkv - 1) / 2.0) * param
        lev = top - rng.uniform(2.0, 8.0, T)                     # every other key of a block sits 2..8 below its top
        for j in range(nkv):
            valid = min(T, (j + 1) * KV) - j * KV
            s = j * KV + (17 * j + 5) % valid
            lev[s] = top[s]
            top_keys[s] = True
    elif name == "dominant":
        s = dominant_key(param, T)
        lev[s] = DOMINANT_GAP
        top_keys[s] = True
    elif name == "offset":
        lev[:] = OFFSET_NATURAL * LOG2E
    return lev, top_keys


def _row_mult(variant, i):
    """Multiplier of the variant's q channel for the i-th row of that variant in a head: ramps alternate 1 / 1.5 and
    offsets +1 / -1 every 8 rows, so neighbouring row groups rescale by different alphas."""
    name = variant[0]
    if name == "ramp":
        return 1.5 if (i >> 3) & 1 else 1.0
    if name == "offset":
        return -1.0 if (i >> 3) & 1 else 1.0
    return 1.0


def _perm_head(variant, T, d, rng):
    """diag / onehot: q_t = g r_pi(t), k_s = g r_s with random sign vectors r, so q_t . k_pi(t) = g^2 d stands about
    sqrt(d) standard deviations above every other logit."""
    gap = DIAG_GAP if variant[0] == "diag" else ONEHOT_GAP
    g2 = gap / ((math.sqrt(d) - 4.0) * LOG2E)
    g = math.ceil(math.sqrt(g2) / GRID) * GRID
    r = rng.choice([-1.0, 1.0], size=(T, d))
    pi = np.arange(T) if variant[0] == "diag" else rng.integers(0, T, T)
    return g * r[pi], g * r


def head_qk(rows, T, d, rng):
    """q, k [T, d] (float64 holding fp16 values on the 1/4 grid) for one head whose query row t belongs to rows[t]."""
    sig = LOG2E / math.sqrt(d)
    kinds = list(dict.fromkeys(rows))
    if any(v[0] in ("diag", "onehot") for v in kinds):
        assert len(kinds) == 1, "diag / onehot take a whole head"
        return _perm_head(kinds[0], T, d, rng)
    chans = {v: i for i, v in enumerate(v for v in kinds if v[0] != "uniform")}
    free = np.arange(len(chans), d)
    q = np.zeros((T, d))
    k = np.zeros((T, d))
    k[:, free] = _fp16_grid(rng.normal(0.0, NOISE, (T, free.size)))
    counts = {v: 0 for v in kinds}
    for t, v in enumerate(rows):
        if v[0] != "uniform":
            q[t, free] = _round_grid(rng.normal(0.0, NOISE, free.size))
    for v, c in chans.items():
        lev, top_keys = _key_levels(v, T, rng)
        top = max(1.0, float(np.nanmax(np.abs(lev))))
        qs = max(0.5, 2.0 ** math.ceil(math.log2(top / (sig * 1024.0))))   # |k| <= 1024: level error <= qs sig / 4
        has = ~np.isnan(lev)
        k[has, c] = _fp16_grid(lev[has] / (qs * sig))
        k[np.ix_(np.flatnonzero(top_keys), free)] = 0.0
        for t, rv in enumerate(rows):
            if rv == v:
                q[t, c] = qs * _row_mult(v, counts[v])
                counts[v] += 1
    return q, k


def mixed_rows(T):
    return [MIXED[(t % 128) // 64][((t % 128) // 8) % 4] for t in range(T)]


def make_case(seed, N, T, d, slots):
    """qkv [N, T, 3C] fp16 (C = heads * d, heads = len(slots) // N) and the per-row variant labels [N, heads, T].
    slots[n * heads + h] is a variant for the whole head, or "mixed"."""
    assert len(slots) % N == 0
    heads = len(slots) // N
    rng = np.random.default_rng(seed)
    qkv = np.zeros((N, T, 3 * heads * d), dtype=np.float16)
    labels = np.empty((N, heads, T), dtype=object)
    for i, slot in enumerate(slots):
        n, h = divmod(i, heads)
        rows = mixed_rows(T) if slot == "mixed" else [slot] * T
        q, k = head_qk(rows, T, d, rng)
        assert np.all(q == _round_grid(q)) and np.all(k == _round_grid(k))
        assert float((np.abs(q) @ np.abs(k).T).max()) < S_EXACT_LIMIT, f"{slot} at d={d} T={T}: S would round"
        base = 3 * d * h
        qkv[n, :, base:base + d] = q
        qkv[n, :, base + d:base + 2 * d] = k
        qkv[n, :, base + 2 * d:base + 3 * d] = rng.standard_normal((T, d))
        labels[n, h] = [label(v) for v in rows]
    return qkv, labels


def slices(d):
    """(k, slices, nv) of attention_hd_kernel at head width d (ops.cu attn_launch_create); d = 64 is attention_kernel."""
    k = d // 64
    s = (k + 3) // 4
    nv = (k + s - 1) // s
    return k, (k + nv - 1) // nv, nv


def instance(d):
    """The kernel template a head width dispatches to."""
    if d == 64:
        return "attention_kernel"
    k, _, nv = slices(d)
    return f"attention_hd_kernel<{nv},{'true' if k <= 8 else 'false'}>"


# The GPU cases: (name, d, T, N, slots).  Each width runs every whole-head variant plus a mixed head in one launch (one sample's
# heads, then the next sample's), and a second, single-head launch at other lengths.  Widths and their (k, slices, nv):
#   64: attention_kernel | 128: (2, 1, 2) | 192: (3, 1, 3) | 256: (4, 1, 4) | 320: (5, 2, 3), slices 3 + 2
#   448: (7, 2, 4), 4 + 3 | 512: (8, 2, 4) | 576: (9, 3, 3), Q streamed | 640: (10, 3, 4), 4 + 4 + 2
#   832: (13, 4, 4), 4 + 4 + 4 + 1 | 1024: (16, 4, 4)
WIDTHS = (64, 128, 192, 256, 320, 448, 512, 576, 640, 832, 1024)
FAMILY_SLOTS = VARIANTS[:7] + ["mixed"] + VARIANTS[7:]                 # 14 slots: N = 2 samples of 7 heads
LONG_T = {64: 1023, 128: 1023, 192: 1000, 256: 1023, 320: 1000, 448: 1023, 512: 1000, 576: 1023, 640: 1000,
          832: 1023, 1024: 1023}
SHORT_T = {64: (1, 65), 128: (63, 129), 192: (64, 65), 256: (129, 1), 320: (65, 63), 448: (64, 129), 512: (63, 65),
           576: (129, 64), 640: (65, 1), 832: (129, 63), 1024: (65, 129)}
SINGLE_SLOTS = ["mixed", ("ramp", 20.0)]


def case_seed(name):
    return sum((i + 1) * ord(ch) for i, ch in enumerate(name))


def gpu_cases():
    """[(name, d, T, N, slots)] of the GPU test."""
    out = []
    for d in WIDTHS:
        out.append((f"d{d}-T{LONG_T[d]}-families", d, LONG_T[d], 2, FAMILY_SLOTS))
        for T, slot in zip(SHORT_T[d], SINGLE_SLOTS):
            out.append((f"d{d}-T{T}-single-{slot if slot == 'mixed' else label(slot)}", d, T, 1, [slot]))
    return out


# The network with partial output-column slices: one head of 320 channels at 16 x 16 (T = 256, slices 3 + 2) and of
# 640 channels at 8 x 8 (T = 64, slices 4 + 4 + 2).  PEAKED_QKV_SCALE multiplies every attention block's qkv weights:
# the logits grow 9x, and the walk reports rescales in about a fifth of the T = 256 rows (none without it).
PARTIAL_SLICE_CFG = dict(image_size=32, in_channels=4, model_channels=160, out_channels=4, num_res_blocks=1,
                         attention_resolutions=[16, 8], channel_mult=[1, 2, 4], num_classes=10, has_null_class=True,
                         num_groups=32, num_heads=1, num_head_channels=-1, dropout=0.0, use_fp16=False)
PEAKED_QKV_SCALE = 3.0


def peaked_state_dict(sd, scale=PEAKED_QKV_SCALE):
    return {key: (val * scale if key.endswith(".qkv.weight") else val) for key, val in sd.items()}
