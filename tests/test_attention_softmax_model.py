"""CPU: the input families of test_gpu_attention_softmax.py drive the attention kernels' online-softmax paths they are
meant for (attention_softmax_model.walk restates the kernels' block walk), and the walk reproduces what the older
attention tests' random inputs reach: no rescale at all after the first key block."""
import numpy as np
import pytest
import torch

import attention_softmax_model as M

CASES = M.gpu_cases()


@pytest.fixture(scope="module")
def walked():
    return {c[0]: (c,) + _case_stats(c) for c in CASES}


def _case_stats(case):
    name, d, T, N, slots = case
    qkv, labels = M.make_case(M.case_seed(name), N, T, d, slots)
    C = len(slots) // N * d
    return labels.reshape(-1), M.walk_qkv(qkv.astype(np.float32), C, d), qkv


def _rows(walked, prefix):
    """(case, T, per-row stats restricted to rows labelled prefix*) over every GPU case."""
    for (name, d, T, N, slots), labels, st, qkv in walked.values():
        sel = np.array([str(l).startswith(prefix) for l in labels])
        if sel.any():
            yield name, d, T, sel, {k: v[sel] for k, v in st.items()}, labels


def test_ramp_rescales_on_every_block(walked):
    seen = 0
    for name, d, T, sel, st, _ in _rows(walked, "ramp"):
        nkv = (T + 63) // 64
        assert np.all(st["rescales"] == nkv - 1), f"{name}: a ramp row skips a rescale"
        seen += int(sel.sum()) if nkv > 1 else 0
    assert seen > 0
    # delta = 200: alpha flushes to 0 on every rescale
    for name, d, T, sel, st, labels in _rows(walked, "ramp:200"):
        assert np.all(st["alpha_zero"] == st["rescales"]), name


def test_plateau_never_rescales_and_reaches_its_level(walked):
    for name, d, T, sel, st, labels in _rows(walked, "plateau"):
        assert np.all(st["rescales"] == 0), f"{name}: a plateau row rescales"
        if T > 64:
            delta = np.array([float(str(l).split(":")[1]) for l in labels[sel]])
            assert np.all(st["p_exp_max"] > delta - 0.1), f"{name}: a plateau row stays below 2^(delta - 0.1)"
            assert np.all(st["p_exp_max"] < 8.0)


@pytest.mark.parametrize("prefix", ["uniform", "offset"])
def test_uniform_and_offset_never_rescale(walked, prefix):
    for name, d, T, sel, st, _ in _rows(walked, prefix):
        assert np.all(st["rescales"] == 0), f"{name}: a {prefix} row rescales"


def test_dominant_key_is_the_maximum_and_rescales_where_it_lies(walked):
    for name, d, T, sel, st, labels in _rows(walked, "dominant"):
        pos = np.array([M.dominant_key(str(l).split(":")[1], T) for l in labels[sel]])
        assert np.all(st["argmax"] == pos), name
        assert np.all(st["gap"] > 8.5), name
        assert np.all(st["rescales"] == (pos >= 64)), f"{name}: a dominant key past block 0 must move the maximum"


def test_diag_and_onehot_rows(walked):
    for name, d, T, sel, st, _ in _rows(walked, "diag"):
        assert np.all(st["argmax"] == np.arange(T)), name
        assert np.all(st["gap"] > 8.5), name
        if T > 64:
            assert np.all(st["rescales"][64:] >= 1)
    for name, d, T, sel, st, _ in _rows(walked, "onehot"):
        if T > 1:
            assert np.all(st["gap"] >= 30.0), f"{name}: a one-hot row's gap is {st['gap'].min():.1f}"


def test_mixed_heads_rescale_differently_in_neighbouring_rows(walked):
    """Rows r and r + 8 of a warp (and the two warpgroup halves) take different rescale paths in the mixed heads."""
    for (name, d, T, N, slots), labels, st, qkv in walked.values():
        if "mixed" not in slots or T < 129:
            continue
        i = slots.index("mixed")
        r = st["rescales"][i * T:(i + 1) * T]
        tile = r[:128]
        assert np.any(tile[:64] != tile[64:]), name
        assert np.any(tile[:120] != tile[8:]), name


def test_every_instance_meets_every_family():
    want = {"plateau", "ramp", "dominant", "diag", "onehot", "uniform", "offset", "mixed"}
    got = {}
    for name, d, T, N, slots in CASES:
        fams = {s if s == "mixed" else s[0] for s in slots}
        got.setdefault(M.instance(d), set()).update(fams)
    assert set(got) == {"attention_kernel", "attention_hd_kernel<2,true>", "attention_hd_kernel<3,true>",
                        "attention_hd_kernel<4,true>", "attention_hd_kernel<3,false>", "attention_hd_kernel<4,false>"}
    for inst, fams in got.items():
        assert fams == want, f"{inst} misses {want - fams}"
    # every partial last slice: k = 5, 7, 10, 13 (and the Q-streaming <3, false> at k = 9)
    layouts = {M.slices(d) for d in M.WIDTHS if d > 64}
    assert {(5, 2, 3), (7, 2, 4), (9, 3, 3), (10, 3, 4), (13, 4, 4)} <= layouts
    Ts = {c[2] for c in CASES}
    assert {1, 63, 64, 65, 129} <= Ts and max(Ts) >= 1000


# ------------------------------------------------------------------------------------------------------------------
# the older tests' inputs
# ------------------------------------------------------------------------------------------------------------------
def _walk_reference_layout(qh, C, d):
    """walk over qh [N, 3C, T] (the reference's layout of test_gpu_heads / test_gpu_geometry)."""
    return M.walk_qkv(qh.permute(0, 2, 1).float().numpy(), C, d)


def test_existing_heads_and_geometry_inputs_never_rescale():
    rows = 0
    # test_gpu_heads.py::test_attention_heads_matches_torch
    for d, T in [(d, T) for d in (128, 192, 256, 384, 512, 1024) for T in (64, 256, 1024)] + \
            [(d, 4096) for d in (128, 192, 256)]:
        C = 2 * d if d <= 512 else d
        N = 1 if T == 4096 else 2
        qh = torch.randn(N, 3 * C, T, generator=torch.Generator().manual_seed(d * 7 + T)).half()
        st = _walk_reference_layout(qh, C, d)
        assert int((st["rescales"] > 0).sum()) == 0
        rows += st["rescales"].size
    assert rows == 54144
    # test_gpu_geometry.py::test_attention_any_length_matches_torch
    rows = 0
    for d in (64, 128, 192, 512):
        for T in (1, 15, 16, 36, 60, 100, 144, 240, 576, 1000):
            C = 2 * d if d < 512 else d
            qh = torch.randn(2, 3 * C, T, generator=torch.Generator().manual_seed(T * 7 + d)).half()
            st = _walk_reference_layout(qh, C, d)
            assert int((st["rescales"] > 0).sum()) == 0
            rows += st["rescales"].size
    assert rows == 30632


def test_existing_load_test_inputs_rescale_rarely():
    """test_gpu_ops.py::test_attention_is_deterministic_under_load, sample 0 (d = 64): about 1 % of the rows rescale."""
    hit = rows = 0
    for N, T, C in [(32, 256, 768), (32, 1024, 512), (8, 4096, 256)]:
        qkv = (torch.randn(N, T, 3 * C, generator=torch.Generator().manual_seed(T)) * 1.5).half()
        st = M.walk_qkv(qkv[:1].float().numpy(), C, 64)
        hit += int((st["rescales"] > 0).sum())
        rows += st["rescales"].size
    assert rows == 27648
    print(f"[model] load-test sample 0: {hit} of {rows} rows rescale after block 0")
    assert 0 < hit < 0.03 * rows


# ------------------------------------------------------------------------------------------------------------------
# the partial-slice network with peaked attention
# ------------------------------------------------------------------------------------------------------------------
def _attention_qkv(cfg, sd, monkeypatch):
    from oracle import unet_ref
    seen = []
    orig = unet_ref._attention

    def spy(x, sd_, p, groups, head_ch):
        b, c, hh, ww = x.shape
        xf = x.reshape(b, c, -1)
        qkv = torch.nn.functional.conv1d(unet_ref._group_norm(xf, sd_, p + ".norm", groups), sd_[p + ".qkv.weight"],
                                         sd_[p + ".qkv.bias"])
        seen.append((p, head_ch, qkv))
        return orig(x, sd_, p, groups, head_ch)

    monkeypatch.setattr(unet_ref, "_attention", spy)
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.standard_normal((1, 4, 32, 32)).astype(np.float32))
    unet_ref.unet_forward(cfg, sd, x, torch.tensor([500]), torch.tensor([3]))
    return seen


def test_peaked_network_attention_rescales(monkeypatch):
    from oracle import unet_ref
    cfg = M.PARTIAL_SLICE_CFG
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=77)
    frac = {}
    for tag, s in (("plain", sd), ("peaked", M.peaked_state_dict(sd))):
        hit = rows = 0
        for p, d, qkv in _attention_qkv(cfg, s, monkeypatch):
            assert (d, qkv.shape[-1]) in ((320, 256), (640, 64))
            if d == 640:
                continue                    # T = 64: one key block, nothing to rescale
            st = M.walk_qkv(qkv.permute(0, 2, 1).half().float().numpy(), qkv.shape[1] // 3, d)
            hit += int((st["rescales"] > 0).sum())
            rows += st["rescales"].size
        frac[tag] = hit / rows
        print(f"[model] partial-slice network, {tag}: {hit} of {rows} T = 256 rows rescale after block 0")
    assert frac["plain"] == 0.0 and frac["peaked"] > 0.15
