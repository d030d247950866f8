"""CPU: the bounds of tests/network_ends_model.py hold for the faithful two-term split and fail for each dropped term, on
the inputs tests/test_gpu_network_ends.py uses; and the embedding cases of that test reach every kernel that the launch
rule can pick for a network."""
import pytest
import torch

import network_ends_model as NM
from oracle import unet_ref

CFGS = NM.golden_cfgs()


@pytest.mark.parametrize("cin", [4, 3, 7])
def test_stem_bound_sees_each_split_term(cin):
    cfg = dict(CFGS["tiny"], in_channels=cin)
    sd = NM.coherent_state_dict(cfg)
    x = NM.stem_input(1, cin, 32, 32, seed=cin)
    w, b = sd["input_blocks.0.0.weight"], sd["input_blocks.0.0.bias"]
    ref, S = NM.stem_reference(x, w, b)
    bound = NM.stem_bound(S, w, b)
    r = {m: NM.worst(NM.split_products(x, w, m) + b.double()[None, :, None, None], ref, bound)[0] for m in NM.MODES}
    print(f"[ends-model] stem Cin={cin}: " + "  ".join(f"{m} {v:.3f}" for m, v in r.items()))
    assert r["split"] <= 0.1
    for m in ("no_lo", "no_wl", "none"):
        assert r[m] >= 5.0, f"stem bound does not see the dropped term ({m}: {r[m]:.2f}x)"


def _head_case(cfg):
    sd = NM.coherent_state_dict(cfg)
    x = torch.randn(1, cfg["in_channels"], 32, 32, generator=torch.Generator().manual_seed(3))
    taps = {}
    unet_ref.unet_forward(cfg, sd, x, torch.tensor([250]), torch.tensor([4]), taps=taps)
    blocks, _ = unet_ref._topology(cfg)
    eps, y, dy = NM.head_reference(taps[blocks[-1]["layers"][-1][1]], sd, cfg["num_groups"])
    return sd, eps, y, dy


def test_head_bound_sees_the_weight_split():
    """The split head against its bound.  The weights are coherent (positive, off the grid), so a dropped Wl or a dropped
    split shifts every output the same way.  The activation is a normalised tensor whose lo terms have random signs; a
    dropped a_lo is a random walk over 9 C products, printed but not required to exceed the bound."""
    sd, eps, y, dy = _head_case(CFGS["tiny"])
    w, b = sd["out.2.weight"], sd["out.2.bias"]
    split = NM.head_bound(y, dy, w, b, split=True)
    unsplit = NM.head_bound(y, dy, w, b, split=False)
    emu = lambda m: NM.split_products(y, w, m) + b.double()[None, :, None, None]
    r = {m: NM.worst(emu(m), eps, split)[0] for m in NM.MODES}
    r_un = NM.worst(emu("none"), eps, unsplit)[0]
    print(f"[ends-model] head tiny: " + "  ".join(f"{m} {v:.3f}" for m, v in r.items()) + f"  fp16 head vs its own bound {r_un:.3f}")
    assert r["split"] <= 0.1
    assert r["no_wl"] >= 5.0 and r["none"] >= 5.0
    assert r_un <= 0.5


def test_embedding_bound_holds_for_torch_fp32():
    """The oracle's fp32 torch embedding (another fp32 evaluation order) lies inside the bound at the widest config."""
    cfg = CFGS["large"]
    sd = unet_ref.make_synthetic_state_dict(cfg, seed=5)
    t = torch.tensor([0, 1, 500, 998, 999])
    c = torch.tensor([3, -1, 999, 0, 7])
    taps = {}
    unet_ref.unet_forward(cfg, sd, torch.zeros(5, 4, 16, 16), t, c, taps=taps)
    ref, bound = NM.embedding_reference(cfg, sd, t, c)
    r = NM.worst(taps["emb"], ref, bound)[0]
    film, fb = NM.film_reference(cfg, sd, taps["emb"])
    W, bf = NM.film_weights(cfg, sd)
    rf = NM.worst(torch.nn.functional.linear(torch.nn.functional.silu(taps["emb"]), W, bf), film, fb)[0]
    print(f"[ends-model] torch fp32 emb {r:.3f}, film {rf:.3f}")
    assert r <= 0.5 and rf <= 0.5


# configuration -> what tests/test_gpu_network_ends.py expects each embedding stage to run
EMBED_CASES = {
    "tiny": ("linear_tiled_kernel<2>", "linear_warp_kernel<2>", "film_table_kernel, full tiles"),
    "single": ("linear_tiled_kernel<2>", "linear_warp_kernel<4>", "film_table_kernel, full tiles"),
    "large": ("linear_warp_kernel<2>", "linear_warp_kernel<8>", "film_table_kernel, full tiles"),
    "g8": ("linear_rows_kernel", "linear_tiled_kernel<2>", "film_table_kernel, partial tile"),
    "g4_40": ("linear_rows_kernel", "linear_rows_kernel", "linear_rows_kernel"),
    "mc96": ("linear_tiled_kernel<2>", "linear_tiled_kernel<2>", "film_table_kernel, full tiles"),
}


def test_embedding_cases_reach_every_kernel_a_network_reaches():
    reached = set()
    for tag, want in EMBED_CASES.items():
        k = NM.embedding_kernels(CFGS[tag])
        assert (k["time_embed.1"], k["time_embed.3"], k["film"]) == want, tag
        reached.update(want)
    assert NM.film_total(CFGS["large"]) == 40960 and NM.film_total(CFGS["g8"]) % 128 == 96
    # every kernel the rule picks for some model width, except linear_tiled_kernel<4>
    possible = set()
    for mc in range(1, 2048):
        possible.update(NM.embedding_kernels(dict(CFGS["tiny"], model_channels=mc)).values())
    possible.update(f"film_table_kernel, {s}" for s in ("full tiles", "partial tile"))
    assert "linear_tiled_kernel<4>" not in possible
    assert possible <= reached, possible - reached
    # linear_tiled_kernel<4> takes O >= 8192 outputs: the time_embed Linears of model_channels >= 2048, 8x the widest
    # shipped model (256).  No test builds such a network; DESIGN.md §2 says so.
    assert NM.linear_kernel(2048, 8192) == "linear_tiled_kernel<4>" and NM.linear_kernel(8192, 8192) == "linear_tiled_kernel<4>"
