"""CPU: the super-resolution stage of the multiview pipeline - its flags and output directory suffixes, every argument error
raised before any device work, the class / seed tags of scene names, the render size of a scene file, and the plumbing
of sample_all into the stage."""
import os

import numpy as np
import pytest
import torch

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
from ivid_b200.inference import sample as sample_cli
from ivid_b200.inference import superres, upsample
from ivid_b200.inference.render import scene_image_size
from ivid_b200.inference.utils import save_scene
from ivid_b200.utils import edict

T = 1000
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64, num_classes=10, has_null_class=True)
TINY_COND = dict(TINY, in_channels=9)
TINY_SR = dict(TINY, in_channels=8)


def _fw(cls=frameworks.SuperResCFG, cfg=TINY_SR):
    return cls(backbones.AdmUnet2d(**cfg), timesteps=T, beta_schedule="linear")


# ---------------------------------------------------------------------------------------------------------------------
# CLI
# ---------------------------------------------------------------------------------------------------------------------
def test_flags_defaults_and_suffixes():
    plain = sample_cli.parse_args([])
    assert plain.config_sr is None and "_sr" not in sample_cli.output_dir_name(plain)
    o = sample_cli.parse_args(["--config_sr", "sr.json"])
    assert o.steps_sr == 50 and o.sr_replace == (0.1, 0.2) and o.ckpt_sr is None
    assert sample_cli.output_dir_name(o).endswith("_sr50")
    o = sample_cli.parse_args(["--config_sr", "sr.json", "--ckpt_sr", "sr.pt", "--steps_sr", "20", "--sr_replace", "none"])
    assert o.ckpt_sr == "sr.pt" and o.steps_sr == 20 and o.sr_replace is None
    assert sample_cli.output_dir_name(o).endswith("_sr20-noreplace")
    o = sample_cli.parse_args(["--config_sr", "sr.json", "--sr_replace", "0.3,0"])
    assert o.sr_replace == (0.3, 0.0) and sample_cli.output_dir_name(o).endswith("_sr50-replace0.3-0.0")
    o = sample_cli.parse_args(["--config_sr", "sr.json", "--sr_replace", "0.1,0.2"])
    assert sample_cli.output_dir_name(o).endswith("_sr50")
    o = sample_cli.parse_args(["--config_sr", "sr.json", "--apg", "0"])
    assert sample_cli.output_dir_name(o).endswith("_apg0.0_sr50")


@pytest.mark.parametrize("argv", [["--ckpt_sr", "sr.pt"], ["--steps_sr", "50"], ["--sr_replace", "none"],
                                  ["--sr_replace", "0.1,0.2"], ["--config_sr", "sr.json", "--steps_sr", "0"],
                                  ["--config_sr", "sr.json", "--sr_replace", "0.1"],
                                  ["--config_sr", "sr.json", "--sr_replace", "1.5,0.2"],
                                  ["--config_sr", "sr.json", "--sr_replace", "0.1,-0.2"],
                                  ["--config_sr", "sr.json", "--sr_replace", "a,b"]])
def test_flag_errors(argv):
    with pytest.raises(SystemExit):
        sample_cli.parse_args(argv)


def test_upsample_flags():
    with pytest.raises(SystemExit):
        upsample.main(["--scene_dir", "x"])                     # --config_sr is required
    with pytest.raises(SystemExit):
        upsample.main(["--scene_dir", "x", "--config_sr", "sr.json", "--sr_replace", "2,0"])
    assert upsample.output_dir(os.path.join("a", "run") + os.sep, 20) == os.path.join("a", "run_sr20")


# ---------------------------------------------------------------------------------------------------------------------
# argument errors before any device work
# ---------------------------------------------------------------------------------------------------------------------
def _no_device(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(backbones.AdmUnet2d, "_ensure_packed", no_device)
    monkeypatch.setattr(superres, "DeviceWarp", no_device)
    monkeypatch.setattr(backbones.AdmUnet2d, "set_precision", no_device)


BAD = [
    (dict(size=48), ValueError, "integer multiple"),
    (dict(size=32), ValueError, "integer multiple"),
    (dict(size=16), ValueError, "integer multiple"),
    (dict(size=None), ValueError, "integer multiple"),          # the backbone's image_size (32) is x1
    (dict(size=64.0), ValueError, "positive integer"),
    (dict(size=64, replace=(1.5, 0.2)), ValueError, "in \\[0, 1\\]"),
    (dict(size=64, replace=(0.1, -0.1)), ValueError, "in \\[0, 1\\]"),
    (dict(size=64, replace=(0.1, float("nan"))), ValueError, "in \\[0, 1\\]"),
    (dict(size=64, replace=(0.1,)), ValueError, "replace must be"),
    (dict(size=64, apg=0.0), AssertionError, "needs classes"),
    (dict(size=64, apg=(0.0, 0.0, 2.0), classes=[1]), AssertionError, "momentum beta"),
    (dict(size=64, cache_interval=0), AssertionError, "cache_interval"),
    (dict(size=64, cache_branch=5), AssertionError, "cache_branch"),
    (dict(size=64, pag_scale=1.0, pag_layers=("nope",)), Exception, "nope"),
    (dict(size=64, dynamic_threshold=1.5), AssertionError, "dynamic_threshold"),
    (dict(size=64, guidance_interval=(10, 2000)), AssertionError, "guidance_interval"),
    (dict(size=64, solver="ddpm"), AssertionError, "solver"),
    (dict(size=64, steps=0), AssertionError, "steps"),
    (dict(size=64, seeds=[1, 2]), AssertionError, "one seed per sample"),
]


@pytest.mark.parametrize("kw,exc,msg", BAD, ids=[f"case{i}" for i in range(len(BAD))])
def test_stage_rejects_before_device_work(kw, exc, msg, monkeypatch):
    fw = _fw()
    _no_device(monkeypatch)
    views = torch.zeros(1, 2, 4, 32, 32)
    mvs = sample_cli.build_modelviews("3x9", 1)[:2]
    state = torch.get_rng_state()
    with pytest.raises(exc, match=msg):
        superres.superresolve_views(fw, views, mvs, **kw)
    assert torch.equal(state, torch.get_rng_state())


def test_stage_rejects_other_frameworks(monkeypatch):
    _no_device(monkeypatch)
    for fw in (_fw(frameworks.ClassifierFreeGuidance, TINY), _fw(frameworks.InpaintCFG, TINY_COND)):
        with pytest.raises(ValueError, match="SuperResCFG"):
            superres.superresolve_views(fw, torch.zeros(1, 1, 4, 16, 16), sample_cli.build_modelviews("uncond", 1))


def test_sample_all_rejects_before_device_work(monkeypatch):
    """sample_all checks the stage's arguments before the first view is sampled."""
    _no_device(monkeypatch)
    fw_u, fw_c = _fw(frameworks.ClassifierFreeGuidance, TINY), _fw(frameworks.InpaintCFG, TINY_COND)
    mv = sample_cli.build_modelviews("3x9", 1)
    for kw, exc in ((dict(framework_sr=_fw()), ValueError), (dict(framework_sr=_fw(), sr_size=80), ValueError),
                    (dict(framework_sr=_fw(), sr_size=64, sr_replace=(0.1, 2.0)), ValueError),
                    (dict(framework_sr=fw_u, sr_size=64), ValueError),
                    (dict(framework_sr=_fw(), sr_size=64, steps_sr=0), AssertionError)):
        with pytest.raises(exc):
            next(sample_cli.sample_all(fw_u, fw_c, 1, 10, 10, mv, classes=[3], **kw))
    # the stage's own guidance: APG needs it > 0 even where the 128^2 networks' guidance is
    with pytest.raises(AssertionError, match="strength > 0"):
        next(sample_cli.sample_all(fw_u, fw_c, 1, 10, 10, mv, classes=[3], framework_sr=_fw(), sr_size=64, sr_guidance=0.0,
                                   apg=0.0))


# ---------------------------------------------------------------------------------------------------------------------
# sample_all -> stage plumbing (samplers and warp replaced by recorders)
# ---------------------------------------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self):
        self.calls = []

    def sampler(self, name):
        rec = self

        class Fake:
            def __init__(self, fw):
                self.fw = fw

            def sample(self, num, **kw):
                """x_T as the native samplers take it: the given noise, else drawn from the torch RNG at image_size (None:
                the backbone's), followed by the draw of the Philox seed; the fake returns x_T."""
                rec.calls.append((name, type(self.fw).__name__, kw))
                if kw.get("noise") is not None:
                    x = kw["noise"].clone()
                else:
                    S = kw.get("image_size") or self.fw.backbone.image_size
                    x = torch.randn(num, 4, S, S)
                torch.randint(0, 2 ** 62, (1,))
                return edict(samples=x)
        return Fake


class _FakeWarp:
    def __init__(self, bs, image_size, **kw):
        self.bs, self.S, self.added = bs, image_size, 0

    def reset(self):
        self.added = 0

    def aggregate(self, mv, **kw):
        return torch.zeros(self.bs, 7, self.S, self.S)

    def add_view(self, *a, **k):
        self.added += 1


def test_sample_all_runs_the_stage_with_every_option(monkeypatch):
    rec = _Recorder()
    for name in ("DdimSampler", "DdpmSampler", "DpmSolverSampler", "UniPcSampler"):
        monkeypatch.setattr(sample_cli.samplers, name, rec.sampler(name))
    monkeypatch.setattr(sample_cli, "DeviceWarp", _FakeWarp)
    monkeypatch.setattr(superres, "DeviceWarp", _FakeWarp)
    fw_u, fw_c, fw_sr = _fw(frameworks.ClassifierFreeGuidance, TINY), _fw(frameworks.InpaintCFG, TINY_COND), _fw()
    mvs = sample_cli.build_modelviews("random", 3, rng=np.random.default_rng(0))
    opts = dict(solver="unipc", guidance_interval=(0, 600), cache_interval=2, dynamic_threshold=0.99, pag_scale=0.5, apg=0.0)
    plain = list(sample_cli.sample_all(fw_u, fw_c, [4, 5, 6], 10, 4, mvs, classes=[1, 2, 3], batchsize=2, **opts))
    n_plain = len(rec.calls)
    rec.calls.clear()
    outs = list(sample_cli.sample_all(fw_u, fw_c, [4, 5, 6], 10, 4, mvs, classes=[1, 2, 3], batchsize=2, framework_sr=fw_sr,
                                      steps_sr=7, sr_size=64, sr_guidance=1.5, sr_replace=(0.3, 0.4), **opts))
    sr_calls = [c for c in rec.calls if c[1] == "SuperResCFG"]
    assert len(rec.calls) - len(sr_calls) == n_plain and len(sr_calls) == 2 * 2      # 2 batches x 2 views
    for name, _, kw in sr_calls:
        assert name == "UniPcSampler" and kw["steps"] == 7 and kw["strength"] == 1.5
        assert kw["guidance_interval"] == (0, 600) and kw["cache_interval"] == 2 and kw["dynamic_threshold"] == 0.99
        assert kw["pag_scale"] == 0.5 and kw["apg"] == 0.0 and "constrain_depth" not in kw
        assert kw["noise"].shape[-1] == 64
    assert "replace_rgb" not in sr_calls[0][2] and sr_calls[1][2]["replace_rgb"][0] == 0.3
    assert sr_calls[1][2]["replace_depth"][0] == 0.4
    assert sr_calls[0][2]["classes"].tolist() == [1, 2] and sr_calls[2][2]["classes"].tolist() == [3]
    assert "replace_rgb" not in sr_calls[2][2] and "replace_rgb" in sr_calls[3][2]
    # seeded x_T: row v of randn(V, 4, S', S') of the sample's own generator
    want = torch.randn(2, 4, 64, 64, generator=torch.Generator().manual_seed(6))
    assert torch.equal(sr_calls[2][2]["noise"][0], want[0]) and torch.equal(sr_calls[3][2]["noise"][0], want[1])
    # the stage's y is the low-res view it yields as conds["lowres"]
    assert torch.equal(sr_calls[1][2]["y"][1], outs[1][3]["lowres"][1]) and torch.equal(sr_calls[2][2]["y"][0], outs[2][3]["lowres"][0])
    for (m0, c0, s0, d0), (m1, c1, s1, d1) in zip(plain, outs):
        assert torch.equal(d1["lowres"], s0) and s1.shape == (2, 4, 64, 64)
        assert torch.equal(d1["color"], d0["color"]) and m1[0].depth.shape == (64, 64, 1) and c1[1].shape == (64, 64, 3)


def test_sample_all_uncond_creates_conds(monkeypatch):
    rec = _Recorder()
    for name in ("DdimSampler", "DdpmSampler"):
        monkeypatch.setattr(sample_cli.samplers, name, rec.sampler(name))
    monkeypatch.setattr(superres, "DeviceWarp", _FakeWarp)
    fw_u = _fw(frameworks.ClassifierFreeGuidance, TINY)
    outs = list(sample_cli.sample_all(fw_u, None, 2, 10, 4, sample_cli.build_modelviews("uncond", 1), classes=[1, 2],
                                      framework_sr=_fw(), sr_size=64, sr_replace=None))
    assert len(outs) == 2
    for _, _, samples, conds in outs:
        assert set(conds) == {"lowres"} and conds["lowres"].shape == (1, 4, 32, 32) and samples.shape == (1, 4, 64, 64)
    sr_calls = [kw for _, fw, kw in rec.calls if fw == "SuperResCFG"]
    assert len(sr_calls) == 1 and all(kw["noise"] is None and kw["image_size"] == 64 for kw in sr_calls)


def test_sample_all_unseeded_keeps_the_lowres_views(monkeypatch):
    """Unseeded, the stage draws from a reseeded fork of the torch RNG: the next batch's views are those of the run without
    the stage, and the stage's x_T does not repeat them."""
    rec = _Recorder()
    for name in ("DdimSampler", "DdpmSampler"):
        monkeypatch.setattr(sample_cli.samplers, name, rec.sampler(name))
    monkeypatch.setattr(sample_cli, "DeviceWarp", _FakeWarp)
    monkeypatch.setattr(superres, "DeviceWarp", _FakeWarp)
    fw_u, fw_c = _fw(frameworks.ClassifierFreeGuidance, TINY), _fw(frameworks.InpaintCFG, TINY_COND)
    mvs = sample_cli.build_modelviews("random", 3, rng=np.random.default_rng(0))
    fw_sr = _fw()                               # before seeding: building a network draws its initial weights
    torch.manual_seed(3)
    plain = list(sample_cli.sample_all(fw_u, fw_c, 3, 10, 4, mvs, classes=[1, 2, 3], batchsize=2))
    after_plain = torch.get_rng_state()
    torch.manual_seed(3)
    outs = list(sample_cli.sample_all(fw_u, fw_c, 3, 10, 4, mvs, classes=[1, 2, 3], batchsize=2, framework_sr=fw_sr, sr_size=64))
    assert torch.equal(after_plain, torch.get_rng_state())
    for (_, _, s0, _), (_, _, s1, d1) in zip(plain, outs):
        assert torch.equal(d1["lowres"], s0) and s1.shape == (2, 4, 64, 64)
    # the stage's x_T of batch 0 is not the start of batch 1's draws
    first = outs[0][2][0].flatten()[:64]
    assert not torch.equal(first, outs[2][3]["lowres"][0].flatten()[:64])


def test_sample_all_rejected_stage_changes_no_precision(monkeypatch):
    _no_device(monkeypatch)                     # set_precision raises
    fw_u, fw_c = _fw(frameworks.ClassifierFreeGuidance, TINY), _fw(frameworks.InpaintCFG, TINY_COND)
    mv = sample_cli.build_modelviews("3x9", 1)
    for kw in (dict(sr_size=80), dict(sr_size=64, sr_replace=(0.1, 2.0))):
        with pytest.raises(ValueError):
            next(sample_cli.sample_all(fw_u, fw_c, 1, 10, 10, mv, classes=[3], precision="fp8", framework_sr=_fw(), **kw))
    assert fw_u.backbone.precision == fw_c.backbone.precision == "fp16"


# ---------------------------------------------------------------------------------------------------------------------
# saved scenes
# ---------------------------------------------------------------------------------------------------------------------
def test_scene_tags():
    assert upsample.scene_tags("scene_class003_seed00004.npz") == (3, 4)
    assert upsample.scene_tags("scene_seed00017.npz") == (None, 17)
    assert upsample.scene_tags("scene_class999_00012.npz") == (999, None)
    assert upsample.scene_tags("scene_00012.npz") == (None, None)


def _synthetic_scene(path, n, views=2):
    yy, xx = np.mgrid[0:n, 0:n] / n
    meshes, colors = [], []
    for v, mv in enumerate(sample_cli.build_modelviews("3x9", 1)[:views]):
        meshes.append(edict(depth=(1.5 + 0.2 * np.sin(5 * xx + v))[..., None].astype(np.float32), fov=45.0, modelview=mv))
        colors.append(np.stack([xx, yy, 0.5 + 0 * xx], -1))
    save_scene(path, meshes, colors)


def test_render_size_of_a_scene(tmp_path):
    for n in (32, 64):
        p = os.path.join(tmp_path, f"scene_{n}.npz")
        _synthetic_scene(p, n)
        assert scene_image_size(p) == n


def test_scene_to_model_space(tmp_path):
    p = os.path.join(tmp_path, "scene_class001_seed00002.npz")
    _synthetic_scene(p, 16)
    from ivid_b200.inference import load_scene_views
    views = load_scene_views(p)
    x = upsample.scene_to_model_space(views, 0.6, 5)
    assert x.shape == (2, 4, 16, 16) and x.dtype == torch.float32
    assert torch.equal(x[1, :3], torch.from_numpy(views[1].color.astype(np.float32) * 2 - 1).permute(2, 0, 1))
    d = (1 / 0.6 - 1 / np.clip(views[0].depth[..., 0], 0.6, 5)) / (1 / 0.6 - 1 / 5)
    assert np.allclose(x[0, 3].numpy(), d * 2 - 1, atol=1e-6)
