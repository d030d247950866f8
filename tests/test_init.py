"""CPU: the host side of starting a run from a given image (`init` / `init_strength`, `sample_all(init_views=...)`,
`--init_image`): the datasets' preprocessing restated on the host against the reference's, the executed-step arithmetic,
the argument checks of the C ABI and of the Python samplers (before any device work), and the CLI."""
import ctypes
import inspect
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
import ivid_b200.samplers as samplers
from ivid_b200 import _lib
from ivid_b200.inference import sample as sample_cli

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = np.load(os.path.join(HERE, "golden", "init_golden.npz"))
CASES = json.loads(GOLDEN["prep_cases"].tobytes())
T = 1000
TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64)
SAMPLERS = (samplers.DdpmSampler, samplers.DdimSampler, samplers.DpmSolverSampler, samplers.UniPcSampler)


def _tiny_fw():
    return frameworks.ClassifierFreeGuidance(backbones.AdmUnet2d(**TINY), timesteps=T, beta_schedule="linear")


def _case(tag):
    args = json.loads(GOLDEN[f"prep_{tag}_args"].tobytes())
    return GOLDEN[f"prep_{tag}_image"], GOLDEN[f"prep_{tag}_disparity"], args, GOLDEN[f"prep_{tag}_x0"]


@pytest.mark.parametrize("tag", CASES)
def test_preprocessing_matches_reference(tag):
    """preprocess_init_view equals BaseDataset.get_file + process_file of the reference bit for bit: every prepocess_depth
    mode, landscape, portrait and grayscale images, and the conditional config's dataset.args at its image_size."""
    img, disp, args, ref = _case(tag)
    got = sample_cli.preprocess_init_view(Image.fromarray(img), disp, **args).numpy()
    assert got.dtype == np.float32 and got.shape == ref.shape
    assert np.array_equal(got, ref), f"{tag}: max |diff| {np.abs(got - ref).max()}"


@pytest.mark.parametrize("fmt", ["npz", "npy"])
def test_load_init_view_reads_files(tmp_path, fmt):
    """--init_image / --init_depth files: a PNG and a disparity map stored as .npz (arr_0) or .npy."""
    img, disp, args, ref = _case("cond")
    Image.fromarray(img).save(tmp_path / "view.png")
    depth_path = tmp_path / f"view.{fmt}"
    np.savez(depth_path, disp) if fmt == "npz" else np.save(depth_path, disp)
    size = args.pop("image_size")
    got = sample_cli.load_init_view(str(tmp_path / "view.png"), str(depth_path), args, size)
    assert np.array_equal(got.numpy(), ref)


@pytest.mark.parametrize("steps", [1, 2, 10, 50, 1000])
def test_executed_steps(steps):
    """n = min(steps, max(1, round(s * steps))): strength 1 runs the full grid, a tiny strength one step."""
    assert samplers.init_steps(1.0, steps) == steps
    assert samplers.init_steps(1e-9, steps) == 1
    for s in np.linspace(0.01, 1.0, 37):
        n = samplers.init_steps(float(s), steps)
        assert 1 <= n <= steps and n == min(steps, max(1, int(s * steps + 0.5)))
    assert samplers.init_steps(0.25, 1000) == 250 and samplers.init_steps(0.5, 50) == 25
    assert samplers.init_steps(0.5, 3) == 2 and samplers.init_steps(0.1, 4) == 1


def test_native_rejects_bad_start_step_and_diffuse():
    """start_step outside [0, steps) (steps = T for DDPM), and a diffuse with t outside [0, T) or a per-sample count that is
    not a multiple of 4: IVID_ERR_INVALID_ARGUMENT before any device work (the pointers are never dereferenced)."""
    L = _lib.lib()
    unet = ctypes.c_void_p()
    _lib.check(L.ivid_unet_create(json.dumps(TINY).encode(), ctypes.byref(unet)))
    s = samplers.DdimSampler(_tiny_fw())
    fake = ctypes.c_void_p(256)
    try:
        for kind, steps, bad in ((0, 10, (-1, T, T + 5)), (1, 10, (-1, 10, 11)), (2, 25, (-3, 25))):
            for start in bad:
                a = _lib.StepArgsT()
                a.kind, a.start_step = kind, start
                rc = L.ivid_sampler_run(s._handle, unet, fake, 1, steps, ctypes.byref(a), None, None, None, None, None)
                assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "start_step" in _lib.last_error(), (kind, start)
        for t, count in ((-1, 16), (T, 16), (5, 6), (5, 0)):
            rc = L.ivid_sampler_diffuse(s._handle, fake, None, 1, count, t, 0, fake, None)
            assert rc == _lib.IVID_ERR_INVALID_ARGUMENT and "diffuse" in _lib.last_error(), (t, count)
    finally:
        L.ivid_unet_destroy(unet)


BAD_INIT = [
    (dict(init_strength=0.5), "init_strength needs init"),
    (dict(init=torch.zeros(1, 4, 32, 32)), "init needs init_strength"),
    (dict(init=torch.zeros(1, 4, 32, 32), init_strength=0.0), "init_strength must be in"),
    (dict(init=torch.zeros(1, 4, 32, 32), init_strength=1.5), "init_strength must be in"),
    (dict(init=torch.zeros(1, 4, 32, 32), init_strength=True), "init_strength must be in"),
    (dict(init=torch.zeros(1, 3, 32, 32), init_strength=0.5), "init must be an"),
    (dict(init=torch.zeros(4, 32, 32), init_strength=0.5), "init must be an"),
    (dict(init=torch.zeros(1, 4, 32, 32), init_strength=0.5, image_size=32), "image_size"),
    (dict(init=torch.zeros(2, 4, 32, 32), init_strength=0.5, noise=torch.zeros(1, 4, 32, 32)), "noise"),
]


@pytest.mark.parametrize("kw,msg", BAD_INIT, ids=[f"case{i}" for i in range(len(BAD_INIT))])
def test_python_rejects_bad_init(kw, msg, monkeypatch):
    """AssertionError from every sampler's sample, before the network is packed and before any torch draw."""
    fw = _tiny_fw()

    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(type(fw.backbone), "_ensure_packed", no_device)
    for cls in SAMPLERS:
        s = cls(fw)
        state = torch.get_rng_state()
        with pytest.raises(AssertionError, match=msg):
            s.sample(1, steps=10, verbose=False, **kw)
        assert torch.equal(state, torch.get_rng_state())


def test_python_surface():
    for cls in SAMPLERS:
        params = inspect.signature(cls.sample).parameters
        assert params["init"].default is None and params["init_strength"].default is None
        assert "init" not in inspect.signature(cls.sample_once).parameters
    params = inspect.signature(sample_cli.sample_all).parameters
    assert params["init_views"].default is None and params["init_strength"].default is None
    assert _lib.StepArgsT().start_step == 0, "a zeroed ivid_step_args_t runs the whole grid"
    names = [f[0] for f in _lib.StepArgsT._fields_]
    assert names[names.index("start_step") + 1:] == ["dynamic_threshold", "threshold_ratio", "threshold_max"], \
        "start_step follows every field but the dynamic-threshold ones, which stay last"


def test_sample_all_rejects_bad_init_views():
    fw = _tiny_fw()
    mv = sample_cli.build_modelviews("uncond", 1)
    with pytest.raises(AssertionError, match="init_strength needs init_views"):
        next(sample_cli.sample_all(fw, None, 1, 10, 10, mv, init_strength=0.5))
    with pytest.raises(AssertionError, match="framework_uncond is needed"):
        next(sample_cli.sample_all(None, fw, 1, 10, 10, mv, init_views=torch.zeros(1, 4, 32, 32), init_strength=0.5))
    with pytest.raises(AssertionError, match="init_views must be"):
        next(sample_cli.sample_all(None, fw, 1, 10, 10, mv, init_views=torch.zeros(1, 3, 32, 32)))


def test_cli_parses():
    o = sample_cli.parse_args(["--init_image", "photo.png", "--init_depth", "photo.npz", "--init_strength", "0.6"])
    assert (o.init_image, o.init_depth, o.init_strength) == ("photo.png", "photo.npz", 0.6)
    assert sample_cli.output_dir_name(o).endswith("_init-photo_strength0.6")
    o = sample_cli.parse_args(["--init_image", "photo.png", "--init_depth", "photo.npy"])
    assert o.init_strength is None and sample_cli.output_dir_name(o).endswith("_init-photo")
    plain = sample_cli.parse_args([])
    assert (plain.init_image, plain.init_depth, plain.init_strength) == (None, None, None)
    assert "init" not in os.path.basename(sample_cli.output_dir_name(plain))
    for bad in (["--init_strength", "0.5"], ["--init_image", "a.png"], ["--init_depth", "a.npz"],
                ["--init_image", "a.png", "--init_depth", "a.npz", "--init_strength", "0"],
                ["--init_image", "a.png", "--init_depth", "a.npz", "--init_strength", "1.2"],
                ["--init_image", "a.png", "--init_depth", "a.npz", "--init_strength", "x"]):
        with pytest.raises(SystemExit):
            sample_cli.parse_args(bad)
