"""CPU: the sampler options shared by the samplers, the pipeline and both command lines (ivid_b200/samplers/options.py):
both command lines parse the shared flags to the same SamplerOptions, the keywords each kind of framework's sampler
takes, and the output directory names the sampling command line derives from them."""
import pytest

import ivid_b200.backbones as backbones
import ivid_b200.frameworks as frameworks
from ivid_b200.inference import sample as sample_cli
from ivid_b200.inference import upsample
from ivid_b200.samplers.options import SamplerOptions, check_arguments

TINY = dict(image_size=32, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=1,
            attention_resolutions=[16], channel_mult=[1, 2], num_head_channels=64)

FLAGS = ["--guidance_interval", "100,600", "--cache_interval", "3", "--cache_branch", "1", "--dynamic_threshold", "0.9,2",
         "--pag_scale", "1.5", "--pag_layers", "input_blocks.7.1,middle_block.1", "--apg", "0,2,-0.5"]


class _Parsed(Exception):
    pass


def _upsample_args(argv, monkeypatch):
    """The namespace upsample.main parses from argv: main stops once its flags are checked."""
    def stop(ap, opt):
        check_arguments(ap, opt)
        raise _Parsed(opt)
    monkeypatch.setattr(upsample, "check_arguments", stop)
    with pytest.raises(_Parsed) as e:
        upsample.main(["--scene_dir", "x", "--config_sr", "sr.json"] + argv)
    return e.value.args[0]


@pytest.mark.parametrize("argv", [[], FLAGS, ["--solver", "unipc", "--precision", "fp8", "--dynamic_threshold", "0.995",
                                              "--apg", "1", "--pag_scale", "0"]])
def test_both_command_lines_parse_the_same_options(argv, monkeypatch):
    a, b = sample_cli.parse_args(argv), _upsample_args(argv, monkeypatch)
    assert SamplerOptions.from_args(a) == SamplerOptions.from_args(b)
    assert (a.solver, a.precision) == (b.solver, b.precision)
    if argv == FLAGS:
        assert SamplerOptions.from_args(a) == SamplerOptions((100, 600), 3, 1, (0.9, 2.0), 1.5,
                                                             ("input_blocks.7.1", "middle_block.1"), (0.0, 2.0, -0.5))


@pytest.mark.parametrize("bad", [["--pag_layers", "middle_block.1"], ["--solver", "euler"], ["--cache_branch", "-1"]])
def test_both_command_lines_reject(bad, monkeypatch):
    with pytest.raises(SystemExit):
        sample_cli.parse_args(bad)
    with pytest.raises(SystemExit):
        _upsample_args(bad, monkeypatch)


def test_sampler_kwargs():
    cfg = frameworks.ClassifierFreeGuidance(backbones.AdmUnet2d(**TINY), timesteps=1000, beta_schedule="linear")
    plain = frameworks.GaussianDiffusion(backbones.AdmUnet2d(**TINY), timesteps=1000, beta_schedule="linear")
    o = SamplerOptions(guidance_interval=[100, 600], cache_interval=3, cache_branch=1)
    assert o.sampler_kwargs(cfg, 2.0) == dict(strength=2.0, guidance_interval=(100, 600), cache_interval=3, cache_branch=1)
    assert o.sampler_kwargs(plain, 2.0) == dict(cache_interval=3, cache_branch=1)
    o = SamplerOptions(guidance_interval=(100, 600), pag_scale=1.0, dynamic_threshold=0.99)
    assert o.sampler_kwargs(plain, 2.0) == dict(guidance_interval=(100, 600), pag_scale=1.0, pag_layers=None, dynamic_threshold=0.99)
    assert SamplerOptions().sampler_kwargs(cfg, 3.0) == dict(strength=3.0)
    assert SamplerOptions().sampler_kwargs(plain, 3.0) == {}
    assert SamplerOptions(apg=(0.0, 1.0)).sampler_kwargs(cfg, 3.0) == dict(strength=3.0, apg=(0.0, 1.0))


# output_dir_name of these command lines: the directories of existing runs carry these names, so they must not change
DIR_NAMES = [
    ([], "viewset_3x9_steps_u1000_c50_guidance3.0"),
    (["--solver", "dpmpp", "--precision", "fp8"], "viewset_3x9_steps_u1000_c50_guidance3.0_dpmpp_fp8"),
    (["--guidance_interval", "100,600", "--cache_interval", "3", "--cache_branch", "1"],
     "viewset_3x9_steps_u1000_c50_guidance3.0_interval100-600_cache3b1"),
    (["--dynamic_threshold", "0.995"], "viewset_3x9_steps_u1000_c50_guidance3.0_dthresh0.995"),
    (["--dynamic_threshold", "0.9,2", "--init_image", "dir/photo.png", "--init_depth", "photo.npz", "--init_strength", "0.6"],
     "viewset_3x9_steps_u1000_c50_guidance3.0_dthresh0.9-2.0_init-photo_strength0.6"),
    (["--pag_scale", "1.5", "--pag_layers", "input_blocks.7.1,middle_block.1", "--apg", "0,2"],
     "viewset_3x9_steps_u1000_c50_guidance3.0_pag1.5-input_blocks.7.1+middle_block.1_apg0.0,2.0"),
    (["--solver", "unipc", "--guidance_interval", "0,999", "--cache_interval", "2", "--dynamic_threshold", "0.99,1.5",
      "--init_image", "a.jpg", "--init_depth", "a.npy", "--pag_scale", "2", "--apg", "0.5,0,-0.5", "--config_sr", "sr.json",
      "--steps_sr", "20"],
     "viewset_3x9_steps_u1000_c50_guidance3.0_unipc_interval0-999_cache2b0_dthresh0.99-1.5_init-a_pag2.0_apg0.5,0.0,-0.5_sr20"),
    (["--solver", "dpmpp_sde", "--pag_scale", "0", "--pag_layers", "middle_block.1", "--apg", "1", "--config_sr", "sr.json",
      "--sr_replace", "none"],
     "viewset_3x9_steps_u1000_c50_guidance3.0_dpmpp_sde_pag0.0_apg1.0_sr50-noreplace"),
]


@pytest.mark.parametrize("argv,name", DIR_NAMES)
def test_output_dir_names_unchanged(argv, name):
    assert sample_cli.output_dir_name(sample_cli.parse_args(argv)) == "samples/imagenet128/" + name
