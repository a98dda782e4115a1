"""CPU tests of what every kernel-backed module shares (models/base.py): `.to(dtype)` selects the output dtype only,
`generation` counts parameter changes, there is no CPU engine, and `.config` reads like a mapping."""
import pytest
import torch

BOC, HEADS, CROSS, GROUPS = (32, 64, 128, 128), 4, 64, 8


def _net(cls_name, cin):
    def make():
        from powerpaint_b200 import models
        from powerpaint_b200.engine import NetConfig

        return getattr(models, cls_name)(NetConfig(in_channels=cin, block_out_channels=BOC, attention_head_dim=HEADS,
                                                   cross_attention_dim=CROSS, norm_num_groups=GROUPS))
    return make


def _vae():
    from powerpaint_b200.models import AutoencoderKL

    return AutoencoderKL(block_out_channels=(16, 32, 32, 32), norm_num_groups=8, layers_per_block=1)


def _clip():
    from powerpaint_b200.models import CLIPTextModel

    return CLIPTextModel(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1,
                         num_attention_heads=2, max_position_embeddings=8)


MODULES = {"unet": _net("UNet2DConditionModel", 9), "brushnet": _net("BrushNetModel", 4),
           "controlnet": _net("ControlNetModel", 4), "vae": _vae, "text_encoder": _clip}
CONFIG_KEYS = {"unet": "in_channels", "brushnet": "in_channels", "controlnet": "in_channels",
               "vae": "scaling_factor", "text_encoder": "hidden_size"}


@pytest.mark.parametrize("name", list(MODULES))
def test_to_dtype_selects_the_output_dtype_only(name):
    m = MODULES[name]()
    assert m.dtype == torch.float32
    assert m.to(torch.float16) is m
    assert m.dtype == torch.float16 and all(p.dtype == torch.float32 for p in m.parameters())
    assert m.to(dtype=torch.bfloat16) is m and m.dtype == torch.bfloat16
    assert m.to("cpu", torch.float16) is m and m.dtype == torch.float16
    assert all(p.dtype == torch.float32 for p in m.parameters())


@pytest.mark.parametrize("name", list(MODULES))
def test_generation_rises_when_the_parameters_change(name):
    m = MODULES[name]()
    g0 = m.generation
    m.load_state_dict(m.state_dict(), strict=True)
    g1 = m.generation
    assert g1 > g0
    m.to("cpu")
    assert m.generation > g1
    g2 = m.generation
    m.to(torch.float16)  # a dtype alone moves no parameter
    assert m.generation == g2


@pytest.mark.parametrize("name", list(MODULES))
def test_no_engine_on_the_cpu(name):
    m = MODULES[name]()
    with pytest.raises(RuntimeError, match="CUDA"):
        m.engine()
    assert m._engine is None


def _schedulers():
    from powerpaint_b200 import schedulers as S

    return [S.DDIMScheduler(), S.UniPCMultistepScheduler(), S.DPMSolverMultistepScheduler(),
            S.EulerDiscreteScheduler(), S.EulerAncestralDiscreteScheduler(), S.PNDMScheduler(skip_prk_steps=True)]


@pytest.mark.parametrize("name", list(MODULES))
def test_config_mapping_access(name):
    cfg = MODULES[name]().config
    key = CONFIG_KEYS[name]
    assert cfg[key] == getattr(cfg, key) and cfg.get(key) == getattr(cfg, key)
    assert key in cfg and "no_such_key" not in cfg and cfg.get("no_such_key", 7) == 7
    assert key in cfg.keys() and set(cfg.keys()) == set(vars(cfg))


def test_scheduler_config_mapping_access():
    for s in _schedulers():
        cfg = s.config
        assert cfg["num_train_timesteps"] == cfg.num_train_timesteps == cfg.get("num_train_timesteps") == 1000
        assert "beta_schedule" in cfg and "no_such_key" not in cfg and cfg.get("no_such_key") is None
        assert set(cfg.keys()) == set(vars(cfg))
        assert type(s).from_config(cfg).config == cfg
