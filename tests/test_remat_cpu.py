"""use_remat, the recompute-in-the-backward flag of the transformer models, on the host (no GPU): every class takes
it, the parameters and the checkpoint layout do not depend on it, config() carries it only when it is set (UViT, whose
reference declares it, always carries it), and a logged config with use_remat: true rebuilds a model with the flag."""
import json

import numpy as np
import pytest
import torch

from flaxdiff_b200 import checkpoint as ckpt_io
from flaxdiff_b200.inference import parse_config
from flaxdiff_b200.inputs import DiffusionInputConfig
from flaxdiff_b200.models.mmdit import HierarchicalMMDiT, SimpleMMDiT
from flaxdiff_b200.models.params import FlatParams, from_tree, nest
from flaxdiff_b200.models.simple_dit import SimpleDiT
from flaxdiff_b200.models.ssm_dit import HybridSSMAttentionDiT
from flaxdiff_b200.models.udit import SimpleUDiT
from flaxdiff_b200.models.uvit import UViT

CASES = {
    "simple_dit": (SimpleDiT, dict(patch_size=2, emb_features=128, num_layers=3, num_heads=2, learn_sigma=True,
                                   context_dim=64)),
    "hybrid_dit": (HybridSSMAttentionDiT, dict(patch_size=2, emb_features=128, num_layers=4, num_heads=2,
                                               ssm_state_dim=32, use_hilbert=True)),
    "simple_mmdit": (SimpleMMDiT, dict(patch_size=2, emb_features=128, num_layers=2, num_heads=2, context_dim=64)),
    "hierarchical_mmdit": (HierarchicalMMDiT, dict(base_patch_size=2, emb_features=(64, 128), num_layers=(2, 1),
                                                   num_heads=(2, 2), context_dim=64)),
    "simple_udit": (SimpleUDiT, dict(patch_size=2, emb_features=128, num_layers=4, num_heads=2, context_dim=64)),
    "uvit": (UViT, dict(patch_size=2, emb_features=128, num_layers=4, num_heads=2, add_residualblock_output=True)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_every_class_takes_the_flag_and_keeps_its_parameters(case):
    cls, kw = CASES[case]
    off, on = cls(**kw), cls(**kw, use_remat=True)
    assert off.use_remat is False and on.use_remat is True
    assert on.param_specs() == off.param_specs()
    assert on.layout().table == off.layout().table and on.layout().total == off.layout().total


@pytest.mark.parametrize("case", sorted(CASES))
def test_config_carries_the_flag_only_when_set(case):
    cls, kw = CASES[case]
    off, on = cls(**kw), cls(**kw, use_remat=True)
    if cls is UViT:                         # the reference's UViT declares use_remat: always in its config
        assert off.config()["use_remat"] is False
    else:
        assert "use_remat" not in off.config()
        assert off.config() == cls(**kw, use_remat=False).config()
    cfg = on.config()
    assert cfg["use_remat"] is True
    assert {k: v for k, v in cfg.items() if k != "use_remat"} == {k: v for k, v in off.config().items()
                                                                  if k != "use_remat"}
    assert cls(**cfg).use_remat is True and cls(**off.config()).use_remat is False


@pytest.mark.parametrize("architecture", ["uvit", "simple_dit"])
def test_parse_config_rebuilds_a_logged_flag(architecture):
    cls, kw = CASES[architecture]
    model = cls(**kw, use_remat=True)
    logged = json.loads(json.dumps(model.config()))
    assert logged["use_remat"] is True
    ic = DiffusionInputConfig("image", (16, 16, 3), [])
    out = parse_config({"model": logged, "architecture": architecture, "input_config": ic.serialize(),
                        "arguments": {}})
    assert type(out["model"]) is cls and out["model"].use_remat is True
    assert out["model"].config() == model.config()


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("write_on", [False, True])
def test_checkpoint_written_with_either_setting_loads_with_the_other(case, write_on, tmp_path):
    cls, kw = CASES[case]
    writer, reader = cls(**kw, use_remat=write_on), cls(**kw, use_remat=not write_on)
    g = torch.Generator().manual_seed(3)
    fp = FlatParams(writer.layout(), torch.randn(writer.layout().total, generator=g))
    ckpt_io.save_tree(str(tmp_path), 5, {"params": nest({k: v.numpy() for k, v in fp.named.items()})})
    _, back = ckpt_io.load_tree(str(tmp_path))
    got = from_tree(reader.layout(), back["params"], "cpu")
    assert all(np.array_equal(got.named[k].numpy(), fp.named[k].numpy()) for k in fp.named)
