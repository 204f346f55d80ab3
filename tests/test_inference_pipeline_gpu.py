"""From a trained run to images: DiffusionInferencePipeline.from_checkpoint on a checkpoint written by
GeneralDiffusionTrainer.save and a hand-written run config, against a direct sampler call on the same parameter tree
with the same key, bit for bit; and raw prompts through DiffusionSampler.generate_samples against their embeddings.

The images are 8 x 8: there no launch of these models accumulates with atomics, so two runs of one computation are
bit-identical and any difference is a difference in what the pipeline computes."""
import json

import numpy as np
import pytest
import torch

from clip_text_ref import Tok, clip_model, token_batch
from flaxdiff_b200 import checkpoint as ckpt_io
from flaxdiff_b200 import utils
from flaxdiff_b200.inference import DiffusionInferencePipeline
from flaxdiff_b200.inputs import CLIPTextEncoder, ConditionalInputConfig, DiffusionInputConfig
from flaxdiff_b200.models.mmdit import SimpleMMDiT
from flaxdiff_b200.models.simple_unet import Unet
from flaxdiff_b200.models.ssm_dit import HybridSSMAttentionDiT
from flaxdiff_b200.predictors import KarrasPredictionTransform
from flaxdiff_b200.samplers import DDIMSampler, EulerAncestralSampler, HeunSampler
from flaxdiff_b200.schedulers import EDMNoiseScheduler, KarrasVENoiseScheduler
from flaxdiff_b200.trainer import GeneralDiffusionTrainer, adamw
from flaxdiff_b200.utils import RandomMarkovState

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
RES = 8
PROMPTS = ["a red fox in snow", "a lighthouse at dusk", ""]


def _text_input_config():
    enc = CLIPTextEncoder(clip_model("tiny"), Tok(1000), modelname="tiny-random", backend="fdx")
    cond = ConditionalInputConfig(encoder=enc, conditioning_data_key="text", pretokenized=True,
                                  unconditional_input="", model_key_override="textcontext")
    return DiffusionInputConfig("image", (RES, RES, 3), [cond])


def _train_and_save(model, input_config, tmp_path, steps=3):
    """A few training steps, then trainer.save: -> (checkpoint directory, the tree it holds)."""
    tr = GeneralDiffusionTrainer(model, adamw(1e-3), EDMNoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                                 input_config, rngs=4, unconditional_prob=0.25,
                                 model_output_transform=KarrasPredictionTransform(0.5), device=dev,
                                 checkpoint_base_path=str(tmp_path))
    step = tr._define_train_step()
    rng = np.random.default_rng(0)
    for i in range(steps):
        batch = {"image": torch.from_numpy(rng.integers(0, 256, (4, RES, RES, 3), dtype=np.uint8))}
        if input_config.conditions:
            ids, mask = token_batch(1000, [3, 10, 0, 20], seed=i)
            batch["text"] = {"input_ids": ids, "attention_mask": mask}
        tr.state, _, tr.rngstate = step(tr.state, tr.rngstate, batch)
    tr.save(0, steps)
    _, tree = ckpt_io.load_tree(tr.checkpoint_path())
    return tr.checkpoint_path(), tree


def _run_config(architecture, model_kwargs, input_config):
    """training.py's CONFIG shape, as a wandb run would log it."""
    return json.loads(json.dumps({"model": model_kwargs, "architecture": architecture, "noise_schedule": "edm",
                                  "input_config": input_config.serialize(), "arguments": {"image_size": RES},
                                  "autoencoder": None, "autoencoder_opts": "{}"}))


def _direct(model, input_config, tree, sampler_class, guidance_scale, embeddings, steps):
    smp = sampler_class(model, KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                        KarrasPredictionTransform(0.5), input_config, guidance_scale=guidance_scale)
    return smp.generate_samples(tree, num_samples=len(PROMPTS), resolution=RES, diffusion_steps=steps,
                                start_step=1000, rngstate=RandomMarkovState(utils.PRNGKey(42)),
                                model_conditioning_inputs=embeddings)


def test_text_conditioned_unet_from_checkpoint_matches_direct_sampling(tmp_path):
    ic = _text_input_config()
    kwargs = {"attention_configs": [None, None, {"heads": 4}, {"heads": 8}], "dtype": "bfloat16",
              "activation": "swish"}
    model = Unet(attention_configs=(None, None, {"heads": 4}, {"heads": 8}), dtype=torch.bfloat16)
    ckdir, tree = _train_and_save(model, ic, tmp_path)
    cfg_path = tmp_path / "config.json"
    cfg_path.write_text(json.dumps(_run_config("unet", kwargs, ic)))
    # the serialised input config names "tiny-random", which no local cache holds: hand over the trainer's
    pipe = DiffusionInferencePipeline.from_checkpoint(ckdir, str(cfg_path), input_config=ic)
    assert pipe.model.context_dim == 64 and pipe.input_config is ic
    assert pipe._packed == {}                      # the trees stay on the host until a call samples from them
    emb = (ic.conditions[0].encoder(PROMPTS),)
    steps = 8
    outs = {}
    for sampler_class, ema, best in ((EulerAncestralSampler, True, False), (EulerAncestralSampler, False, True),
                                     (EulerAncestralSampler, False, False), (DDIMSampler, True, False),
                                     (HeunSampler, True, False)):
        got = pipe.generate_samples(num_samples=len(PROMPTS), resolution=RES, conditioning_data=PROMPTS,
                                    diffusion_steps=steps, start_step=1000, guidance_scale=3.0,
                                    sampler_class=sampler_class, use_ema=ema, use_best_params=best)
        st = tree["best_state" if best else "state"]
        want = _direct(model, ic, st["ema_params" if ema else "params"], sampler_class, 3.0, emb, steps)
        assert got.shape == (len(PROMPTS), RES, RES, 3) and torch.isfinite(got).all()
        assert torch.equal(got, want), (sampler_class.__name__, ema, best)
        outs[(sampler_class, ema, best)] = got
    # each tree a call used was packed once: EMA and params of `state`, params of `best_state`
    assert len(pipe._packed) == 3
    # the three parameter trees are different, and so are their images
    a, b, c = (outs[(EulerAncestralSampler, e, bst)] for e, bst in ((True, False), (False, True), (False, False)))
    assert not torch.equal(a, b) and not torch.equal(a, c) and not torch.equal(b, c)
    # a second call reuses the cached sampler and its graphs, and returns the same images (the reference's key)
    smp = pipe.get_sampler(3.0, EulerAncestralSampler)
    graphs = dict(smp._graphs)
    again = pipe.generate_samples(num_samples=len(PROMPTS), resolution=RES, conditioning_data=PROMPTS,
                                  diffusion_steps=steps, start_step=1000, guidance_scale=3.0, use_ema=True)
    assert torch.equal(again, a) and dict(smp._graphs) == graphs


def test_simple_mmdit_from_checkpoint_matches_direct_sampling(tmp_path):
    ic = _text_input_config()
    kwargs = {"patch_size": 2, "emb_features": 128, "num_layers": 2, "num_heads": 2, "dtype": "bfloat16"}
    model = SimpleMMDiT(patch_size=2, emb_features=128, num_layers=2, num_heads=2, dtype=torch.bfloat16)
    ckdir, tree = _train_and_save(model, ic, tmp_path)
    pipe = DiffusionInferencePipeline.from_checkpoint(ckdir, _run_config("simple_mmdit", kwargs, ic), input_config=ic)
    assert pipe.model.config() == model.config()
    emb = (ic.conditions[0].encoder(PROMPTS),)
    got = pipe.generate_samples(num_samples=len(PROMPTS), resolution=RES, conditioning_data=PROMPTS,
                                diffusion_steps=6, start_step=1000, guidance_scale=3.0, use_ema=True)
    want = _direct(model, ic, tree["state"]["ema_params"], EulerAncestralSampler, 3.0, emb, 6)
    assert torch.isfinite(got).all() and torch.equal(got, want)


def test_unconditioned_hybrid_zigzag_from_checkpoint_matches_direct_sampling(tmp_path):
    ic = DiffusionInputConfig("image", (RES, RES, 3), [])
    kwargs = {"patch_size": 2, "emb_features": 128, "num_layers": 4, "num_heads": 2, "ssm_state_dim": 16,
              "use_zigzag": True, "ssm_attention_ratio": "1:1", "dtype": "bfloat16"}
    model = HybridSSMAttentionDiT(patch_size=2, emb_features=128, num_layers=4, num_heads=2, ssm_state_dim=16,
                                  use_zigzag=True, ssm_attention_ratio="1:1", dtype=torch.bfloat16)
    ckdir, tree = _train_and_save(model, ic, tmp_path)
    # the unconditioned input config is rebuilt from the run config itself
    pipe = DiffusionInferencePipeline.from_checkpoint(ckdir, _run_config("hybrid_dit+zigzag", kwargs, ic))
    assert pipe.model.config() == model.config() and pipe.input_config.conditions == []
    for ema in (True, False):
        got = pipe.generate_samples(num_samples=len(PROMPTS), resolution=RES, diffusion_steps=6, start_step=1000,
                                    guidance_scale=0.0, use_ema=ema)
        want = _direct(model, ic, tree["state"]["ema_params" if ema else "params"], EulerAncestralSampler, 0.0,
                       None, 6)
        assert torch.isfinite(got).all() and torch.equal(got, want), ema


@pytest.mark.parametrize("sampler_class", [EulerAncestralSampler, HeunSampler])
def test_raw_prompts_through_the_sampler_match_their_embeddings(sampler_class):
    """With a utils.jax_key state EulerAncestral takes the whole-step graph, as Heun always does: the prompts'
    embeddings reach the captured step exactly as model_conditioning_inputs do."""
    ic = _text_input_config()
    model = Unet(attention_configs=(None, None, None, {"heads": 8}), dtype=torch.bfloat16)
    fp = model.init(3, textcontext=ic.conditions[0].get_unconditional(), device=dev)
    outs = []
    for kw in ({"conditioning": PROMPTS}, {"model_conditioning_inputs": (ic.conditions[0].encoder(PROMPTS),)}):
        smp = sampler_class(model, KarrasVENoiseScheduler(1, sigma_max=80, rho=7, sigma_data=0.5),
                            KarrasPredictionTransform(0.5), ic, guidance_scale=2.0)
        outs.append(smp.generate_samples(fp, len(PROMPTS), RES, diffusion_steps=6, start_step=1000,
                                         rngstate=RandomMarkovState(utils.jax_key(7)), **kw))
        assert any(k[0] == "step" for k in smp._graphs)           # the whole-step graph ran
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])
