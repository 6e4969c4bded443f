"""The oracle's (and the product class's) top-level wiring against the REFERENCE'S OWN file.

tests/golden/ref_wiring_tiny.pt was produced by importing the reference's src/unet_spatio_temporal_condition.py unmodified
(tests/golden/make_ref_wiring_golden.py, through oracle/ref_wiring.py) and running it in fp64 on two clips. These CPU tests
need only the committed fixture.
What is pinned: construction (:71-246), forward wiring (:357-490), a train-mode backward, plugin-API key set and behaviour
(:248-274), parameter census of the SVD configuration. The arithmetic inside the blocks is the oracle's on both sides (unpinned against diffusers)."""
import hashlib
import importlib.util
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_wiring_tiny.pt")


def _gen():
    spec = importlib.util.spec_from_file_location("make_ref_wiring_golden", os.path.join(ROOT, "tests", "golden", "make_ref_wiring_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLDEN, weights_only=False)


def test_oracle_forward_equals_reference_file_golden(gold):
    from oracle.svd_unet_oracle import UNetSpatioTemporalConditionModel as Oracle
    gen = _gen()
    m = gen.build(Oracle)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == gold["tiny_keys"]
    chk = float(sum(p.detach().double().abs().sum() for p in m.parameters()))
    assert abs(chk - gold["tiny_param_checksum"]) < 1e-9 * gold["tiny_param_checksum"], "seeded init differs from the generator's"
    with torch.no_grad(), gen.timestep_embeddings(gold["tiny_timestep_embeddings"], record=False):
        out = gen.forward(m, gold["tiny_batch"]).sample
    assert out.shape == gold["tiny_out"].shape == (2, 4, 4, 16, 16)
    err = ((out - gold["tiny_out"]).norm() / gold["tiny_out"].norm()).item()
    assert err < 1e-12, err      # identical blocks, identical wiring: fp64 round-off only
    assert sorted(m_name + ".processor" for m_name, mod in m.named_modules() if hasattr(mod, "get_processor")) == gold["tiny_attn_processor_keys"]


def test_svd_configuration_census_equals_reference_file(gold):
    """names, shapes and counts the reference's constructor produces for the SVD configuration: oracle AND product class"""
    from oracle.svd_unet_oracle import SVD_CONFIG, UNetSpatioTemporalConditionModel as Oracle
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours
    assert gold["svd_total_params"] == 1_524_623_082 and gold["svd_temporal_params"] == 397_620_480
    for cls in (Oracle, Ours):
        with torch.device("meta"):
            m = cls(**SVD_CONFIG)
        keys = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
        assert len(keys) == gold["svd_num_keys"]
        assert hashlib.sha256(repr(keys).encode()).hexdigest() == gold["svd_keys_sha256"], cls
        assert m.num_upsamplers == gold["svd_num_upsamplers"]
    assert len(m.attn_processors) == gold["svd_attn_processors"] == 64


def test_product_class_plugin_keys_equal_reference_file(gold):
    from oracle.svd_unet_oracle import TINY_CONFIG
    from svd_xtend_b200.unet import UNetSpatioTemporalConditionModel as Ours
    m = Ours(**TINY_CONFIG)
    assert sorted(m.attn_processors.keys()) == gold["tiny_attn_processor_keys"]
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == gold["tiny_keys"]


def test_oracle_train_step_equals_reference_file_golden(gold):
    """train-mode forward + backward of the as-scripted trainable set, and the reference file's plugin API, against what the
    reference file itself computed and did when the fixture was generated"""
    from oracle.svd_unet_oracle import UNetSpatioTemporalConditionModel as Oracle
    gen = _gen()
    ora = gen.build(Oracle)
    with gen.timestep_embeddings(gold["tiny_timestep_embeddings"], record=False):
        out, grads = gen.train_step(ora, gold["tiny_batch"])
    assert ((out - gold["tiny_train_out"]).norm() / gold["tiny_train_out"].norm()).item() < 1e-12
    assert sorted(grads) == sorted(gold["tiny_train_grads"])
    for n, (norm, idx, vals) in gold["tiny_train_grads"].items():
        g = grads[n].reshape(-1)
        assert abs(float(g.norm()) - norm) <= 1e-12 * norm, n
        assert ((g[idx] - vals).abs().max() <= 1e-12 * norm).item(), n
    # the plugin API of the reference file on the oracle's Attention modules
    assert gold["default_processor_types"] == ["AttnProcessor"]
    assert gold["empty_processor_dict_raises"] == "ValueError"
    assert gold["gradient_checkpointing_modules"] == sum(1 for m in ora.modules() if hasattr(m, "gradient_checkpointing"))
