"""Generates tests/golden/ref_wiring_tiny.pt by running the REFERENCE'S OWN top-level file.

    python tests/golden/make_ref_wiring_golden.py <reference checkout>      (pixeli99/SVD_Xtend)

<reference checkout>/src/unet_spatio_temporal_condition.py is imported unmodified from where it lies (oracle/ref_wiring.py
provides a stand-in for the absent `diffusers` package whose block classes are the oracle's), instantiated with the
small test topology and run in fp64 on a batch of TWO clips. The fixture freezes what the reference's file itself
decides: state-dict names and shapes, channel bookkeeping of the down / mid / up blocks, the order of embedding
repeats and skip connections in forward(), the attention-processor key set, a train-mode forward + backward of the
as-scripted trainable set, and what the file's plugin API does — so the oracle's top-level restatement
(and through it the CUDA path) is pinned to reference code, not to a recollection of it. The block arithmetic is the
oracle's on both sides and stays unpinned against diffusers (see the header of oracle/svd_unet_oracle.py).
"""
import contextlib
import hashlib
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import svd_unet_oracle  # noqa: E402
from oracle.ref_wiring import load_reference_unet_class  # noqa: E402
from oracle.svd_unet_oracle import SVD_CONFIG, TINY_CONFIG, synthetic_batch  # noqa: E402

SEED = 20260923


# The fixture is compared at fp64 round-off (1e-12), so nothing the comparison consumes may depend on the CPU it runs on.
# torch's fp32 random transforms (randn, the uniform_ of default init) and fp32 exp / sin / cos differ in the last bit
# between vector code paths, and one fp32 ulp moves this model's fp64 output by up to 1e-8. Hence: parameters from integer
# draws scaled by single correctly rounded operations, the input batch stored in the fixture, and the fp32 timestep
# embeddings (the reference computes them in fp32) recorded on the reference side and replayed on the oracle side.
def build(cls):
    m = cls(**TINY_CONFIG).double()
    with torch.no_grad():
        g = torch.Generator().manual_seed(SEED + 1)
        for n, p in m.named_parameters():
            u = torch.randint(-2 ** 20, 2 ** 20 + 1, p.shape, generator=g, dtype=torch.int64).double() / 2 ** 20   # exact, [-1, 1]
            if n.endswith("mix_factor"):
                p.copy_(0.5 + 0.1 * u)
            elif "norm" in n and n.endswith("weight"):
                p.copy_(1.0 + 0.1 * u)          # de-symmetrised affine terms, so that every affine / blend path matters
            elif "norm" in n or n.endswith("bias") or p.dim() < 2:
                p.copy_(0.1 * u)
            else:
                p.copy_(u / math.sqrt(p[0].numel()))   # the bound of the default (kaiming-uniform) init
    return m.eval()


def batch():
    """the input batch the fixture was made with is stored in it (`tiny_batch`): use that one for comparisons"""
    b = synthetic_batch(2, 4, 16, 16, seed=4321, cross_dim=TINY_CONFIG["cross_attention_dim"], dtype=torch.float64)
    return {k: b[k] for k in ("sample", "timestep", "encoder_hidden_states", "added_time_ids")}


@contextlib.contextmanager
def timestep_embeddings(table, record):
    """record=True: store every fp32 timestep embedding computed inside the block in `table`; record=False: return the stored
    one instead, after checking that the freshly computed value agrees with it to fp32 accuracy"""
    orig = svd_unet_oracle.get_timestep_embedding

    def emb(timesteps, embedding_dim, *args, **kw):
        fresh = orig(timesteps, embedding_dim, *args, **kw)
        key = (embedding_dim, tuple(timesteps.double().tolist()), args, tuple(sorted(kw.items())))
        if record:
            table[key] = fresh.clone()
            return fresh
        stored = table[key]
        assert (fresh - stored).abs().max().item() <= 1e-6 * max(1.0, stored.abs().max().item()), key
        return stored.clone()

    svd_unet_oracle.get_timestep_embedding = emb
    try:
        yield table
    finally:
        svd_unet_oracle.get_timestep_embedding = orig


def forward(m, b):
    return m(b["sample"], b["timestep"].double(), b["encoder_hidden_states"], b["added_time_ids"])


def train_step(m, b):
    """train-mode forward + backward of the as-scripted trainable set (train_svd.py:761-766): output and gradients"""
    m.train()
    m.requires_grad_(False)
    for n, p in m.named_parameters():
        if "temporal_transformer_block" in n:
            p.requires_grad_(True)
    out = forward(m, b).sample
    out.square().mean().backward()
    return out.detach(), {n: p.grad.clone() for n, p in m.named_parameters() if p.requires_grad}


GRAD_SAMPLE = 64


def grad_digest(grads):
    """per gradient: its norm and a fixed seeded sample of GRAD_SAMPLE entries (flat index, value); keeps the fixture small"""
    g = torch.Generator().manual_seed(SEED + 2)
    out = {}
    for n, t in grads.items():
        flat = t.reshape(-1)
        idx = torch.randperm(flat.numel(), generator=g)[:GRAD_SAMPLE].clone()
        out[n] = (float(flat.norm()), idx, flat[idx].clone())
    return out


def main():
    ref_root = sys.argv[1]
    ref_file = os.path.join(ref_root, "src", "unet_spatio_temporal_condition.py")
    Ref = load_reference_unet_class(ref_root)
    ref = build(Ref)
    b = batch()
    embeddings = {}
    with torch.no_grad(), timestep_embeddings(embeddings, record=True):
        out = forward(ref, b).sample
        out_t = ref(b["sample"], b["timestep"].double(), b["encoder_hidden_states"], b["added_time_ids"], return_dict=False)[0]
    assert torch.equal(out, out_t)
    with torch.device("meta"):
        big = Ref(**SVD_CONFIG)
    big_keys = [(k, tuple(v.shape)) for k, v in big.state_dict().items()]
    fixture = {
        "seed": SEED,
        "reference_file_sha256": hashlib.sha256(open(ref_file, "rb").read()).hexdigest(),
        "tiny_keys": [(k, tuple(v.shape)) for k, v in ref.state_dict().items()],
        "tiny_param_checksum": float(sum(p.detach().double().abs().sum() for p in ref.parameters())),
        "tiny_batch": b,
        "tiny_out": out.clone(),
        "tiny_attn_processor_keys": sorted(ref.attn_processors.keys()),
        "svd_keys_sha256": hashlib.sha256(repr(big_keys).encode()).hexdigest(),
        "svd_num_keys": len(big_keys),
        "svd_total_params": sum(v.numel() for v in big.state_dict().values()),
        "svd_temporal_params": sum(p.numel() for n, p in big.named_parameters() if "temporal_transformer_block" in n),
        "svd_num_upsamplers": big.num_upsamplers,
        "svd_attn_processors": len(big.attn_processors),
    }
    train_ref = build(Ref)
    with timestep_embeddings(embeddings, record=True):
        t_out, t_grads = train_step(train_ref, b)
    fixture["tiny_timestep_embeddings"] = embeddings
    fixture["tiny_train_out"] = t_out
    fixture["tiny_train_grads"] = grad_digest(t_grads)
    train_ref.set_default_attn_processor()
    fixture["default_processor_types"] = sorted({type(p).__name__ for p in train_ref.attn_processors.values()})
    try:
        train_ref.set_attn_processor({})
        fixture["empty_processor_dict_raises"] = None
    except Exception as e:      # noqa: BLE001
        fixture["empty_processor_dict_raises"] = type(e).__name__
    train_ref.enable_gradient_checkpointing()
    fixture["gradient_checkpointing_modules"] = sum(bool(getattr(m, "gradient_checkpointing", False)) for m in train_ref.modules())
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_wiring_tiny.pt")
    torch.save(fixture, path)
    print("wrote", path, "out std", float(out.std()), "svd params", fixture["svd_total_params"], fixture["svd_temporal_params"],
          "processors", fixture["svd_attn_processors"])


if __name__ == "__main__":
    main()
