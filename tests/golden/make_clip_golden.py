"""Writes tests/golden/clip_golden.pt — run where transformers and a reference checkout are available:

    python tests/golden/make_clip_golden.py /path/to/SVD_Xtend

* transformers' CLIPVisionModelWithProjection at the tiny config (head dim 80), once with hidden_act "gelu" and once with
  "quick_gelu", in fp64 with parameters drawn from integers (oracle.svd_clip_oracle.integer_init_) on integer-grid inputs:
  image_embeds and every 8th token of last_hidden_state.
* the reference's own `_resize_with_antialiasing` (read out of its train_svd.py at generation time; nothing of it is stored)
  on seeded fp64 inputs: a downscale 320x512 -> 224, an upscale 100x150 -> 224 and an odd size 291x397 -> 224, as 4096
  sampled output values plus the fp64 sum and sum of squares of the whole output.
Everything the checks need besides these outputs (parameters, inputs) is regenerated from the seeds stored here.
"""
import ast
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.svd_clip_oracle import TINY_CLIP_CONFIG, CLIPVisionModelWithProjection, integer_init_, integer_pixels  # noqa: E402

RESIZE_CASES = ((320, 512, 11), (100, 150, 12), (291, 397, 13))
CLIP_SEEDS = dict(gelu=(101, 201), quick_gelu=(102, 202))        # (parameter seed, input seed)
SAMPLES = 4096


def reference_resize(reference_root):
    """`_resize_with_antialiasing` and its helpers, executed from the reference's train_svd.py source"""
    path = os.path.join(reference_root, "train_svd.py")
    tree = ast.parse(open(path).read())
    names = {"_resize_with_antialiasing", "_compute_padding", "_filter2d", "_gaussian", "_gaussian_blur2d"}
    mod = ast.Module(body=[n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names], type_ignores=[])
    ns = {"torch": torch}
    exec(compile(mod, path, "exec"), ns)
    return ns["_resize_with_antialiasing"]


def main(reference_root):
    from transformers import CLIPVisionConfig
    from transformers import CLIPVisionModelWithProjection as HF
    out = dict(clip={}, resize={})
    for act, (pseed, xseed) in CLIP_SEEDS.items():
        cfg = dict(TINY_CLIP_CONFIG, hidden_act=act)
        ours = integer_init_(CLIPVisionModelWithProjection(**cfg).double(), pseed)
        hf = HF(CLIPVisionConfig(**cfg)).double().eval()
        hf.load_state_dict(ours.state_dict(), strict=True)
        x = integer_pixels((2, 3, 224, 224), xseed)
        with torch.no_grad():
            r = hf(pixel_values=x)
        out["clip"][act] = dict(config=cfg, param_seed=pseed, input_seed=xseed, image_embeds=r.image_embeds.clone(),
                                last_hidden_state_every8=r.last_hidden_state[:, ::8].clone())
    resize = reference_resize(reference_root)
    for h, w, seed in RESIZE_CASES:
        x = integer_pixels((1, 3, h, w), seed)
        y = resize(x, (224, 224))
        idx = torch.randperm(y.numel(), generator=torch.Generator().manual_seed(seed))[:SAMPLES]
        out["resize"][(h, w)] = dict(seed=seed, index=idx.to(torch.int32), values=y.flatten()[idx].clone(),
                                     sum=y.sum().item(), sumsq=(y * y).sum().item())
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "clip_golden.pt")
    torch.save(out, dst)
    print(dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit("usage: python tests/golden/make_clip_golden.py <reference checkout>")
    main(sys.argv[1])
