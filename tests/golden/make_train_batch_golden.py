"""Generates tests/golden/train_batch_golden.pt by running the REFERENCE'S OWN training-step code.

    python tests/golden/make_train_batch_golden.py <reference checkout>      (pixeli99/SVD_Xtend)

From <reference checkout>/train_svd.py it takes, with `ast`, the module-level `rand_log_normal` and `tensor_to_vae_latent`, the
nested `_get_add_time_ids` of `main`, and the body of `with accelerator.accumulate(unet):` from its first statement through
`loss = loss.mean()`, and executes them unmodified (no source text is copied into this repository) in fp64 on the CPU with
deterministic stand-ins for `vae` (a pooled linear map to the moments, with one logvar channel below and one above the clamp),
`encode_image`, `unet` (its prediction is a leaf tensor, so `loss.backward()` yields d loss / d model_pred) and `accelerator`.
torch.rand / randn / randn_like are intercepted: every draw comes, in fp32, from one CPU generator seeded per case and is
recorded in order, under the names of svd_xtend_b200.video_train.draw_train_noise. A case may replace a draw's value (the
conditioning-dropout uniform of the region and boundary cases); the replaced names are recorded.
"""
import ast
import hashlib
import os
import sys
from types import SimpleNamespace

import torch
import torch.nn.functional as TF

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

NAMES = ("latent_eps", "noise", "cond_u", "cond_pixel_eps", "cond_latent_eps", "sigma_u", "dropout_u")
SF = 0.18215
D = 16          # image embedding width of the stand-ins
P = 0.1
f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))      # noqa: E731
# (name, B, F, H, W, conditioning_dropout_prob, seed, replaced draws)
CASES = [
    ("drop_prompt", 1, 3, 16, 24, P, 11, {"dropout_u": 0.05}),
    ("drop_both", 1, 3, 16, 24, P, 12, {"dropout_u": 0.15}),
    ("drop_image", 1, 3, 16, 24, P, 13, {"dropout_u": 0.25}),
    ("drop_none", 1, 3, 16, 24, P, 14, {"dropout_u": 0.5}),
    ("at_p", 1, 3, 16, 24, P, 15, {"dropout_u": f32(P)}),
    ("at_2p", 1, 3, 16, 24, P, 16, {"dropout_u": f32(2 * P)}),
    ("at_3p", 1, 3, 16, 24, P, 17, {"dropout_u": f32(3 * P)}),
    ("no_dropout", 1, 3, 16, 24, None, 18, {}),
    ("natural", 1, 3, 16, 24, P, 19, {}),
    ("batch2", 2, 3, 16, 24, P, 20, {}),
]


def extract(ref_file):
    """(module-level functions, _get_add_time_ids, the step body) of train_svd.py as compiled code objects"""
    tree = ast.parse(open(ref_file).read(), filename=ref_file)
    funcs = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("rand_log_normal", "tensor_to_vae_latent")]
    main = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "main")
    time_ids = next(n for n in ast.walk(main) if isinstance(n, ast.FunctionDef) and n.name == "_get_add_time_ids")
    with_node = next(n for n in ast.walk(main) if isinstance(n, ast.With) and ast.unparse(n.items[0].context_expr) == "accelerator.accumulate(unet)")
    body = []
    for st in with_node.body:
        body.append(st)
        if ast.unparse(st).replace(" ", "") == "loss=loss.mean()":
            break
    else:
        raise RuntimeError("`loss = loss.mean()` not found in the step body")
    comp = lambda nodes: compile(ast.fix_missing_locations(ast.Module(body=nodes, type_ignores=[])), ref_file, "exec")   # noqa: E731
    assert len(funcs) == 2
    return comp(funcs), comp([time_ids]), comp(body)


class Draws:
    """intercepts torch.rand / randn / randn_like: fp32 draws from one CPU generator, in order, under NAMES"""

    def __init__(self, seed, dropout, replace):
        self.g = torch.Generator().manual_seed(seed)
        self.names = [n for n in NAMES if dropout or n != "dropout_u"]
        self.replace = replace
        self.log = []
        self.orig = (torch.rand, torch.randn, torch.randn_like)

    def _draw(self, fn, shape, dtype):
        name = self.names[len(self.log)]
        v = fn(tuple(shape), generator=self.g, dtype=torch.float32)
        if name in self.replace:
            v = torch.full_like(v, self.replace[name])
        self.log.append((name, tuple(v.shape), v.clone()))
        return v.to(dtype or torch.float32)         # the script's default dtype is fp32

    def __enter__(self):
        rand, randn, _ = self.orig

        def shape_of(a):
            return a[0] if len(a) == 1 and isinstance(a[0], (list, tuple, torch.Size)) else (a[0],) if len(a) == 1 else a

        torch.rand = lambda *a, dtype=None, **kw: self._draw(rand, shape_of(a), dtype)
        torch.randn = lambda *a, dtype=None, **kw: self._draw(randn, shape_of(a), dtype)
        torch.randn_like = lambda t, **kw: self._draw(randn, t.shape, t.dtype)
        return self

    def __exit__(self, *exc):
        torch.rand, torch.randn, torch.randn_like = self.orig


class Dist:
    def __init__(self, moments):
        self.mean, self.logvar = torch.chunk(moments, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self):
        return self.mean + self.std * torch.randn(self.mean.shape, dtype=self.mean.dtype)


class StandInVae:
    """moments = A @ avgpool8(frames) + bias; logvar channel 6 sits above the clamp, channel 7 below it"""
    A = torch.tensor([[1, 0.5, -0.25], [-0.5, 1, 0.25], [0.25, -0.5, 1], [0.5, 0.5, 0.5],
                      [0.5, -0.25, 0.125], [-0.25, 0.5, 0.25], [0.125, 0.25, -0.5], [0.5, 0.25, 0.125]], dtype=torch.float64)
    bias = torch.tensor([0.1, -0.2, 0.3, 0.0, -1.0, -0.5, 25.0, -35.0], dtype=torch.float64)

    def __init__(self):
        self.config = SimpleNamespace(scaling_factor=SF)
        self.inputs, self.moments = [], []

    def encode(self, t):
        pooled = TF.avg_pool2d(t.double(), 8)
        m = torch.einsum("kc,nchw->nkhw", self.A, pooled) + self.bias.view(1, -1, 1, 1)
        self.inputs.append(t.clone())
        self.moments.append(m.clone())
        return SimpleNamespace(latent_dist=Dist(m))


def stand_in_encode_image(records):
    M = torch.linspace(-1, 1, 3 * D, dtype=torch.float64).reshape(3, D)

    def encode_image(pixel_values):
        e = pixel_values.double().mean(dim=(2, 3)) @ M + 0.01
        records.append(e.clone())
        return e
    return encode_image


class StandInUnet:
    def __init__(self):
        self.config = SimpleNamespace(addition_time_embed_dim=32)
        self.add_embedding = SimpleNamespace(linear_1=SimpleNamespace(in_features=96))
        self.calls = []

    def __call__(self, sample, timestep, encoder_hidden_states, added_time_ids):
        B = sample.shape[0]
        pred = (0.5 * sample[:, :, :4] - 0.25 * sample[:, :, 4:] + 0.01 * timestep.double().reshape(B, 1, 1, 1, 1)
                + 0.001 * encoder_hidden_states.reshape(B, -1).sum(1).reshape(B, 1, 1, 1, 1)).detach().requires_grad_(True)
        self.calls.append(dict(sample=sample.clone(), timestep=timestep.clone(), encoder_hidden_states=encoder_hidden_states.clone(),
                               added_time_ids=added_time_ids.clone(), model_pred=pred))
        return SimpleNamespace(sample=pred)


def pixels(B, F, H, W, seed):
    g = torch.Generator().manual_seed(seed + 1000)
    return torch.randint(-256, 257, (B, F, 3, H, W), generator=g).double() / 256       # exact in fp32 and bf16


def run_case(code, name, B, F, H, W, p, seed, replace):
    funcs, time_ids, body = code
    from einops import rearrange
    vae, unet, embeds = StandInVae(), StandInUnet(), []
    ns = dict(torch=torch, rearrange=rearrange)
    exec(funcs, ns)
    ns.update(unet=unet)
    exec(time_ids, ns)
    px = pixels(B, F, H, W, seed)
    ns.update(vae=vae, encode_image=stand_in_encode_image(embeds), accelerator=SimpleNamespace(device=torch.device("cpu")),
              batch={"pixel_values": px}, weight_dtype=torch.float64, args=SimpleNamespace(conditioning_dropout_prob=p),
              generator=None)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)          # the step's own tensors (timesteps) in fp64
    try:
        with Draws(seed, p is not None, replace) as d:
            exec(body, ns)
    finally:
        torch.set_default_dtype(prev)
    loss = ns["loss"]
    call = unet.calls[-1]
    loss.backward()
    assert len(vae.inputs) == 2 and len(embeds) == 1 and len(unet.calls) == 1
    return dict(name=name, B=B, F=F, H=H, W=W, p=p, seed=seed, replaced=sorted(replace), pixel_values=px, draws=d.log,
                clip_frames=vae.inputs[0], cond_frames=vae.inputs[1], clip_moments=vae.moments[0], cond_moments=vae.moments[1],
                image_embeds=embeds[0], sample=call["sample"], timestep=call["timestep"],
                encoder_hidden_states=call["encoder_hidden_states"], added_time_ids=call["added_time_ids"],
                model_pred=call["model_pred"].detach(), latents=ns["latents"].detach(), noisy=ns["noisy_latents"].detach(),
                sigmas=ns["sigmas"].detach(), loss=loss.detach(), dloss_dpred=call["model_pred"].grad.clone())


def main():
    ref_file = os.path.join(sys.argv[1], "train_svd.py")
    code = extract(ref_file)
    fixture = {"reference_file_sha256": hashlib.sha256(open(ref_file, "rb").read()).hexdigest(), "scaling_factor": SF,
               "cases": [run_case(code, *c) for c in CASES]}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "train_batch_golden.pt")
    torch.save(fixture, path)
    print("wrote", path, [(c["name"], float(c["loss"])) for c in fixture["cases"]])


if __name__ == "__main__":
    main()
