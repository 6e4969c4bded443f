"""LoRA adapters on disk, and their merge into the base weights.

The file is diffusers' LoRA layout for a UNet, as `StableVideoDiffusionPipeline.save_lora_weights` writes it at the end of
train_svd_lora.py (:1146-1153): one `pytorch_lora_weights.safetensors` (or `.bin` through torch.save) whose keys are
`unet.<linear>.lora.down.weight` [r, in] and `unet.<linear>.lora.up.weight` [out, r], with optional `unet.<linear>.alpha`.

  * save_lora_weights takes what the script passes: `convert_state_dict_to_diffusers(get_peft_model_state_dict(unet))`,
    i.e. PEFT names with the adapter name removed, in either spelling (`…lora_A.weight` / `…lora.down.weight`).
  * load_into (behind `unet.load_lora_adapter`; read_state_dict + parse) accepts that file, a directory holding it, or a state dict; keys with or without `unet.`, in either spelling.
    Rank comes from each module's shapes; `lora_alpha` from `<module>.alpha` when present, else r (the script's LoraConfig,
    train_svd_lora.py:659-664, has lora_alpha = rank). Malformed input, and factors for a linear without a LoRA side path
    on this build (anything but the attention projections), are rejected, naming the keys, before anything changes.
  * lora_adapter_state_dict: one adapter's factors under PEFT's names, what get_peft_model_state_dict returns, plus
    `<module>.alpha` where lora_alpha != r, so that a written adapter loads back with its own scaling.
  * merge_into_base: the fuse / unfuse arithmetic (oracle/svd_lora_oracle.py) over many layers in one svdx_lora_merge launch.
"""
from __future__ import annotations

import os
import struct
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import raw

SAFE_NAME = "pytorch_lora_weights.safetensors"
BIN_NAME = "pytorch_lora_weights.bin"
PREFIX = "unet."
# keys of the other components of a pipeline's LoRA file: a UNet cannot take them
_OTHER_COMPONENTS = ("text_encoder.", "text_encoder_2.", "vae.", "image_encoder.", "transformer.")
# suffix -> (role, canonical diffusers suffix)
_SUFFIXES = ((".lora.down.weight", "down"), (".lora.up.weight", "up"), (".lora_A.weight", "down"), (".lora_B.weight", "up"),
             (".alpha", "alpha"))
_DIFFUSERS = {"down": ".lora.down.weight", "up": ".lora.up.weight", "alpha": ".alpha"}


def _split(key: str) -> Tuple[Optional[str], Optional[str]]:
    """(module name, role) of a LoRA key without prefix, or (None, None)"""
    for suffix, role in _SUFFIXES:
        if key.endswith(suffix) and len(key) > len(suffix):
            return key[:-len(suffix)], role
    return None, None


# ----------------------------------------------------------------------------- writer
def save_lora_weights(save_directory: str, unet_lora_layers: Dict[str, torch.Tensor], weight_name: Optional[str] = None,
                      safe_serialization: bool = True, **kwargs) -> str:
    """write `unet_lora_layers` (PEFT names without the adapter name, `…lora_A.weight` or `…lora.down.weight`) as
    `<save_directory>/pytorch_lora_weights.safetensors`, or `.bin` through torch.save with safe_serialization=False, under
    diffusers' keys `unet.<module>.lora.down.weight` / `.lora.up.weight`. Returns the file's path."""
    if not unet_lora_layers:
        raise ValueError("save_lora_weights: no LoRA layers given (unet_lora_layers is empty)")
    out, bad = {}, []
    for k, v in unet_lora_layers.items():
        name = k[len(PREFIX):] if k.startswith(PREFIX) else k
        module, role = _split(name)
        if module is None or not torch.is_tensor(v):
            bad.append(k)
            continue
        out[PREFIX + module + _DIFFUSERS[role]] = v.detach().cpu().contiguous()
    if bad:
        raise ValueError(f"save_lora_weights: not LoRA factor keys of a UNet: {bad[:8]}")
    os.makedirs(save_directory, exist_ok=True)
    path = os.path.join(save_directory, weight_name or (SAFE_NAME if safe_serialization else BIN_NAME))
    if safe_serialization:
        from safetensors.torch import save_file
        save_file(out, path, metadata={"format": "pt"})
    else:
        torch.save(out, path)
    return path


# ----------------------------------------------------------------------------- reader
def read_state_dict(path_or_dict, weight_name: Optional[str] = None) -> Dict[str, torch.Tensor]:
    if isinstance(path_or_dict, dict):
        return dict(path_or_dict)
    path = os.fspath(path_or_dict)
    if os.path.isdir(path):
        names = [weight_name] if weight_name else [SAFE_NAME, BIN_NAME]
        found = [os.path.join(path, n) for n in names if os.path.isfile(os.path.join(path, n))]
        if not found:
            raise FileNotFoundError(f"no LoRA weights ({', '.join(names)}) under {path}")
        path = found[0]
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path)
    return torch.load(path, map_location="cpu", weights_only=True)


def parse(sd: Dict[str, torch.Tensor], linears: Dict[str, Tuple[int, int]], adaptable) -> Dict[str, dict]:
    """{module: {"down", "up", "alpha"}} of a LoRA state dict, checked against `linears` ({module name: (out, in)}) and
    `adaptable` (the names among them that take a LoRA side path). Every problem raises ValueError naming its keys."""
    mods: Dict[str, dict] = {}
    other, unknown = [], []
    for k, v in sd.items():
        if k.startswith(_OTHER_COMPONENTS):
            other.append(k)
            continue
        module, role = _split(k[len(PREFIX):] if k.startswith(PREFIX) else k)
        if module is None or not torch.is_tensor(v):
            unknown.append(k)
            continue
        ent = mods.setdefault(module, {})
        if role in ent:
            raise ValueError(f"LoRA file: module {module!r} has its {role} factor twice (both key spellings?): {k}")
        ent[role] = v
        ent.setdefault("keys", []).append(k)
    if other:
        raise ValueError(f"LoRA file: keys of another pipeline component, not the UNet: {other[:8]}")
    if unknown:
        raise ValueError(f"LoRA file: keys that are not LoRA factors (`.lora.down/up.weight`, `.lora_A/B.weight`, `.alpha`): {unknown[:8]}")
    if not mods:
        raise ValueError("LoRA file: no LoRA factors found")
    missing = [e["keys"] for m, e in mods.items() if m not in linears]
    if missing:
        raise ValueError(f"LoRA file: keys naming no nn.Linear of the UNet: {missing[:8]}")
    refused = [e["keys"] for m, e in mods.items() if m not in adaptable]
    if refused:
        raise ValueError("LoRA file: keys of linears without a LoRA side path on this build (only the attention projections "
                         f"to_q / to_k / to_v / to_out.0 take one; the others would be ignored unfused): {refused[:8]}")
    unpaired = [e["keys"] for e in mods.values() if "down" not in e or "up" not in e]
    if unpaired:
        raise ValueError(f"LoRA file: down / up factors without their pair: {unpaired[:8]}")
    misfit = []
    for m, e in mods.items():
        out_f, in_f = linears[m]
        d, u = e["down"], e["up"]
        if d.dim() != 2 or u.dim() != 2 or d.shape[0] < 1 or d.shape[0] != u.shape[1] or d.shape[1] != in_f or u.shape[0] != out_f:
            misfit.append((e["keys"], tuple(d.shape), tuple(u.shape), f"layer [{out_f}, {in_f}]"))
        elif "alpha" in e and e["alpha"].numel() != 1:
            misfit.append((e["keys"], "alpha must be one number"))
    if misfit:
        raise ValueError(f"LoRA file: factor shapes that do not fit their layer: {misfit[:8]}")
    return mods


def load_into(unet, path_or_dict, adapter_name: Optional[str] = None, weight_name: Optional[str] = None) -> str:
    """read a LoRA file into `unet` as a new adapter (next free `default_<i>` when unnamed), in the base weights' dtype and
    device, made the active adapter. The factors are loaded frozen (requires_grad False). Returns the adapter name."""
    sd = read_state_dict(path_or_dict, weight_name)
    slots = {full: (parent, attr, child) for full, parent, attr, child in unet._linear_slots()}
    mods = parse(sd, {full: (child.out_features, child.in_features) for full, (_, _, child) in slots.items()}, unet._adaptable())
    if adapter_name is None:
        i = 0
        while f"default_{i}" in unet.peft_config:
            i += 1
        adapter_name = f"default_{i}"
    unet._check_new_adapter_name(adapter_name)
    plan = []
    for m, e in mods.items():
        r = int(e["down"].shape[0])
        alpha = float(e["alpha"].reshape(()).item()) if "alpha" in e else float(r)
        parent, attr, child = slots[m]
        plan.append((parent, attr, child, r, alpha, "kaiming"))
    unet._inject(adapter_name, plan)
    with torch.no_grad():
        for m, e in mods.items():
            parent, attr, _ = slots[m]
            layer = getattr(parent, attr)
            for fac, t in ((layer.lora_A[adapter_name].weight, e["down"]), (layer.lora_B[adapter_name].weight, e["up"])):
                fac.copy_(t)
                fac.requires_grad_(False)
    targets = sorted({m.rsplit(".", 1)[-1] if not m.endswith("to_out.0") else "to_out.0" for m in mods})
    ranks = {int(e["down"].shape[0]) for e in mods.values()}
    unet.peft_config[adapter_name] = _LoadedConfig(r=max(ranks), lora_alpha=None, target_modules=targets)
    return adapter_name


class _LoadedConfig:
    """what is known of a loaded adapter's LoraConfig (rank and alpha are per layer on the LoraLinear modules)"""

    def __init__(self, r: int, lora_alpha, target_modules: List[str]):
        self.r, self.lora_alpha, self.target_modules = r, lora_alpha, target_modules

    def __repr__(self):
        return f"LoadedLoraConfig(r={self.r}, target_modules={self.target_modules})"


def lora_adapter_state_dict(unet, adapter_name: str = "default") -> Dict[str, torch.Tensor]:
    """one adapter's factors under PEFT's names without the adapter name (`<module>.lora_A.weight` / `.lora_B.weight`), as
    `get_peft_model_state_dict(unet, adapter_name=...)` returns them; plus `<module>.alpha` for a layer whose lora_alpha is
    not its rank (an adapter loaded from such a file), which PEFT's dict would lose"""
    if adapter_name not in unet.peft_config:
        raise ValueError(f"unknown adapter {adapter_name!r}; present: {list(unet.peft_config)}")
    out = {}
    for full, _, _, layer in unet._linear_slots():
        if hasattr(layer, "lora_A") and adapter_name in layer.lora_A:
            out[f"{full}.lora_A.weight"] = layer.lora_A[adapter_name].weight.detach()
            out[f"{full}.lora_B.weight"] = layer.lora_B[adapter_name].weight.detach()
            alpha = getattr(layer, "lora_alpha", {}).get(adapter_name)
            if alpha is not None and float(alpha) != float(layer.r[adapter_name]):
                out[f"{full}.alpha"] = torch.tensor(float(alpha))
    return out


# ----------------------------------------------------------------------------- merge
def merge_cost(items) -> Tuple[float, float]:
    """(operations, HBM bytes) of one merge launch, from shapes: 2 r N K per term, W read and written once, each factor
    read once per tile row / column it meets (counted once here: the floor)"""
    flops = nbytes = 0.0
    for w, terms in items:
        N, K = w.shape
        nbytes += 2.0 * w.numel() * w.element_size()
        for A, B, _ in terms:
            flops += 2.0 * A.shape[0] * N * K
            nbytes += (A.numel() + B.numel()) * A.element_size()
    return flops, nbytes


def merge_into_base(items: Sequence[Tuple[torch.Tensor, Sequence[Tuple[torch.Tensor, torch.Tensor, float]]]]) -> None:
    """items: (W [N, K], [(A [r, K], B [N, r], scale), ...]) -> W += sum of scale * B A, in place, all in one svdx_lora_merge
    launch (arithmetic: oracle/svd_lora_oracle.py). Scales are Python floats, rounded to fp32 here."""
    items = [(w, tl) for w, tl in items if tl]
    jobs, terms, prefix = bytearray(), bytearray(), []
    tiles = nterms = 0
    keep = []
    dev = None
    for w, tl in items:
        if w.dim() != 2 or not w.is_contiguous() or not w.is_cuda:
            raise ValueError("lora merge: base weights must be contiguous 2-D CUDA tensors")
        dev = w.device if dev is None else dev
        N, K = w.shape
        for A, B, s in tl:
            if A.dtype != B.dtype or A.dim() != 2 or B.dim() != 2 or A.shape[1] != K or B.shape[0] != N or A.shape[0] != B.shape[1] \
                    or A.shape[0] < 1:
                raise ValueError(f"lora merge: factors A {tuple(A.shape)} / B {tuple(B.shape)} do not fit W [{N}, {K}]")
            A, B = A.detach().contiguous(), B.detach().contiguous()
            if A.device != w.device or B.device != w.device:
                raise ValueError("lora merge: factors must be on the base weight's device")
            keep += [A, B]
            terms += struct.pack("<qqiifi", A.data_ptr(), B.data_ptr(), A.shape[0], raw.dtype_code(A, "LoRA factor"), float(s), 0)
        jobs += struct.pack("<qqqiiii", w.data_ptr(), N, K, raw.dtype_code(w, "base weight"), nterms, len(tl), 0)
        prefix.append(tiles)
        nterms += len(tl)
        tiles += ((N + raw.LM_TILE - 1) // raw.LM_TILE) * ((K + raw.LM_TILE - 1) // raw.LM_TILE)
    if not prefix:
        return
    if tiles >= 2 ** 31:
        raise ValueError("lora merge: more than 2^31 tiles in one launch")
    jt = torch.frombuffer(jobs, dtype=torch.uint8).to(dev)
    tt = torch.frombuffer(terms, dtype=torch.uint8).to(dev)
    pt = torch.tensor(prefix, dtype=torch.int32, device=dev)
    flops, nbytes = merge_cost(items)
    raw.lora_merge(jt, tt, pt, len(prefix), tiles, flops, nbytes)
