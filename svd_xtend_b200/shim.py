"""Launcher shim: run the reference's training scripts UNCHANGED on the H100 path.

    python -m svd_xtend_b200.shim train_svd.py --pretrained_model_name_or_path=... [script args]
    accelerate launch -m svd_xtend_b200.shim train_svd.py ...

Before the script body runs, this package's classes are installed under the names the reference imports them from:
  * the UNet as `diffusers.UNetSpatioTemporalConditionModel` (train_svd.py:49) and
    `src.unet_spatio_temporal_condition.UNetSpatioTemporalConditionModel` (train_svd_lora.py:60);
  * the VAE as `diffusers.AutoencoderKLTemporalDecoder` (train_svd.py:47-50; the per-step encode of :283-291 and the decode of
    every validation video), in a subclass whose `from_pretrained` loads the temporal decoder, as diffusers' class has one;
  * the pipeline as `diffusers.StableVideoDiffusionPipeline` (the validation loop, :1093-1157, and the final
    `save_pretrained`, :1166-1180), built from the passed training modules;
  * the EMA as `diffusers.training_utils.EMAModel` (train_svd.py:52, used with --use_ema);
  * for a run with --use_8bit_adam, the 8-bit AdamW as `bitsandbytes.optim.AdamW8bit` (train_svd.py:746-773);
  * where transformers is importable, the image encoder as `transformers.CLIPVisionModelWithProjection` (train_svd.py:646-647).
diffusers / accelerate are NOT part of this image (no network), so this shim is exercised only where a
user's environment provides them; it fails loudly when they are missing.
"""
from __future__ import annotations

import importlib
import importlib.machinery
import runpy
import sys
import types


def wants_8bit_adam(argv) -> bool:
    """the script's arguments ask for the 8-bit optimizer (`--use_8bit_adam`, a store_true flag, or a prefix argparse accepts
    for it: no other flag of the scripts starts with `--use_8`)"""
    return any(a.startswith("--use_8") and "--use_8bit_adam".startswith(a) for a in argv)


def install(use_8bit_adam: bool | None = None) -> None:
    """use_8bit_adam: also install the 8-bit AdamW (install_adam8bit); None reads `--use_8bit_adam` from sys.argv. Without
    it bitsandbytes is left alone: no import of an installed one, no stand-in that other libraries' probes would find."""
    from .unet import UNetSpatioTemporalConditionModel
    try:
        diffusers = importlib.import_module("diffusers")
    except ModuleNotFoundError as e:
        raise RuntimeError("svd_xtend_b200.shim: the reference scripts need `diffusers`, which is not installed here") from e
    from .pipeline import StableVideoDiffusionPipeline
    from .vae import AutoencoderKLTemporalDecoderWithDecoder
    for name, cls, modnames in (
            ("UNetSpatioTemporalConditionModel", UNetSpatioTemporalConditionModel,
             ("diffusers.models", "diffusers.models.unets", "diffusers.models.unets.unet_spatio_temporal_condition")),
            ("AutoencoderKLTemporalDecoder", AutoencoderKLTemporalDecoderWithDecoder,
             ("diffusers.models", "diffusers.models.autoencoders", "diffusers.models.autoencoders.autoencoder_kl_temporal_decoder")),
            ("StableVideoDiffusionPipeline", StableVideoDiffusionPipeline,
             ("diffusers.pipelines", "diffusers.pipelines.stable_video_diffusion",
              "diffusers.pipelines.stable_video_diffusion.pipeline_stable_video_diffusion"))):
        setattr(diffusers, name, cls)
        for modname in modnames:
            try:
                m = importlib.import_module(modname)
                setattr(m, name, cls)
            except Exception:
                pass
    # train_svd_lora.py imports `from src.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel`
    pkg = sys.modules.get("src") or types.ModuleType("src")
    pkg.__path__ = getattr(pkg, "__path__", [])
    sub = types.ModuleType("src.unet_spatio_temporal_condition")
    sub.UNetSpatioTemporalConditionModel = UNetSpatioTemporalConditionModel
    sys.modules["src"] = pkg
    sys.modules["src.unet_spatio_temporal_condition"] = sub
    pkg.unet_spatio_temporal_condition = sub
    # train_svd.py:52 `from diffusers.training_utils import EMAModel` (--use_ema): the EMA on this package's kernels, whose
    # copy_to / restore move the parameters' version counters (svd_xtend_b200.ema)
    from .ema import EMAModel
    try:
        tu = importlib.import_module("diffusers.training_utils")
        tu.EMAModel = EMAModel
    except ModuleNotFoundError:
        pass
    if wants_8bit_adam(sys.argv[1:]) if use_8bit_adam is None else use_8bit_adam:
        install_adam8bit()
    install_clip()
    install_lora_writer(getattr(diffusers, "StableVideoDiffusionPipeline", None))


def install_lora_writer(pipeline_cls) -> bool:
    """train_svd_lora.py:1064-1074 and :1146-1153 call `StableVideoDiffusionPipeline.save_lora_weights(...)`, which some
    diffusers releases lack. Where the class lacks it, the writer of svd_xtend_b200.lora (diffusers' file layout) is set;
    an existing one is left alone. Returns whether it was set."""
    if pipeline_cls is None or hasattr(pipeline_cls, "save_lora_weights"):
        return False
    from .lora import save_lora_weights
    pipeline_cls.save_lora_weights = staticmethod(save_lora_weights)
    return True


def install_adam8bit():
    """install the block-wise 8-bit AdamW on this package's kernels as `bitsandbytes.optim.AdamW8bit` (train_svd.py:746-773 and
    train_svd_lora.py:732-740 build it for --use_8bit_adam). Where bitsandbytes is importable its module is patched: its own
    update writes the parameters from a kernel that may leave their version counters alone, and the model would then run
    on stale operands. Otherwise a minimal stand-in `bitsandbytes` package (marked `__svdx_standin__ = True`) is registered
    in sys.modules, so the scripts' `import bitsandbytes as bnb` succeeds. The stand-in carries a real module spec, so
    `importlib.util.find_spec("bitsandbytes")` keeps working, and the version "0.0.0+svdx.standin", so libraries that gate
    their bitsandbytes integrations on a minimum version (transformers' `is_bitsandbytes_available`) keep them off: it
    provides the optimizer only. Returns the module."""
    from .optim8bit import AdamW8bit
    try:
        bnb = importlib.import_module("bitsandbytes")
        optim = importlib.import_module("bitsandbytes.optim")
    except ModuleNotFoundError:
        bnb = types.ModuleType("bitsandbytes")
        bnb.__spec__ = importlib.machinery.ModuleSpec("bitsandbytes", None, is_package=True)
        bnb.__path__ = []
        bnb.__version__ = "0.0.0+svdx.standin"
        bnb.__svdx_standin__ = True
        optim = types.ModuleType("bitsandbytes.optim")
        optim.__spec__ = importlib.machinery.ModuleSpec("bitsandbytes.optim", None, is_package=True)
        optim.__path__ = []
        bnb.optim = optim
        sys.modules["bitsandbytes"] = bnb
        sys.modules["bitsandbytes.optim"] = optim
    optim.AdamW8bit = AdamW8bit
    return bnb


def install_clip() -> bool:
    """when transformers is importable, install the H100 image encoder as `transformers.CLIPVisionModelWithProjection`
    (train_svd.py:646-647 loads it from there); without transformers nothing changes. Returns whether it was installed."""
    from .clip import CLIPVisionModelWithProjection
    try:
        transformers = importlib.import_module("transformers")
    except ModuleNotFoundError:
        return False
    transformers.CLIPVisionModelWithProjection = CLIPVisionModelWithProjection
    try:
        m = importlib.import_module("transformers.models.clip")
        setattr(m, "CLIPVisionModelWithProjection", CLIPVisionModelWithProjection)
    except Exception:
        pass
    return True


def main(argv=None) -> None:
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        raise SystemExit("usage: python -m svd_xtend_b200.shim <train_svd.py|train_svd_lora.py> [args...]")
    install(use_8bit_adam=wants_8bit_adam(argv[1:]))
    script = argv[0]
    sys.argv = argv
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
