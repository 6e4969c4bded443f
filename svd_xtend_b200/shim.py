"""Launcher shim: run the reference's training scripts UNCHANGED on the H100 path.

    python -m svd_xtend_b200.shim train_svd.py --pretrained_model_name_or_path=... [script args]
    accelerate launch -m svd_xtend_b200.shim train_svd.py ...

Before the script body runs, the replacement class is installed under the two names the reference
imports the UNet from: `diffusers.UNetSpatioTemporalConditionModel` (train_svd.py:49) and
`src.unet_spatio_temporal_condition.UNetSpatioTemporalConditionModel` (train_svd_lora.py:60), and the EMA as
`diffusers.training_utils.EMAModel` (train_svd.py:52, used with --use_ema). Where transformers is
importable, the image encoder is also installed as `transformers.CLIPVisionModelWithProjection` (train_svd.py:646-647).
diffusers / accelerate are NOT part of this image (no network), so this shim is exercised only where a
user's environment provides them; it fails loudly when they are missing.
"""
from __future__ import annotations

import importlib
import runpy
import sys
import types


def install() -> None:
    from .unet import UNetSpatioTemporalConditionModel
    try:
        diffusers = importlib.import_module("diffusers")
    except ModuleNotFoundError as e:
        raise RuntimeError("svd_xtend_b200.shim: the reference scripts need `diffusers`, which is not installed here") from e
    diffusers.UNetSpatioTemporalConditionModel = UNetSpatioTemporalConditionModel
    for modname in ("diffusers.models", "diffusers.models.unets", "diffusers.models.unets.unet_spatio_temporal_condition"):
        try:
            m = importlib.import_module(modname)
            setattr(m, "UNetSpatioTemporalConditionModel", UNetSpatioTemporalConditionModel)
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
    install_clip()


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
    install()
    script = argv[0]
    sys.argv = argv
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
