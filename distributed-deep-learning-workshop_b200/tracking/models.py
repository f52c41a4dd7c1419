"""Model flavour: `mlflow.keras.log_model(model, 'model')` / `mlflow.keras.load_model('runs:/<id>/model')`
(reference P1/03:373,438; registry load `models:/<name>/production`, P2/01:298)."""
from __future__ import annotations

import json
import os
from typing import Optional

import torch


def _augmentation(model) -> Optional[dict]:
    aug = getattr(model, "augmentation", None)
    return aug.to_dict() if aug is not None else None


def _describe(model) -> dict:
    if hasattr(model, "param_specs"):  # native engines (ResNet50Engine, MobileNetV2Engine)
        desc = {"arch": getattr(model, "arch", "resnet50"), "num_classes": model.num_classes, "image_size": model.image_size,
                "dropout": model.dropout, "batch": model.batch, "engine": True, "augmentation": _augmentation(model),
                "seed": model.seed}   # the seed keys the augmentation draws: a reloaded engine continues the sequence
        if desc["arch"] in ("mobilenetv2", "resnet50_head"):
            desc["fine_tune_at"] = model.fine_tune_at
            desc["batchnorm"] = model.batchnorm
        return desc
    from ..models.mobilenet import FrozenBaseClassifier
    from ..models.resnet import ResNet50Head

    if isinstance(model, ResNet50Head):
        return {"arch": "resnet50_head", "num_classes": model.fc.out_features, "dropout": model.dropout.p,
                "fine_tune_at": model.fine_tune_at, "batchnorm": model.batchnorm, "augmentation": _augmentation(model),
                "augmentation_seed": model.augmentation_seed}
    if isinstance(model, FrozenBaseClassifier):
        return {"arch": "mobilenetv2", "num_classes": model.fc.out_features, "dropout": model.dropout.p,
                "freeze_base": model.freeze_base, "fine_tune_at": model.fine_tune_at, "batchnorm": model.batchnorm,
                "augmentation": _augmentation(model), "augmentation_seed": model.augmentation_seed}
    return {"arch": "pickle"}


def save_model(model_or_trainer, path: str) -> None:
    model = getattr(model_or_trainer, "model", model_or_trainer)
    os.makedirs(path, exist_ok=True)
    desc = _describe(model)
    if desc["arch"] == "pickle":
        import cloudpickle

        with open(os.path.join(path, "model.pkl"), "wb") as f:
            cloudpickle.dump(model.cpu() if hasattr(model, "cpu") else model, f)
    else:
        sd = model.state_dict()
        torch.save({k: v.detach().cpu() for k, v in sd.items()}, os.path.join(path, "weights.pt"))
    with open(os.path.join(path, "MLmodel.json"), "w") as f:
        json.dump({"flavor": "b200ddl.model", **desc}, f)


def log_model(model_or_trainer, artifact_path: str = "model") -> str:
    from . import get_artifact_uri, active_run

    path = get_artifact_uri(artifact_path)
    save_model(model_or_trainer, path)
    return f"runs:/{active_run().info.run_id}/{artifact_path}"


def load_model(model_uri: str, batch_size: Optional[int] = None, device=None):
    """Returns a compiled-for-inference `Trainer` (has `.predict`, `.summary`, `.model`)."""
    from . import resolve_uri
    from ..models import Augmentation, build_model
    from ..train import Trainer

    path = resolve_uri(model_uri)
    with open(os.path.join(path, "MLmodel.json")) as f:
        desc = json.load(f)
    if desc["arch"] == "pickle":
        import cloudpickle

        with open(os.path.join(path, "model.pkl"), "rb") as f:
            model = cloudpickle.load(f)
        return Trainer(model, device=device)
    sd = torch.load(os.path.join(path, "weights.pt"), map_location="cpu")
    aug = Augmentation.from_dict(desc.get("augmentation"))
    if desc["arch"] == "resnet50":
        if torch.cuda.is_available():
            model = build_model(desc["image_size"], desc["image_size"], 3, desc["num_classes"], desc["dropout"],
                                arch="resnet50", batch_size=batch_size or desc["batch"], device=device, augmentation=aug,
                                seed=desc.get("seed", 0))
            model.load_state_dict(sd)
        else:  # CPU box: same weights in the torchvision-architecture module (inference only: no augmentation)
            model = build_model(num_classes=desc["num_classes"], arch="resnet50_torch")
            model.load_state_dict(sd, strict=False)
    elif desc["arch"] == "resnet50_head":   # the engine on a GPU, the torch module on a CPU (same state-dict keys)
        gpu = desc.get("engine") and torch.cuda.is_available()
        size = desc["image_size"] if gpu else 224
        model = build_model(size, size, 3, desc["num_classes"], desc["dropout"], arch="resnet50_head",
                            batch_size=batch_size or desc.get("batch", 32), device=device if gpu else "cpu",
                            fine_tune_at=desc.get("fine_tune_at"), augmentation=aug,
                            seed=desc.get("seed", desc.get("augmentation_seed", 0)),
                            batchnorm=desc.get("batchnorm", "inference"))
        if gpu:
            model.load_state_dict(sd)
        else:   # the engine keeps no num_batches_tracked
            missing = model.load_state_dict(sd, strict=False).missing_keys
            assert all(k.endswith("num_batches_tracked") for k in missing), missing
    elif desc.get("engine") and torch.cuda.is_available():  # saved from the native MobileNetV2 engine
        model = build_model(desc["image_size"], desc["image_size"], 3, desc["num_classes"], desc["dropout"],
                            arch="mobilenetv2", batch_size=batch_size or desc["batch"], device=device,
                            fine_tune_at=desc.get("fine_tune_at"), augmentation=aug, seed=desc.get("seed", 0),
                            batchnorm=desc.get("batchnorm", "inference"))
        model.load_state_dict(sd)
    else:
        model = build_model(num_classes=desc["num_classes"], dropout=desc["dropout"], arch="mobilenetv2_torch",
                            freeze_base=desc.get("freeze_base", True), fine_tune_at=desc.get("fine_tune_at"),
                            augmentation=aug, seed=desc.get("augmentation_seed", 0),
                            batchnorm=desc.get("batchnorm", "inference"))
        model.load_state_dict(sd)
    return Trainer(model, device=device)
