"""The convolution plans of the flagship workloads and of the bit-exact kernel cases, as a table.

``tests/golden/conv_plans.json`` holds, for every ``ConvForward``, ``ConvDgrad`` and ``ConvWgrad`` that the workloads
below construct (in construction order), the inputs of each of its plans as ``ops.conv.plan_conv`` /
``ops.conv.plan_wgrad`` take them and the tiling the plan got.  ``test_conv_planning.py`` replays the inputs through
the planner on the CPU; ``test_conv_plans.py`` builds the workloads on the GPU and compares every plan with the table.

``python tests/conv_plan_table.py OUT.json`` (on a GPU) records the table again.
"""
from __future__ import annotations

import contextlib
import dataclasses
import gc
import json
import os
import sys

import torch

TABLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_plans.json")

CONV_PROPS = ("block_n", "resident_filter", "halo", "tiles", "grid", "stats_mode", "has_tail")
WGRAD_PROPS = ("grid", "units", "stages", "G", "px_chunks", "mode")


def _resnet(training: bool):
    from b200ddl.models.resnet_engine import ResNet50Engine

    return ResNet50Engine(batch=256, image_size=224).build(training=training)


def _mobilenet(fine_tune_at):
    from b200ddl.models.mobilenet_engine import MobileNetV2Engine

    return MobileNetV2Engine(batch=32, image_size=224, fine_tune_at=fine_tune_at).build(training=True)


def _exact_cases():
    """Every convolution case of test_conv_exact.py, each under its own A/B switches."""
    import pytest

    import test_conv_exact as T

    kept = []
    for case in T.CONV_CASES + list(T.TAIL_CASES):
        with pytest.MonkeyPatch.context() as mp:
            kept.append(T._setup(case, mp)["op"])
    for case in T.WG_CASES:
        kept.append(T._wgrad_op(case)[0])
    return kept


WORKLOADS = {
    "resnet50_b256_train": lambda: _resnet(True),
    "resnet50_b256_infer": lambda: _resnet(False),
    "mobilenetv2_b32_frozen": lambda: _mobilenet(None),
    "mobilenetv2_b32_fine_tune_at_0": lambda: _mobilenet(0),
    "mobilenetv2_b32_fine_tune_at_14": lambda: _mobilenet(14),
    "conv_exact_cases": _exact_cases,
}


def _plain(v):
    if dataclasses.is_dataclass(v):
        return _plain(dataclasses.asdict(v))
    if isinstance(v, dict):
        return {k: _plain(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [_plain(x) for x in v]
    return v


@contextlib.contextmanager
def recording(ops: list):
    """Appends one entry per constructed ConvForward / ConvDgrad / ConvWgrad to ``ops``: its planner inputs per plan
    (captured at the ``plan_conv`` / ``plan_wgrad`` call) and, filled in by :func:`finish`, the tilings it got."""
    from b200ddl.ops import conv as C

    inputs = []
    saved = {}

    def capture(name):
        fn = getattr(C, name)

        def wrapped(**kw):
            inputs.append(_plain({k: v for k, v in kw.items() if k != "sm_count"}))
            return fn(**kw)
        saved[name] = fn
        setattr(C, name, wrapped)

    def wrap(cls):
        init = cls.__init__

        def wrapped(self, *a, **kw):
            del inputs[:]
            init(self, *a, **kw)
            ops.append({"op": cls.__name__, "obj": self, "inputs": list(inputs)})
        saved[cls] = init
        cls.__init__ = wrapped

    capture("plan_conv")
    capture("plan_wgrad")
    for cls in (C.ConvForward, C.ConvDgrad, C.ConvWgrad):
        wrap(cls)
    try:
        yield
    finally:
        for k, v in saved.items():
            if isinstance(k, str):
                setattr(C, k, v)
            else:
                k.__init__ = v


def finish(entry: dict) -> dict:
    """The table entry of a recorded op: plan inputs, pixel box and plan properties (read after the workload is built)."""
    op = entry.pop("obj")
    if entry["op"] == "ConvDgrad":
        plans, boxes, props = [p for p, _, _ in op.parts], op.boxes, CONV_PROPS
    else:
        plans, boxes = [op.plan], [op.box]
        props = WGRAD_PROPS if entry["op"] == "ConvWgrad" else CONV_PROPS
    assert len(entry["inputs"]) == len(plans), entry
    entry["plans"] = [{"inputs": i, "box": list(b), "props": {k: _plain(getattr(p, k)) for k in props}}
                      for i, b, p in zip(entry.pop("inputs"), boxes, plans)]
    return entry


def build_workload(name: str) -> list:
    ops = []
    with recording(ops):
        keep = WORKLOADS[name]()
    torch.cuda.synchronize()
    table = [dict(workload=name, **finish(e)) for e in ops]
    del keep, ops
    gc.collect()
    torch.cuda.empty_cache()
    return table


def record() -> dict:
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    ops = []
    for name in WORKLOADS:
        ops += build_workload(name)
    return {"device": props.name, "sm_count": props.multi_processor_count, "ops": ops}


def write(table: dict, path: str) -> None:
    """One op per line, so that a change of plan shows as a readable diff."""
    head = {k: v for k, v in table.items() if k != "ops"}
    with open(path, "w") as f:
        f.write(json.dumps(head)[:-1] + ', "ops": [\n')
        f.write(",\n".join(json.dumps(op, separators=(",", ":")) for op in table["ops"]))
        f.write("\n]}\n")


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import b200ddl  # noqa: F401

    write(record(), sys.argv[1])
