"""GPU checks of the convolution plans: the flagship workloads and the bit-exact cases get the tilings recorded in
tests/golden/conv_plans.json, and the plan bindings reject every tiling the kernels cannot run (construction only:
nothing is launched)."""
from __future__ import annotations

import dataclasses
import json

import pytest
import torch

import conv_plan_table as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def table():
    with open(T.TABLE) as f:
        return json.load(f)


@pytest.mark.parametrize("workload", list(T.WORKLOADS))
def test_plans_match_recorded_table(workload, table, monkeypatch):
    sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    if sm != table["sm_count"]:
        pytest.skip(f"the table was recorded on a {table['sm_count']}-SM device, this one has {sm}")
    for k in ("B200DDL_BLOCK_N", "B200DDL_NO_RESIDENT_FILTER", "B200DDL_NO_HALO"):
        monkeypatch.delenv(k, raising=False)
    want = [op for op in table["ops"] if op["workload"] == workload]
    got = T.build_workload(workload)
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{workload} op {i} ({w['op']})"


def _C():
    import b200ddl  # noqa: F401
    from b200ddl.ops import _build
    from b200ddl.ops import conv as C

    return C, _build.load("_b200_conv")


def _conv_plan(change: dict, N=2, H=8, W=56, cin=64, cout=64, R=3, stride=1, block_grad=False):
    """Builds the ConvPlan binding of a forward conv with the planner's tiling, changed by ``change``."""
    C, ext = _C()
    pad = R // 2
    bf = dict(device="cuda", dtype=torch.bfloat16)
    x = torch.zeros(N, H, W, cin, **bf)
    taps = C.make_taps(x, R, R, stride, pad)
    y = torch.zeros(N, (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1, cout, **bf)
    w = torch.zeros(R * R * cout, cin, **bf)
    outputs = {}
    if block_grad:
        z = torch.zeros(cout, device="cuda")
        outputs = dict(stat_sum=z, stat_sqsum=z.clone(), bwd_y=torch.zeros_like(y), add_src=torch.zeros_like(y),
                       relu_mask=torch.zeros(y.numel() // 8, device="cuda", dtype=torch.uint8))
    t = C.plan_conv(grid=tuple(y.shape[:3]), view_widths=[v.shape[2] for v in taps.views], cin=cin, cout=cout,
                    tap_map=taps.tap_map, tap_dw=taps.tap_dw, tap_dh=taps.tap_dh, flat=R == 1 and stride == 1,
                    stats_mode=3 if block_grad else 0, max_ctas=0, sm_count=C.sm_count(), switches=C.ConvSwitches())
    t = dataclasses.replace(t, **change)
    bw, bh, bn = t.box
    return ext.ConvPlan(taps.views, w, y, taps.tap_map, taps.tap_dw, taps.tap_dh, bw=bw, bh=bh, bn=bn,
                        block_n=t.block_n, resident_filter=t.resident_filter, halo=t.halo, grid=t.grid, **outputs)


CONV_REJECTS = [
    ("block_n_96", dict(change=dict(block_n=96, resident_filter=False, halo=False))),
    ("block_n_128_cout_192", dict(change=dict(block_n=128), cin=128, cout=192)),
    ("resident_two_n_blocks", dict(change=dict(block_n=64, resident_filter=True), cin=64, cout=128)),
    ("resident_18_filter_tiles", dict(change=dict(resident_filter=True), cin=128, cout=64)),
    ("resident_block_gradient", dict(change=dict(resident_filter=True), H=8, W=8, R=1, block_grad=True)),
    ("halo_without_resident", dict(change=dict(resident_filter=False))),
    ("halo_1x1", dict(change=dict(halo=True), H=8, W=56, R=1, stride=2)),
    ("halo_strided", dict(change=dict(halo=True, box=(28, 4, 1)), H=16, W=56, stride=2)),
    ("halo_flat", dict(change=dict(halo=True), R=1)),
    ("halo_narrow_box", dict(change=dict(box=(8, 2, 1)))),
    ("halo_width_not_8k", dict(change=dict(box=(28, 4, 1), halo=True), H=8, W=28)),
    ("halo_two_images", dict(change=dict(box=(8, 4, 2), halo=True), H=8, W=8)),
    ("halo_stage_over_224", dict(change=dict(box=(64, 2, 1), halo=True), H=8, W=64)),
    ("grid_0", dict(change=dict(grid=0))),
    ("grid_over_tiles", dict(change=dict(grid=1000))),
]


def test_conv_reject_cases_start_from_valid_plans():
    """Each reject case changes one property of a plan the binding accepts."""
    for _, kw in CONV_REJECTS:
        kw = dict(kw, change={})
        _conv_plan(**kw)


@pytest.mark.parametrize("name,kw", CONV_REJECTS, ids=[c[0] for c in CONV_REJECTS])
def test_conv_plan_rejects_malformed_tiling(name, kw):
    check = {"block": "block_n", "resident": "resident filter", "halo": "halo mode", "grid": "grid"}[name.split("_")[0]]
    with pytest.raises(RuntimeError, match=check):
        _conv_plan(**kw)


def _wgrad_plan(change: dict, N=2, H=12, W=20, cin=64, cout=128, R=3):
    """Builds the WgradPlan binding of a box-mode weight gradient with the planner's tiling, changed by ``change``
    (values may be callables of the planned tiling)."""
    C, ext = _C()
    x = torch.zeros(N, H, W, cin, device="cuda", dtype=torch.bfloat16)
    dy = torch.zeros(N, H, W, cout, device="cuda", dtype=torch.bfloat16)
    dw = torch.zeros(R * R * cout, cin, device="cuda")
    taps = C.make_taps(x, R, R, 1, R // 2)
    t = C.plan_wgrad(grid=(N, H, W), cin=cin, cout=cout, R=R, S=R, flat=False, px_chunks=0, max_ctas=0, smem_budget=0,
                     sm_count=C.sm_count())
    t = dataclasses.replace(t, **{k: v(t) if callable(v) else v for k, v in change.items()})
    bw, bh, bn = t.box
    return ext.WgradPlan(dy, taps.views, dw, R, R, taps.tap_map, taps.tap_dw, taps.tap_dh, bw=bw, bh=bh, bn=bn,
                         cb_per_group=t.cb_per_group, stages=t.stages, px_chunks=t.px_chunks, grid=t.grid)


def _iters(t):
    bw, bh, bn = t.box
    return (20 // bw) * (12 // bh) * -(-2 // bn)


def _uneven_chunks(t):
    """A pixel-chunk count that leaves a chunk empty."""
    n = _iters(t)
    return next(pc for pc in range(1, n + 1) if -(-n // -(-n // pc)) != pc)


WGRAD_REJECTS = [
    ("stages_1", dict(stages=1)),
    ("stages_over_budget", dict(stages=lambda t: t.stages + 1)),
    ("cb_per_group_not_dividing", dict(cb_per_group=3)),
    ("px_chunks_0", dict(px_chunks=0)),
    ("px_chunks_over_iterations", dict(px_chunks=lambda t: _iters(t) + 1)),
    ("px_chunks_with_an_empty_chunk", dict(px_chunks=_uneven_chunks)),
    ("grid_0", dict(grid=0)),
    ("grid_over_units", dict(grid=lambda t: t.units + 1)),
]


def test_wgrad_plan_rejects_malformed_tiling():
    p = _wgrad_plan({})
    assert (p.stages, p.G) == (3, 3)      # the base case has a full 227 KB stage budget
    for name, change in WGRAD_REJECTS:
        check = {"stages": "stages", "cb": "cb_per_group", "px": "px_chunks", "grid": "grid"}[name.split("_")[0]]
        with pytest.raises(RuntimeError, match=check):
            _wgrad_plan(change)
            pytest.fail(name)
