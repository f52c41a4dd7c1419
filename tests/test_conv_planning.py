"""CPU tests of the convolution planning layer (pixel boxes, tap tables, parity views, tilings)."""
import json

import pytest
import torch
from hypothesis import given, settings, strategies as st

from b200ddl.ops import conv as C
from conv_plan_table import TABLE, WORKLOADS


@settings(max_examples=60, deadline=None)
@given(n=st.integers(1, 300), hw=st.sampled_from([7, 14, 28, 56, 112]), rows=st.sampled_from([64, 128]),
       mult=st.sampled_from([1, 16]))
def test_pick_box_invariants(n, hw, rows, mult):
    bw, bh, bn = C.pick_box(n, hw, hw, rows=rows, multiple_of=mult)
    assert hw % bw == 0 and hw % bh == 0            # exact spatial tiling (no halo pickup)
    assert 1 <= bw * bh * bn <= rows and (bw * bh * bn) % mult == 0


def _emulate(x, taps: C.TapTable, w_tck, R, S, Ho, Wo):
    """Evaluate the tap table the way the kernel does: out[p] = sum_t view[t][p + offset_t] @ w[t]^T, OOB = 0."""
    N = x.shape[0]
    out = torch.zeros(N, Ho, Wo, w_tck.shape[1])
    for t, (vi, dw, dh) in enumerate(zip(taps.tap_map, taps.tap_dw, taps.tap_dh)):
        v = taps.views[vi]
        Hv, Wv = v.shape[1], v.shape[2]
        pad = torch.zeros(N, Hv + 8, Wv + 8, v.shape[3])
        pad[:, 4:4 + Hv, 4:4 + Wv] = v
        win = pad[:, 4 + dh:4 + dh + Ho, 4 + dw:4 + dw + Wo]
        out += win @ w_tck[t].T
    return out


@pytest.mark.parametrize("R,stride,pad,H", [(1, 1, 0, 8), (3, 1, 1, 8), (3, 2, 1, 8), (1, 2, 0, 8), (3, 2, 1, 14)])
def test_tap_table_matches_conv2d(R, stride, pad, H):
    torch.manual_seed(0)
    x = torch.randn(2, H, H, 5)
    w = torch.randn(R * R, 4, 5)
    taps = C.make_taps(x, R, R, stride, pad)
    Ho = (H + 2 * pad - R) // stride + 1
    got = _emulate(x, taps, w, R, R, Ho, Ho)
    ref = C.conv_reference(x, w, R, R, stride, pad)
    assert torch.allclose(got, ref, atol=1e-4)
    assert len(taps.views) <= 4


@pytest.mark.parametrize("R,stride,pad,H", [(1, 1, 0, 6), (3, 1, 1, 6), (3, 2, 1, 8), (1, 2, 0, 8), (3, 2, 1, 14)])
def test_dgrad_parity_parts_match_conv_transpose(R, stride, pad, H):
    """The dgrad GEMMs (one per output-parity class, each a forward-style tap table over dy) sum to conv_transpose."""
    torch.manual_seed(0)
    Ho = (H + 2 * pad - R) // stride + 1
    dy = torch.randn(2, Ho, Ho, 4)
    w = torch.randn(R * R, 4, 5)   # [tap, Cout, Cin]
    dx = torch.zeros(2, H, H, 5)
    for (ph, pw), idx, dw, dh in C.ConvDgrad.parity_parts(R, R, stride, pad):
        out = dx[:, ph::stride, pw::stride]
        taps = C.TapTable([dy], [0] * len(idx), dw, dh)
        out += _emulate(dy, taps, w[idx].transpose(1, 2), 1, 1, out.shape[1], out.shape[2])
    ref = torch.nn.grad.conv2d_input((2, 5, H, H), C.weight_from_kernel_layout(w, R, R), dy.permute(0, 3, 1, 2),
                                     stride=stride, padding=pad).permute(0, 2, 3, 1)
    assert torch.allclose(dx, ref, atol=1e-4)
    # the order the ResNet engine lays its dgrad weight copies out in
    assert C.ConvDgrad.part_taps(3, 3, 2, 1) == [[4], [3, 5], [1, 7], [0, 2, 6, 8]]
    assert C.ConvDgrad.part_taps(3, 3, 1, 1) == [list(range(9))]


def test_weight_layout_roundtrip():
    w = torch.randn(8, 3, 3, 3)
    k = C.weight_to_kernel_layout(w)
    assert k.shape == (9, 8, 3)
    assert torch.equal(C.weight_from_kernel_layout(k, 3, 3), w)
    out = torch.zeros(64, 192)
    ws = torch.randn(49, 64, 3)
    C.pack_stem_weight(ws, out)
    assert torch.equal(out[5, 3 * 17 + 2], ws[17, 5, 2]) and float(out[:, 147:].abs().sum()) == 0.0


def test_dgrad_refuses_fused_reductions_when_strided():
    """A stride-2 dgrad has no fused BatchNorm-backward reduction: asking for one is an error, not silently zero sums."""
    dy = torch.zeros(1, 4, 4, 64, dtype=torch.bfloat16)
    dx = torch.zeros(1, 8, 8, 64, dtype=torch.bfloat16)
    w = torch.zeros(9, 64, 64)
    z = torch.zeros(64)
    with pytest.raises(ValueError, match="bwd_stats: stride-1"):
        C.ConvDgrad(dy, w, dx, 3, 3, 2, 1, bwd_stats=(dx, z, z, z.clone(), z.clone()))
    with pytest.raises(ValueError, match="block_grad: stride-1"):
        C.ConvDgrad(dy, w, dx, 3, 3, 2, 1, block_grad=(dx, z, dx, z.clone(), z.clone()))


def _forward_tiling(h, w, cin=64, cout=64, R=3, stride=1, pad=1, switches=C.ConvSwitches()):
    """plan_conv of a box-mode forward conv over a (2, h, w, cin) input (views and tap table from make_taps), and its
    output grid."""
    taps = C.make_taps(torch.empty(2, h, w, cin, device="meta"), R, R, stride, pad)
    grid = (2, (h + 2 * pad - R) // stride + 1, (w + 2 * pad - R) // stride + 1)
    t = C.plan_conv(grid=grid, view_widths=[v.shape[2] for v in taps.views], cin=cin, cout=cout, tap_map=taps.tap_map,
                    tap_dw=taps.tap_dw, tap_dh=taps.tap_dh, flat=False, stats_mode=0, max_ctas=0, sm_count=132,
                    switches=switches)
    return t, grid


def test_halo_tiling_selection(monkeypatch):
    """Full-width single-image boxes only for the 3x3 / stride-1 / 64->64 layers whose box + halo fits one 28 KB stage and
    whose width is a multiple of 8 (the vertical taps start whole 8-row swizzle atoms into the stage); every other layer
    gets the generic box."""
    def halo(h, w, **kw):
        t, grid = _forward_tiling(h, w, **kw)
        if t.halo:
            assert t.resident_filter
            return t.box
        assert t.box == C.pick_box(*grid)
        return None

    assert halo(56, 56) == (56, 2, 1)                    # 112-pixel tile, 224-pixel halo stage
    assert halo(24, 24) == (24, 4, 1)
    assert halo(28, 28) is None                          # 28-row tap offsets are not whole swizzle atoms
    assert halo(56, 56, cin=128, cout=128) is None       # filter does not fit resident
    assert halo(56, 56, stride=2) is None                # strided
    assert halo(56, 56, R=1, pad=0) is None
    assert halo(112, 112) is None                        # one image row + halo exceeds a stage
    assert halo(56, 56, switches=C.ConvSwitches(no_halo=True)) is None
    assert halo(56, 56, switches=C.ConvSwitches(no_resident_filter=True)) is None
    for k in ("B200DDL_BLOCK_N", "B200DDL_NO_HALO", "B200DDL_NO_RESIDENT_FILTER"):
        monkeypatch.delenv(k, raising=False)
    assert C.conv_switches() == C.ConvSwitches()
    monkeypatch.setenv("B200DDL_NO_HALO", "1")
    monkeypatch.setenv("B200DDL_BLOCK_N", "128")
    assert C.conv_switches() == C.ConvSwitches(block_n=128, no_halo=True)
    monkeypatch.setenv("B200DDL_NO_RESIDENT_FILTER", "1")
    monkeypatch.setenv("B200DDL_BLOCK_N", "96")
    assert C.conv_switches() == C.ConvSwitches(no_halo=True, no_resident_filter=True)


def test_planner_reproduces_recorded_plans():
    """Every plan of the flagship workloads and of the bit-exact kernel cases (tests/golden/conv_plans.json, recorded on
    an H100), replayed through the pure planner: the same tiling, field for field."""
    with open(TABLE) as f:
        table = json.load(f)
    sm = table["sm_count"]
    seen = set()
    for i, op in enumerate(table["ops"]):
        for j, p in enumerate(op["plans"]):
            inp, want = dict(p["inputs"]), p["props"]
            if op["op"] == "ConvWgrad":
                t = C.plan_wgrad(**inp, sm_count=sm)
                got = dict(grid=t.grid, units=t.units, stages=t.stages, G=t.G, px_chunks=t.px_chunks,
                           mode=int(not inp["flat"]))
            else:
                inp["switches"] = C.ConvSwitches(**inp["switches"])
                t = C.plan_conv(**inp, sm_count=sm)
                got = dict(block_n=t.block_n, resident_filter=int(t.resident_filter), halo=int(t.halo), tiles=t.tiles,
                           grid=t.grid, stats_mode=inp["stats_mode"], has_tail=False)
            assert (list(t.box), got) == (p["box"], want), f"op {i} ({op['workload']} {op['op']}) plan {j}: {inp}"
            seen.add(op["workload"])
    assert seen == set(WORKLOADS)
