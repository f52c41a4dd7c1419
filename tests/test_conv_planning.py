"""CPU tests of the convolution planning layer (pixel boxes, tap tables, parity views) against torch conv semantics."""
import pytest
import torch
from hypothesis import given, settings, strategies as st

from b200ddl.ops import conv as C


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


def test_halo_box_selection(monkeypatch):
    """Full-width single-image boxes only for the 3x3 / stride-1 / 64->64 layers whose box + halo fits one 28 KB stage and
    whose width is a multiple of 8 (the vertical taps start whole 8-row swizzle atoms into the stage)."""
    from b200ddl.ops import conv as C

    monkeypatch.delenv("B200DDL_NO_HALO", raising=False)
    monkeypatch.delenv("B200DDL_NO_RESIDENT_FILTER", raising=False)
    assert C.halo_box(56, 56, 64, 64, 3, 3, 1, 1) == (56, 2, 1)      # 112-pixel tile, 224-pixel halo stage
    assert C.halo_box(24, 24, 64, 64, 3, 3, 1, 1) == (24, 4, 1)
    assert C.halo_box(28, 28, 64, 64, 3, 3, 1, 1) is None            # 28-row tap offsets are not whole swizzle atoms
    assert C.halo_box(56, 56, 128, 128, 3, 3, 1, 1) is None          # filter does not fit resident
    assert C.halo_box(56, 56, 64, 64, 3, 3, 2, 1) is None            # strided
    assert C.halo_box(56, 56, 64, 64, 1, 1, 1, 0) is None
    assert C.halo_box(112, 112, 64, 64, 3, 3, 1, 1) is None          # one image row + halo exceeds a stage
    monkeypatch.setenv("B200DDL_NO_HALO", "1")
    assert C.halo_box(56, 56, 64, 64, 3, 3, 1, 1) is None
