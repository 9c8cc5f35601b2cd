"""gemm_nt with two consumer warpgroups taking a CTA's 64-row tiles in turn: the tile-count and slice-width cases that the
schedule has to get right, against an fp64 evaluation of the same bf16 operands (bf16 out <= 3e-3, fp32 out <= 1e-5).

An H100 has 132 SMs; N = 900 plans 5 slices of 192 columns, so 26 groups of CTAs share the tiles."""
import pytest

import gpu_checks as G

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kw", [
    dict(M=64, N=900, K=300),               # one tile: warpgroup 1 of the only busy CTA has none
    dict(M=64 * 27, N=900, K=300),          # group 0 takes two tiles, one per warpgroup; every other group exactly one
    dict(M=64 * 53 + 5, N=900, K=300),      # group 0 takes three: warpgroup 0 two, warpgroup 1 one (the last one partial)
    dict(M=64 * 26 * 40 + 33, N=900, K=300),  # long tile sequences per CTA, partial last tile
])
def test_pingpong_tile_counts(kw):
    r = G.check_linear(**kw)
    assert r["nan"] == 0 and r["rel"] < 3e-3 and r["elem_ratio"] <= 1, r


@pytest.mark.parametrize("N", [32, 64, 96, 128, 160, 192, 224, 256, 250])
def test_pingpong_slice_widths(N):
    """One slice of 1..8 32-column chunks (wgmma N = 32..256); an odd count leaves column half 1 idle in the last round."""
    r = G.check_linear(M=64 * 300 + 7, N=N, K=200)
    assert r["nan"] == 0 and r["rel"] < 3e-3 and r["elem_ratio"] <= 1, r


def test_pingpong_fp32_out_odd_chunks():
    r = G.check_linear(M=64 * 41, N=224, K=300, out_bf16=0)
    assert r["nan"] == 0 and r["rel"] < 1e-5 and r["elem_ratio"] <= 1, r


def test_pingpong_streamed_weights():
    """A 64-column slice whose K = 4000 cannot stay resident: the weight box travels with every A stage."""
    r = G.check_linear(M=64 * 70 + 3, N=64, K=4000)
    assert r["nan"] == 0 and r["rel"] < 3e-3 and r["elem_ratio"] <= 1, r


@pytest.mark.parametrize("kw", [dict(N=300, S=50), dict(N=300, S=64), dict(N=41, S=64, q=224)])
def test_pingpong_additive_pool_segments(kw):
    """Pooling tiles of (64 / seg_len) * seg_len rows: one segment of 50 (14 idle rows) or a whole tile of 64."""
    r = G.check_additive(**kw)
    assert r["fwd_rel"] < 1e-5 and r["fwd_elem_ratio"] <= 1, r
    assert r["dx_rel"] < 3e-3 and r["dW_rel"] < 1e-3 and r["db_rel"] < 1e-3 and r["dq_rel"] < 1e-4, r
