"""gemm_tn's thread-block clusters at their edges, against an fp64 evaluation of the same bf16 operands.

The CTAs of one k-range form a 2 x 2 cluster over (m-tile, n-tile), or 2 x 1 / 1 x 2 when only one tile count is even; each
shares its A chunk along the n-tiles and its B chunk along the m-tiles by TMA multicast.  The output starts as ones (gemm_tn
accumulates), so a tile no cluster wrote, or wrote twice, shows."""
import pytest

import gpu_checks as G

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kw", [
    dict(Kr=1000, Ma=900, Nb=301),            # 8 x 2 tiles: 2 x 2 clusters, Kr % 64 != 0, Nb % 64 != 0
    dict(Kr=64 * 90 + 13, Ma=300, Nb=301, shift=1),   # 3 m-tiles (odd): 1 x 2 clusters, row shift
    dict(Kr=777, Ma=100, Nb=301, shift=-1),   # Ma < 128: one m-tile, 1 x 2
    dict(Kr=2000, Ma=256, Nb=200),            # 2 x 1 tiles: 2 x 1 clusters
    dict(Kr=40, Ma=900, Nb=301),              # one k-chunk in all: a single k-range
    dict(Kr=300, Ma=300, Nb=100),             # 3 x 1 tiles: no cluster
])
def test_gemm_tn_cluster_shapes(kw):
    r = G.check_gemm_tn(**kw)
    assert r["nan"] == 0 and r["rel"] < 1e-5 and r["elem_ratio"] <= 1, r
