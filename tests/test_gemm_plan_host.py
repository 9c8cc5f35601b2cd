"""The planner regimes of the element-by-element GEMM and pooling tests, without a GPU: every case reaches the regimes its
label names under the planner restatement (tests/gemm_plan_ref.py, on an H100 SXM's 132 SMs), and every regime has a case.
A planner change that moves a case off its regime fails here, before any GPU run."""
import pytest

import gemm_cases as C
import gemm_plan_ref as P


def _nt_plan(c):
    M, rpt, _ = C.linear_shape(c)
    return P.plan_nt(M, c["N"], c["K"], c.get("taps", 1), rpt)


def _tn_plan(c):
    reserve = c.get("reserve", 0)
    return P.plan_tn(c["Kr"], c["Ma"], c["Nb"], reserved=P.H100_SMS if reserve == "all" else reserve)


def _pool_plan(c):
    return P.plan_pool(c["n_seg"] * c["seg"], c["D"], c["q"], c["seg"])


@pytest.mark.parametrize("c", C.LINEAR_CASES, ids=lambda c: c["id"])
def test_linear_case_reaches_its_regimes(c):
    got = P.regimes_nt(_nt_plan(c))
    assert set(c["regimes"]) <= got, (c["id"], sorted(got))


@pytest.mark.parametrize("c", C.GEMM_TN_CASES, ids=lambda c: c["id"])
def test_gemm_tn_case_reaches_its_regimes(c):
    got = P.regimes_tn(_tn_plan(c))
    assert set(c["regimes"]) <= got, (c["id"], sorted(got))


@pytest.mark.parametrize("c", C.POOL_CASES, ids=lambda c: c["id"])
def test_pool_case_reaches_its_regimes(c):
    p = _pool_plan(c)
    assert p["n_slices"] == 1  # gemm_additive_pool refuses a second weight slice
    got = P.regimes_nt(p)
    assert set(c["regimes"]) <= got, (c["id"], sorted(got))


@pytest.mark.parametrize("c", C.POOL_BWD_CASES, ids=lambda c: c["id"])
def test_pool_bwd_case_reaches_its_regimes(c):
    p = P.plan_pool_bwd(c["n_seg"], c["seg"], c["D"], c["q"])
    assert p["dpre"]["n_slices"] == 1  # the dPre GEMM reduces each row over the whole query width: one weight slice
    got = P.regimes_bwd(p)
    assert set(c["regimes"]) <= got, (c["id"], sorted(got))


def test_every_pool_bwd_regime_has_a_case():
    bwd = set().union(*(set(c["regimes"]) for c in C.POOL_BWD_CASES))
    assert set(P.BWD_REGIMES) <= bwd, sorted(set(P.BWD_REGIMES) - bwd)
    prefixed = {"dPre " + r for r in P.NT_REGIMES} | {"dX " + r for r in P.NT_REGIMES}
    assert bwd <= set(P.BWD_REGIMES) | prefixed, sorted(bwd - set(P.BWD_REGIMES) - prefixed)
    ids = [c["id"] for c in C.POOL_BWD_CASES]
    assert len(ids) == len(set(ids))


def test_pool_bwd_plans_the_comments_name():
    """The dX slice widths the staging cap gives at seg_len 1 to 4 (gemm_pool_dinput), and the weight-gradient split."""
    assert [P.pool_dinput_max_stride(s) for s in (1, 2, 3, 4, 20, 64)] == [16, 32, 64, 80, 304, 512]
    p = P.plan_pool_bwd(1000, 1, 300, 200)
    assert (p["dx"]["n_stride"], p["dx"]["n_slices"]) == (16, 19)
    assert P.plan_pool_bwd(1000, 4, 400, 200)["dx"]["n_stride"] == 80
    assert P.plan_pool_bwd(3000, 20, 300, 200)["dx"]["n_stride"] == 160       # not capped: the 256-column box limit rules
    # D = 604: columns [0, 512) and [512, 605), the bias column at column 92 of the second launch
    assert [(w["NT"], w["n_tiles"]) for w in P.plan_pool_bwd(100, 20, 604, 200)["wgrad"]] == [(256, 2), (128, 1)]
    assert len(P.plan_pool_bwd(100, 20, 511, 200)["wgrad"]) == 1 and len(P.plan_pool_bwd(100, 20, 512, 200)["wgrad"]) == 2


def _align256(x):
    return (x + 255) // 256 * 256


def pool_bwd_workspace_layout(n_seg, seg_len, q):
    """nr_additive_attention_bwd's workspace: dscore fp32 [rows] at 0, dPre bf16 [rows][round_up(q, 16)] at the next 256-byte
    boundary, 256 bytes of slack.  Returns (dPre offset, total bytes)."""
    rows = n_seg * seg_len
    off = _align256(4 * rows)
    return off, off + _align256(2 * rows * P._round_up(q, 16)) + 256


@pytest.mark.parametrize("n_seg,seg,q", [(0, 20, 200), (1, 1, 1), (1, 20, 200), (37, 20, 200), (3000, 20, 200), (777, 2, 16),
                                         (5000, 3, 24), (50, 30, 256), (13, 7, 17), (100, 64, 100)])
def test_pool_bwd_workspace_layout(n_seg, seg, q):
    import os

    import newsrec_b200
    if not os.path.exists(newsrec_b200.LIB_PATH):
        pytest.skip("library not built (python __graft_entry__.py build)")
    lib = newsrec_b200.load_library()
    assert lib.nr_additive_attention_bwd_workspace(n_seg, seg, q) == pool_bwd_workspace_layout(n_seg, seg, q)[1]


def test_every_regime_has_a_case():
    nt = set().union(*(set(c["regimes"]) for c in C.LINEAR_CASES))
    tn = set().union(*(set(c["regimes"]) for c in C.GEMM_TN_CASES))
    assert nt == set(P.NT_REGIMES), sorted(set(P.NT_REGIMES) - nt)
    assert tn == set(P.TN_REGIMES), sorted(set(P.TN_REGIMES) - tn)
    ids = [c["id"] for c in C.LINEAR_CASES + C.GEMM_TN_CASES + C.POOL_CASES + C.POOL_BWD_CASES]
    assert len(ids) == len(set(ids))


def test_the_shapes_the_planner_comments_name():
    """Shapes whose plans the kernels' comments and the case labels rely on."""
    p = P.plan_nt(64 * 27, 900, 300)
    assert (p["n_slices"], p["n_stride"], p["grid"]) == (5, 192, 130)        # 5 slices of 192 columns, 26 groups
    p = P.plan_nt(4000, 400, 300)
    assert (p["n_stride"], p["n_box"]) == (144, 160)                        # slice 0's last 32-column chunk is cut
    assert P.plan_nt(4000, 256, 1000)["stages"] == 5
    assert P.plan_nt(4000, 64, 4000)["b_stream"] and P.plan_nt(4000, 300, 2000)["b_stream"]
    assert P.plan_pool(1000, 400, 200, 20)["b_stream"]                      # NAML's pooling at F = 400
    assert not P.plan_pool(1000, 300, 200, 20)["b_stream"]
    assert P.plan_pool(1000, 300, 200, 20)["rows_per_tile"] == 60
    t = P.plan_tn(1000, 900, 301)
    assert (t["m_tiles"], t["n_tiles"], t["NT"], t["cluster"]) == (8, 2, 192, (2, 2))
    # every SM reserved: the GEMM keeps half of them
    assert P.plan_tn(64 * 700 + 13, 300, 100, reserved=P.H100_SMS)["k_slices_max"] == P.plan_tn(64 * 700 + 13, 300, 100, sms=66)["k_slices_max"]


def test_schedule_covers_every_tile_once():
    """The (CTA, warpgroup) tile lists of a plan cover each (tile, slice) pair exactly once."""
    for M, N, K, rpt in [(64 * 53 + 5, 900, 300, 64), (4000, 400, 300, 64), (999, 900, 300, 60), (1, 900, 300, 64)]:
        p = P.plan_nt(M, N, K, 1, rpt)
        seen = [(t, p["slice_of"][b]) for b, (w0, w1) in enumerate(p["wg_tiles"]) for t in w0 + w1]
        assert sorted(seen) == [(t, s) for t in range(p["num_m_tiles"]) for s in range(p["n_slices"])]
