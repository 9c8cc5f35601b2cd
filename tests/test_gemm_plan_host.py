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


# ------------------------------------------------------------------------------------------------
# gemm_store's options and store paths (tests/test_gpu_gemm_store.py)
# ------------------------------------------------------------------------------------------------
def _store_plan(c):
    s = C.store_setup(c)
    return P.plan_nt(s["M"], c["N"], c["K"], c.get("taps", 1), s["rpt"]), s


def _store_paths(c):
    plan, s = _store_plan(c)
    out, lo = P.store_paths(plan, c.get("out_bf16", 1), c.get("rm") is not None, s["lo_col0"])
    return out | {"lo " + x for x in lo}


@pytest.mark.parametrize("c", C.STORE_CASES, ids=lambda c: c["id"])
def test_store_case_labels(c):
    """A case sets exactly the options it names, and its plan reaches the NT regimes and takes exactly the store paths it names."""
    assert set(c["options"]) == C.store_options(c), (c["id"], sorted(C.store_options(c)))
    assert set(c["options"]) <= set(P.STORE_OPTIONS)
    plan, s = _store_plan(c)
    got = P.regimes_nt(plan)
    assert set(c["regimes"]) <= got, (c["id"], sorted(got))
    assert set(c["paths"]) == _store_paths(c), (c["id"], sorted(_store_paths(c)))
    if s["lo_col0"] is not None:  # gemm_store accepts the case's low plane
        assert P.lo_chunk_aligned(plan, s["lo_col0"]) and (P.store_use_tma(c["N"], 1, c.get("rm"), s["rpt"]) or s["lo_col0"] % 8 == 0)


def test_every_store_option_path_pair_has_a_case():
    """Every (option, path) pair gemm_store accepts is reached by a case (the low plane by the paths of the plane itself)."""
    want = {(o, p) for o in P.STORE_OPTIONS for p in P.STORE_PATHS if P.store_accepts(o, p)}
    have = set()
    for c in C.STORE_CASES:
        paths = _store_paths(c)
        for o in c["options"]:
            have |= {(o, p[3:]) for p in paths if p.startswith("lo ")} if o == "low plane" else {(o, p) for p in paths if p in P.STORE_PATHS}
    assert want <= have, sorted(want - have)
    assert have <= want, sorted(have - want)
    ids = [c["id"] for c in C.STORE_CASES]
    assert len(ids) == len(set(ids))


def test_store_case_table_reaches_the_edges():
    """The slice edges and production shapes the table exists for: a slice width of 16 mod 32, N < 32, an odd fp32 tail, M = 1,
    M not a multiple of 64, rows_per_tile 1 and 50, dropout at p = 0.2 and 0.5 on both output types with and without a row
    map, taps 2 and 4 at tap_origin 0 and taps - 1, the low plane from column 0 and from a chunk boundary inside slice 1."""
    cases = C.STORE_CASES
    setups = [C.store_setup(c) for c in cases]
    plans = [_store_plan(c)[0] for c in cases]
    assert any(p["n_stride"] % 32 == 16 for p in plans)
    assert any(c["N"] < 32 for c in cases) and any(c.get("out_bf16", 1) == 0 and c["N"] % 2 for c in cases)
    assert any(s["M"] == 1 for s in setups) and any(s["M"] % 64 for s in setups)
    assert {1, 50} <= {s["rpt"] for s in setups}
    for p in (0.2, 0.5):
        assert {(c.get("out_bf16", 1), c.get("rm") is not None) for c in cases if c.get("p") == p} >= {(0, False), (1, False), (1, True)} \
            if p == 0.2 else {(0, False), (0, True), (1, False)}, p
    for taps in (2, 4):
        assert {0, taps - 1} <= {c.get("tap_origin") for c in cases if c.get("taps") == taps}, taps
    lo = {(c["N"], c["K"], C.store_setup(c)["lo_col0"]) for c in cases if c.get("lo_col0") is not None}
    assert any(l0 == 0 for _, _, l0 in lo)
    assert any(P.plan_nt(1, N, K)["n_stride"] < l0 < 2 * P.plan_nt(1, N, K)["n_stride"] for N, K, l0 in lo)
    assert any(c.get("dtanh") and c["N"] % 2 for c in cases)
    assert any(c.get("relu") and c.get("p") for c in cases)


@pytest.mark.parametrize("heads,supported", [(1, 0), (2, 0), (3, 1), (7, 1), (14, 1), (15, 1)])
def test_lo_supported_matches_the_accurate_mhsa_head_counts(heads, supported):
    """nr_mhsa_accurate_supported reaches the low-plane rule through gemm_store_lo_supported(3 sec, d, 2 sec), sec = round_up(d, 8):
    at d_k = 20 the V section starts inside a 32-column chunk of the Q|K|V projection at 1 and 2 heads only."""
    d = 20 * heads
    sec = (d + 7) // 8 * 8
    assert P.lo_supported(3 * sec, d, 2 * sec) == bool(supported)
