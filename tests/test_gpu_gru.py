"""The LSTUR GRU (nr_gru_fwd / _bwd) called through the C ABI on both recurrence paths -- the persistent kernel (one cooperative
launch: 128-row user tiles x 32-unit slices, a release/acquire step counter per row tile) and the per-step sequence (a GEMM
and a gate kernel per step), chosen with nr_debug_set_gru_stepwise -- and compared stage by stage, per element, with fp64
references built from what the kernels themselves stored (tests/gpu_checks.py check_gru_stages).  Every "=" output starts as
NaN, dWih_ext / dWhh_ext with a small pattern, the workspace with 0xFF; every buffer, the read-only operands included, is
followed by a guard; after every call the device watchdog record is clean.

Bounds (u = 2^-24 is the fp32 unit roundoff; bf16 keeps 8 significant bits, so round to nearest is within half an ulp):
  * bit exact: xb = bf16_rn(x) with the ones column at D and zeros up to ldd, x_lo = bf16_rn(x - xb) with zeros from D on;
    hs[0] = h0; hb[t] = bf16_rn(hs[t]) with the ones column at Hd and zeros up to ldh, for t = 0 .. S (the persistent kernel
    writes the ones column and the zeros from its last slice only); out = hs[S]; frozen rows (t >= max(len, 1)) of hs[t+1]
    equal hs[t].
  * gi and every gh[t]: fp32 sums of exact bf16 x bf16 products, within 1e-6 sum |x||w| (with |b|) of the fp64 product of the
    stored operands plus the bias (the Q|K|V convention of test_gpu_mhsa_encoder.py).  In accurate mode gi includes x_lo W^T;
    a reference without it misses the bound by >= 8x.
  * hs[t+1] on active rows, from the stored gi, gh[t], hs[t] (gpu_checks.gru_gate_errors).  Figures: ex2.approx.f32 and
    div.approx.f32 (__fdividef, divisor in [2^-126, 2^126]) are within 2 ulp, at most 2^-22 relative (PTX ISA; the CUDA C++
    Programming Guide's intrinsic-function table), every other fp32 operation within u.
      sigmoid(a) = 1 / (1 + ex2(-a log2e)): a = gi + gh is one fp32 sum, the constant and the product one rounding each, so
        the exponent carries 3u|a| relatively, and ex2 adds 2^-22; 1 + e is one rounding and the division 2^-22.  Since
        d(1 + e)/(1 + e) = (1 - s) de/e, |ds| <= s [(1 - s)(3u|a| + 2^-22) + u + 2^-22].
      tanh(v) = 1 - 2 / (ex2(2 log2e v) + 1): v = gi_n + r gh_n carries |gh_n| dr + u|r gh_n| + u|v| (FMA or not), and dn =
        (1 - n^2) dv; the exponent carries 4u|v| (2 log2e ln2 = 2), ex2 2^-22, and q = 2 / (e + 1) moves by
        q e/(1+e) = (1 - n^2)/2 times that, plus q (u + 2^-22) for the sum and the division, plus u|n| for 1 - q.
      h' = (1 - z) n + z h: |h - n| dz + (1 - z) dn + 3u ((1 - z)|n| + z|h|).
    2^-100 is added to every bound for flush-to-zero below 2^-126.  A reference that adds b_hn outside r (the cuDNN GRU)
    misses the bound by >= 8x.
  * backward, per (t, b): the dh entering step t is rebuilt in fp64 from dout, the gates and the kernels' own stored bf16
    dgh[t+1]: dh_{t-1} = dh_t z_t + dgh[t] W_hh (frozen rows: dh_t).  Its distance A_t from the kernels' fp32 dh obeys
    A_{t-1} = z A_t + |dh| dz + u|dh z| + 1e-6 sum |dgh||w| + u|dh_{t-1}| (frozen rows pass A_t on exactly: dgh = 0 gives a
    GEMM result of exactly 0), A_{S-1} = 0.  dgi and dgh are then judged within half a bf16 ulp plus the first-order error of
    dn = dh (1 - z), dpn = dn (1 - n^2), dz = dh (h - n), dpz = dz z (1 - z), dpr = dpn gh_n r (1 - r), dgh_n = dpn r from A,
    the gate errors above and 2-4u of rounding per product chain.  At t = len - 1 < S - 1 the rebuilt dh is dout itself (so
    A = 0 there); frozen steps are exactly 0; the pad columns [3Hd, ldb) are 0.  A reference with dgh_n = dpn misses by
    >= 8x.  dh0 is bit-equal to dh_direct + dh_rec as the workspace holds them and within A_{-1} of fp64.
  * dx from the stored dgi: 1e-6 sum |dgi||w|, exactly 0 on frozen steps.
  * dWih_ext / dWhh_ext, per element against the pattern + dg^T [X | 1] of the stored operands: the split-K GEMM sums B S
    products per element as ceil(B S / 64) chunks of four k16 tensor-core steps, then adds the k-range partials onto the
    pattern with fp32 atomics.  Taking each step as adding at most 2 ulp (2^-22) of the magnitude summed so far, any split
    is within 2^-22 (5 ceil(B S / 64) + 1) (|pattern| + sum |dg||x|).  The pitch columns keep the pattern bit for bit.
  * end to end, per row: kernel error against the exact fp64 GRU <= 1.5 x the error of the bf16 storage contract (x and h as
    bf16 operands -- x as a hi/lo pair into gi in accurate mode -- dgi, dgh stored in bf16, the weight gradient on the bf16 x
    rows), the contract's error floored at 2e-3 of the row's norm: out, dx, dh0, dWih_ext, dWhh_ext (bias columns included).
  * which path ran, by launch count: 3 (+ 2 in accurate mode) conversions and GEMMs, then 1 persistent launch whatever S,
    or 2 per step; a second forward is bit-identical in all saved state.  Whether the two paths agree bit for bit is
    recorded, not asserted: the two gate codes may contract different FMAs.

SM-dependent shapes come from nr_num_sms()."""
import pytest

import gpu_checks as G

pytestmark = pytest.mark.gpu

BOTH = ("persistent", "stepwise")
BENCH = dict(B=512, S=50, D=900, Hd=900)


def _sms():
    from newsrec_b200 import load_library
    return int(load_library().nr_num_sms())


def assert_gru(r, S, accurate=True, discriminate=True, e2e_grads=True, open_rows=()):
    print({p: {k: v for k, v in m.items() if k.endswith(("ratio", "_ek", "_ec", "launches")) or v is False} for p, m in r["paths"].items()},
          "paths bit-identical:", r.get("paths_bit_identical"))
    for path, m in r["paths"].items():
        ctx = (path, m)
        assert m["fwd_device_error"][0] == 0 and m["bwd_device_error"][0] == 0, ctx
        assert m["guards_intact"] and m["fwd_outputs_finite"] and m["bwd_outputs_finite"], ctx
        persistent = {"persistent": True, "stepwise": False, "default": r["persistent_supported"]}[path]
        assert not persistent or r["persistent_supported"], ctx
        assert m["fwd_launches"] == (5 if accurate else 3) + (1 if persistent else 2 * S), ctx
        assert m["xb_mismatch_rows"] == 0 and m.get("xlo_mismatch_rows", 0) == 0, ctx
        assert m["hs0_exact"] and m["hb_mismatch_rows"] == 0 and m["out_equals_hs_S"] and m["hs_frozen_rows_exact"], ctx
        assert m["gi_ratio"] <= 1.0 and m["gh_ratio"] <= 1.0 and m["hs_ratio"] <= 1.0, ctx
        assert m["workspace_bytes_match"] and m["dg_pad_cols_zero"] and m["dg_frozen_zero"], ctx
        assert m["dh_at_last_active_step_is_dout"] and m["dh0_equals_workspace_sum"], ctx
        assert m["dg_ratio"] <= 1.0 and m["dh0_ratio"] <= 1.0 and m["dx_ratio"] <= 1.0 and m["dx_frozen_zero"], ctx
        assert m["dWih_elem_ratio"] <= 1.0 and m["dWhh_elem_ratio"] <= 1.0, ctx
        assert m["dWih_pitch_cols_untouched"] and m["dWhh_pitch_cols_untouched"], ctx
        for k in ("out", "dx", "dh0", "dWih", "dWhh") if e2e_grads else ("out",):
            if k not in open_rows:  # open_rows: recorded as strict xfails below
                assert m[k + "_row_ratio"] <= 1.5, (k, ctx)
        if discriminate:
            assert m["hs_bhn_outside_r_ratio"] >= 8.0 and m["dgh_n_without_r_ratio"] >= 8.0, ctx
            if accurate:
                assert m["gi_no_lo_ratio"] >= 8.0, ctx
        assert m["fwd_deterministic"], ctx


# ---- persistent shapes, each on both paths -------------------------------------------------------
@pytest.mark.parametrize("accurate", [True, False])
def test_gru_bench_ini_shape(accurate):
    """bench.py's LSTUR ini user encoder: 512 users x 50 steps, D = Hd = 900 (4 row tiles x 29 slices, the last of 4 units;
    15 k-chunks, the last partial)."""
    r = G.check_gru_stages(**BENCH, accurate=accurate, paths=BOTH, seed=3)
    assert r["persistent_supported"], r
    assert_gru(r, 50, accurate)


@pytest.mark.parametrize("Hd", [32, 36, 64, 96, 1024])
def test_gru_persistent_hidden_sizes(Hd):
    """One slice (32), a last slice of 4 units (36), one and two k-chunks (64, 96), and 16 resident k-chunks (1024: 231,424
    bytes of shared memory)."""
    r = G.check_gru_stages(B=129, S=7, D=72, Hd=Hd, paths=BOTH, seed=100 + Hd)
    assert r["persistent_supported"], r
    assert_gru(r, 7)


@pytest.mark.parametrize("which", ["1", "127", "128", "129", "max"])
def test_gru_persistent_row_tiles(which):
    """Partial and full 128-row tiles (a partial tile's TMA reads rows of the next step that no stored row may depend on) and
    the largest batch the cooperative launch holds at Hd = 96: 128 floor(SMs / 3)."""
    B = 128 * (_sms() // 3) if which == "max" else int(which)
    r = G.check_gru_stages(B=B, S=5, D=64, Hd=96, paths=BOTH, seed=200 + B)
    assert r["persistent_supported"], r
    assert_gru(r, 5, open_rows=("dWhh",) if B == 1 else ())


def test_gru_persistent_one_row_tile_per_sm():
    """Hd = 32 at B = 128 SMs: every SM holds a row tile with its own step counter.  This case found the gate warps starting
    their first wgmma before the resident W_hh slice had landed (nothing waited on its barrier): whole row tiles of gh[0]
    were wrong and a second forward differed."""
    B = 128 * _sms()
    r = G.check_gru_stages(B=B, S=3, D=32, Hd=32, paths=BOTH, seed=300)
    assert r["persistent_supported"], r
    assert_gru(r, 3)


@pytest.mark.parametrize("S,Hd", [(1, 128), (2, 128), (64, 128), (200, 128), (2, 64), (200, 64)])
def test_gru_persistent_step_counts(S, Hd):
    """S = 1 (no step barrier), 2, 64, 200; two k-chunks per step (Hd = 128: the 2-stage ring returns to the same phase every
    step) and one (Hd = 64: the phase alternates, as with the bench shape's 15)."""
    r = G.check_gru_stages(B=129, S=S, D=64, Hd=Hd, paths=BOTH, seed=400 + S + Hd)
    assert r["persistent_supported"], r
    assert_gru(r, S, open_rows=("dx", "dh0") if S >= 64 else ())


# ---- shapes only the per-step sequence runs ---------------------------------------------------
@pytest.mark.parametrize("which", ["con", "hd8", "hd1028", "over_limit", "b2000"])
def test_gru_stepwise_shapes(which):
    """bench.py's LSTUR con user encoder (Hd = 450 is not a multiple of 4, h0 = 0), the smallest shape (Hd = D = 8), Hd = 1028
    (17 k-chunks do not fit), one batch row above what the cooperative launch holds at Hd = 900, and B = 2000 at Hd = 450."""
    kw = {"con": dict(B=512, S=50, D=900, Hd=450, h0_zero=True), "hd8": dict(B=37, S=9, D=8, Hd=8),
          "hd1028": dict(B=64, S=4, D=64, Hd=1028), "over_limit": dict(B=128 * (_sms() // 29) + 1, S=6, D=96, Hd=900),
          "b2000": dict(B=2000, S=5, D=64, Hd=450)}[which]
    r = G.check_gru_stages(**kw, seed=500 + len(which))
    assert not r["persistent_supported"], r
    assert_gru(r, kw["S"])


# ---- input variants -----------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["perm", "col2", "slice"])
def test_gru_input_layouts(layout):
    """x as an [S][B][D] permuted view, with column stride 2, and as a slice with s_b > S D (the storage around it is NaN)."""
    r = G.check_gru_stages(B=129, S=9, D=96, Hd=96, x_layout=layout, seed=600)
    assert_gru(r, 9)


def test_gru_saturated_gates():
    """Weights and biases scaled 40x: gate pre-activations beyond |10|, no NaN, every stage bound still met.  The gradient rows
    are not held to the end-to-end rule here: with saturated gates they are sums that cancel to a few percent of their terms,
    and an fp32 evaluation of the bf16 contract itself lands up to 2x the contract's error from fp64 (measured with an fp32
    torch restatement of the kernels); the per-stage bounds judge the kernels on their own inputs instead."""
    r = G.check_gru_stages(B=129, S=9, D=64, Hd=64, wscale=40.0, paths=BOTH, seed=700)
    assert all(m["max_preact"] >= 10.0 for m in r["paths"].values()), r
    assert_gru(r, 9, discriminate=False, e2e_grads=False)


@pytest.mark.parametrize("path", BOTH)
def test_gru_empty_batch_launches_nothing(path):
    r = G.check_gru_stages(B=0, S=5, D=64, Hd=96, paths=(path,))
    m = r["paths"][path]
    assert m["fwd_launches"] == 0 and m["bwd_launches"] == 0 and m["guards_intact"], r


# ---- the contract --------------------------------------------------------------------------
def test_gru_persistent_predicate_matches_the_header():
    """nr_gru_persistent_supported is the rule include/newsrec_b200.h states: B >= 1, Hd % 4 == 0, 32 <= Hd <= 1024 and
    ceil(B / 128) ceil(Hd / 32) <= SMs."""
    from newsrec_b200 import load_library
    lib = load_library()
    sms = _sms()
    bad = []
    for Hd in (8, 28, 30, 32, 34, 36, 64, 450, 900, 960, 964, 1020, 1022, 1024, 1028, 1056, 2048):
        for B in (0, 1, 127, 128, 129, 512, 513, 128 * sms, 128 * sms + 1, 128 * (sms // 29), 128 * (sms // 29) + 1):
            rule = B >= 1 and Hd % 4 == 0 and 32 <= Hd <= 1024 and -(-B // 128) * -(-Hd // 32) <= sms
            if bool(lib.nr_gru_persistent_supported(B, Hd)) != rule:
                bad.append((B, Hd, rule))
    assert not bad, bad


@pytest.mark.parametrize("kw", [dict(B=37, S=50), dict(B=300, S=50), dict(B=5, S=7, D=600, Hd=900), dict(B=9, S=12, D=900, Hd=450),
                                dict(B=700, S=6)])
def test_gru_last_hidden_history_50_mixed_lengths(kw):
    """History 50 at D = Hd = 900 in fast mode: the persistent kernel at B <= 128 floor(SMs / 29), the per-step sequence at
    B = 700 (more CTAs than SMs) and Hd = 450 (not a multiple of 4)."""
    kw = dict(dict(D=900, Hd=900), **kw)
    r = G.check_gru_stages(**kw, accurate=False, seed=3)
    assert r["persistent_supported"] == (-(-kw["B"] // 128) * 29 <= _sms() and kw["Hd"] % 4 == 0), r
    assert_gru(r, kw["S"], accurate=False, open_rows=("dWih", "dWhh") if kw["B"] * kw["S"] < 200 else ())
    for path, m in r["paths"].items():  # and what the whole-tensor check of these shapes asserted against the bf16 contract
        assert m["out_tensor_rel_vs_contract"] < 1e-3, (path, m)
        assert all(m[k + "_tensor_rel_vs_contract"] < 5e-3 for k in ("dx", "dh0", "dWih", "dWhh")), (path, m)


def test_gru_autograd_function_rows():
    """GruLastHiddenFn, the model's entry (operand cache, dW_ext split into weight and bias gradients), end to end per row."""
    r = G.check_gru_autograd(B=37, S=50, D=900, Hd=900, accurate=True)
    for k in ("out", "dx", "dh0", "dWih", "dWhh"):
        assert r[k + "_row_ratio"] <= 1.5, (k, r)


# ---- open findings of the end-to-end row rule: every stage bound of these cases holds; the rows below do not -------------
@pytest.mark.xfail(strict=True, reason="open finding: on an H100 80GB HBM3 (400 W), measured on both paths: B = 1, S = 5 (Hd = 96): "
                                      "dWhh_ext row ratio 1.76 (kernel 4.5e-3, contract 2.5e-3); B = 5, S = 7: dWih_ext 1.81 "
                                      "(4.4e-3 / 2.5e-3), dWhh_ext 1.63; B = 9, S = 12 (Hd = 450): dWih_ext 1.56, dWhh_ext 1.50. "
                                      "Rows of few (5-108) products, where one bf16 rounding of dgi or dgh that falls the other way "
                                      "moves the row by more than the contract's own error")
@pytest.mark.parametrize("kw", [dict(B=1, S=5, D=64, Hd=96, accurate=True, seed=201),
                                dict(B=5, S=7, D=600, Hd=900, accurate=False, seed=3),
                                dict(B=9, S=12, D=900, Hd=450, accurate=False, seed=3)])
def test_gru_weight_gradient_rows_of_short_sums(kw):
    r = G.check_gru_stages(**kw)
    assert all(m["dWih_row_ratio"] <= 1.5 and m["dWhh_row_ratio"] <= 1.5 for m in r["paths"].values()), r


@pytest.mark.xfail(strict=True, reason="open finding: on an H100 80GB HBM3 (400 W), at B = 129 measured on both paths: S = 64, "
                                      "Hd = 128: dx row ratio 1.66 (kernel 3.4e-3, contract 2.0e-3); S = 200, Hd = 128: dx 4.1-4.4, "
                                      "dh0 3.9-4.5; S = 200, Hd = 64: dx 7.9 (3.0e-2 / 3.8e-3), dh0 3.1.  Every per-step bound "
                                      "(dgi, dgh, the rebuilt dh, dh0, dx from the stored dgi) holds: the kernels' fp32 chain and the "
                                      "fp64 contract drift apart over long recurrences")
@pytest.mark.parametrize("S,Hd", [(64, 128), (200, 128), (200, 64)])
def test_gru_input_gradient_rows_of_long_recurrences(S, Hd):
    r = G.check_gru_stages(B=129, S=S, D=64, Hd=Hd, seed=400 + S + Hd)
    assert all(m["dx_row_ratio"] <= 1.5 and m["dh0_row_ratio"] <= 1.5 for m in r["paths"].values()), r
