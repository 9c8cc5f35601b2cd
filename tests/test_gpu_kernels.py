"""Kernel-level parity on the H100 (every call goes through the C ABI).  Tolerances are written here:
  * integer / byte work (gather, padding layout, operand packing): bit exact;
  * a kernel fed bf16 operands, compared with an fp64 evaluation of the SAME bf16 operands:
      fp32 outputs <= 1e-5 norm-wise, bf16 outputs <= 3e-3 (one bf16 rounding of the result);
  * pooling cores against the oracle under the bf16 storage contract: <= 1e-3 norm-wise
    (the north-star tolerance for activations).
The self-attention core is judged element by element in tests/test_gpu_mhsa_core.py."""
import pytest

import gpu_checks as G

pytestmark = pytest.mark.gpu


def test_operand_prep_and_gather_are_bit_exact():
    r = G.check_prep_and_gather()
    for k in ("cast_pad_exact", "cast_pad_T_exact", "gather_exact", "gather_padded_exact", "bad_id_flag", "dropout_ones_col_intact"):
        assert r[k], (k, r)
    assert abs(r["dropout_keep_rate"] - 0.8) < 0.01, r
    assert r["dropout_scale_err"] < 0.01, r      # kept values are x/(1-p) up to one bf16 rounding


@pytest.mark.parametrize("kw", [dict(M=128, N=64, K=64), dict(M=300, N=900, K=300), dict(M=128 * 9 + 17, N=900, K=300),
                                dict(M=128 * 600 + 5, N=900, K=300)])
def test_tcgen05_linear_bf16_out(kw):
    r = G.check_linear(**kw)
    assert r["nan"] == 0 and r["rel"] < 3e-3 and r["elem_ratio"] <= 1, r


@pytest.mark.parametrize("kw", [
    dict(M=1, N=900, K=300),                # one tile: the peer CTA of the pair works on a phantom (zero-filled) tile
    dict(M=128 * 2 + 1, N=300, K=200),      # odd number of 128-row tiles, two weight slices
    dict(M=128 * 5, N=20, K=300),           # narrower than one 32-column chunk: no TMA-store chunk at all
    dict(M=300, N=33, K=64),                # one full chunk + a 1-column tail through the row-per-thread path
    dict(M=300, N=257, K=300),              # two slices, the second one 16 MMA columns wide
    dict(M=4000, N=240, K=16),              # a single k-step
    dict(M=4000, N=512, K=65),              # K tail of one element in the second k-chunk
])
def test_tcgen05_linear_edge_shapes(kw):
    """CTA-pair scheduling, slice splitting and the TMA-store / row-per-thread boundary at awkward shapes."""
    r = G.check_linear(**kw)
    assert r["nan"] == 0 and r["rel"] < 3e-3 and r["elem_ratio"] <= 1, r


def test_tcgen05_linear_fp32_out_k900():
    r = G.check_linear(M=777, N=300, K=900, out_bf16=0)
    assert r["nan"] == 0 and r["rel"] < 1e-5 and r["elem_ratio"] <= 1, r


@pytest.mark.parametrize("kw", [dict(M=37, N=300, K=300, taps=3, seg=20, relu=1), dict(M=11, N=400, K=300, taps=3, seg=50, relu=1)])
def test_tcgen05_conv3_taps(kw):
    r = G.check_linear(**kw)
    assert r["nan"] == 0 and r["rel"] < 3e-3 and r["elem_ratio"] <= 1, r


@pytest.mark.parametrize("kw", [dict(Kr=64, Ma=128, Nb=64), dict(Kr=1000, Ma=900, Nb=301), dict(Kr=64 * 700 + 13, Ma=200, Nb=301),
                                dict(Kr=900, Ma=300, Nb=301, shift=1), dict(Kr=900, Ma=400, Nb=301, shift=-1)])
def test_tcgen05_weight_grad_gemm(kw):
    r = G.check_gemm_tn(**kw)
    assert r["nan"] == 0 and r["rel"] < 1e-5 and r["elem_ratio"] <= 1, r


def test_tcgen05_matches_simt_triage_backend():
    """Triage builds only (`make -C news-recommendation_b200/csrc TRIAGE=1`): the release library has no second backend."""
    from newsrec_b200 import load_library
    if not load_library().nr_has_triage_backends():
        pytest.skip("release build: SIMT triage backend not compiled in")
    r = G.check_backend_agreement()
    assert r["n_bad"] == 0 and r["tc_rerun_maxabs"] == 0.0 and r["tc_vs_ref_rel"] < 1e-5, r


@pytest.mark.parametrize("kw", [dict(), dict(N=9, S=50), dict(N=50, S=4, D=400), dict(N=1, S=20), dict(N=13, S=32, D=296),
                                dict(N=700, S=20, q=64),
                                # hi/lo input planes (NAML view fusion, Exp1 final attention): news-level and history-level lengths
                                dict(S=20, precision="accurate"), dict(N=9, S=50, precision="accurate")])
def test_additive_attention(kw):
    r = G.check_additive(**kw)
    assert r["fwd_rel"] < 1e-5 and r["fwd_elem_ratio"] <= 1, r
    assert r["dx_rel"] < 3e-3 and r["dW_rel"] < 1e-3 and r["db_rel"] < 1e-3 and r["dq_rel"] < 1e-4, r


def test_dot_product_click_predictor():
    r = G.check_dot_score()
    assert r["fwd_rel"] < 1e-6 and r["dc_rel"] < 1e-6 and r["du_rel"] < 1e-6, r


@pytest.mark.parametrize("kw", [dict(), dict(where="device"), dict(where="pageable"), dict(tail=()), dict(B=1, H=3, Cn=2, tail=(50,)),
                                dict(B=5, H=70, Cn=9, tail=(7,)), dict(B=512, H=50, Cn=5)])
def test_batch_feed_pack_slots(kw):
    """Bit-exact: slot-major (B, ...) int64 tensors -> impression-major id block in one launch (pinned host or device inputs;
    pageable inputs take the staged copy)."""
    r = G.check_pack_slots(**kw)
    assert r["equal"] and r["direct_equal"] and r["B"] == kw.get("B", 37), r
    assert r["direct"] == (kw.get("where", "pinned") != "pageable"), r
