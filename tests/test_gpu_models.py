"""Model-level parity of the drop-in packages on the H100 against (a) golden vectors minted from the LIVE
reference modules (tests/golden/*.npz, oracle/make_golden.py) and (b) the oracle.

Tolerances (north_star: "bit-exact for token-ID indexing, within 1e-3 relative for fp32/bf16 activations"):
  * CUDA path vs the oracle evaluated under the SAME bf16 storage contract: logits <= 1e-3 norm-wise;
  * CUDA path vs the reference's own fp32 outputs: the bf16 storage error itself (measured 1e-4 .. 8e-3
    depending on the model, largest for NRMS whose two attention levels amplify rounding) <= 2e-2, and never
    worse than 1.25 x the error of the bf16-contract oracle against the same fp32 reference;
  * every parameter gradient: error against the exact fp32 gradient <= 1.5 x the error the bf16 contract
    itself has (floor 2e-3), and the padding row of the embedding gradient is exactly zero."""
import pytest

import gpu_checks as G

pytestmark = pytest.mark.gpu
CASES = ["nrms", "naml", "naml_f400", "tanr", "lstur_ini", "lstur_con"]
# Norm-wise error of the logits against the fp32 oracle evaluated on bf16-rounded weights / embeddings -- the tolerance
# definition of the blueprint (SURVEY.md 7.3-5), target 1e-3.  NRMS meets it in its default ("accurate") precision mode: V,
# the attention probabilities and the context travel as hi/lo bf16 pairs (the plain bf16 storage of exactly these three is
# what puts the "fast" mode at 6e-3: every token of a title sees the SAME rounding error of V_j, so the pooling does not
# average it out -- DESIGN.md section 4).  NAML / TANR meet it as they are.  LSTUR meets it in ITS default accurate mode: the
# conv output and the news vectors entering the GRU are hi/lo pairs (plain bf16: 1.1e-3 each on the ini case); what is left
# is the bf16 hidden state fed back through the recurrence (5.5e-4).
WEIGHTS_ONLY_BOUND = {"nrms": 1e-3, "naml": 1e-3, "naml_f400": 1e-3, "tanr": 1e-3, "lstur_ini": 1e-3, "lstur_con": 1e-3}


@pytest.mark.parametrize("case", CASES)
def test_golden_case(case):
    r = G.check_golden(case)
    assert r["logits_vs_oracle_bf16"] < 1e-3, r
    assert r["logits_vs_weights_only_oracle"] < WEIGHTS_ONLY_BOUND[case], r
    assert r["logits_vs_reference_fp32"] < 2e-2, r
    assert r["logits_vs_reference_fp32"] < 1.25 * r["oracle_bf16_vs_reference_fp32"] + 1e-4, r
    assert r["worst_grad_ratio_kernel_over_contract"] < 1.5, r
    assert r["emb_row0_grad_zero"], r
    assert not any(k.startswith("missing_grad:") for k in r), r
    if "topic_loss_rel_vs_reference" in r:
        assert r["topic_loss_rel_vs_reference"] < 1e-3, r


def test_nrms_fast_mode_golden_case():
    """config.precision = "fast" (NEWSREC_PRECISION=fast): every activation stored bf16 -- 18 % less time per step, 6e-3 from
    the fp32 oracle on bf16 weights; parity against the oracle under that storage contract stays at 1e-3."""
    r = G.check_golden("nrms", fused=False)
    assert r["logits_vs_oracle_bf16"] < 1e-3, r
    assert r["logits_vs_weights_only_oracle"] < 8e-3, r
    assert r["logits_vs_reference_fp32"] < 1.25 * r["oracle_bf16_vs_reference_fp32"] + 1e-4, r
    assert r["worst_grad_ratio_kernel_over_contract"] < 1.5 and r["emb_row0_grad_zero"], r


@pytest.mark.parametrize("case", ["lstur_ini", "lstur_con"])
def test_lstur_fast_mode_golden_case(case):
    """LSTUR with config.precision = "fast" (plain bf16 conv output / GRU input): parity against the oracle under that contract."""
    r = G.check_golden(case, fused=False)
    assert r["logits_vs_oracle_bf16"] < 1e-3 and r["logits_vs_weights_only_oracle"] < 3e-3, r
    assert r["worst_grad_ratio_kernel_over_contract"] < 1.5 and r["emb_row0_grad_zero"], r


def test_nrms_accurate_mode_golden_case():
    """config.precision = "accurate": V / attention probabilities / context as hi/lo bf16 pairs on the unfused kernels (the
    projection GEMM emits the low plane of V, the title-level attention kernel splits the probabilities and writes both
    context planes) + fp32-accurate user encoder forward.  Meets the blueprint's tolerance: logits within 1e-3 of the fp32
    oracle on bf16-rounded weights / embeddings."""
    r = G.check_golden("nrms", fused="accurate")
    assert r["logits_vs_oracle_bf16"] < 1e-3, r
    assert r["logits_vs_weights_only_oracle"] < 1e-3, r
    assert r["logits_vs_reference_fp32"] < 3.5e-3, r
    assert r["worst_grad_ratio_kernel_over_contract"] < 1.5 and r["emb_row0_grad_zero"], r


@pytest.mark.parametrize("fused", [False, "accurate"])
def test_nrms_mind_shaped_batch_vs_oracle(fused):
    r = G.check_nrms_random(fused=fused)
    assert r["logits_vs_oracle_bf16"] < 1e-3, r
    assert r["logits_vs_exact_fp32"] < 1.25 * r["oracle_bf16_vs_exact"] + 1e-4, r


def test_nrms_in_place_gradient_accumulation_matches_returned_gradients():
    """fp32 red.add order differs between runs, nothing else: the two paths agree to accumulation noise."""
    r = G.check_nrms_direct_grad_accumulation()
    assert r["grads_are_flat_views"], r
    assert r["direct_vs_returned_rel_maxabs"] < 1e-5 and r["after_zero_rel_maxabs"] < 1e-5, r


def test_nrms_prefetched_batch_is_bit_identical():
    r = G.check_nrms_prefetch_equals_direct()
    assert r["maxabs"] == 0.0 and r["maxabs_second"] == 0.0, r


def test_nrms_eval_api_noncontiguous_history():
    r = G.check_nrms_eval_api()
    assert r["user_input_noncontig"] and r["pred_tolist_len"] == 7, r
    assert r["news_vec_rel"] < 1e-3 and r["user_vec_rel"] < 1e-3 and r["pred_rel"] < 1e-5, r


def test_nrms_train_mode_dropout_statistics():
    r = G.check_nrms_train_mode()
    assert r["train_differs_from_eval"] and r["grads_finite"] and r["emb_row0_grad_zero"], r
    assert r["mean_train_vs_eval_rel"] < 0.3, r


@pytest.mark.parametrize("fused", [False, "accurate"])
def test_nrms_train_mode_matches_masked_oracle(fused):
    """The benchmarked configuration (train mode, dropout 0.2), forward and backward, at the eval-mode tolerances
    (fast and accurate kernel sequences: both draw the same masks from the same counter hash)."""
    r = G.check_nrms_train_masked(fused=fused)
    assert r["masks_matter"] > 0.05, r                                   # the masks change the result by far more than any tolerance
    assert r["logits_vs_masked_oracle"] < 1e-3, r                        # same masks, same storage contract
    assert r["logits_vs_masked_exact_fp32"] < 1.25 * r["masked_oracle_vs_masked_exact"] + 1e-4, r
    assert r["worst_grad_ratio_kernel_over_contract"] < 1.5, r           # a wrong backward mask would be off by O(1)
    assert r["emb_row0_grad_zero"], r


@pytest.mark.parametrize("case", ["naml", "naml_f400", "tanr", "lstur_ini", "lstur_con"])
def test_cnn_families_train_mode_match_masked_oracle(case):
    """Train mode of NAML / TANR / LSTUR (both dropout sites of every text encoder, and LSTUR's whole-vector user masking),
    forward and backward, against the oracle under the kernels' own masks."""
    r = G.check_train_masked(case)
    assert r["masks_matter"] > 0.02, r
    assert r["logits_vs_masked_oracle"] < 1e-3, r
    assert r["logits_vs_masked_exact_fp32"] < 1.25 * r["masked_oracle_vs_masked_exact"] + 1e-4, r
    assert r["worst_grad_ratio_kernel_over_contract"] < 1.5, r
    assert not any(k.startswith("missing_grad:") for k in r), r
    if "topic_loss_rel_vs_masked_exact" in r:
        assert r["topic_loss_rel_vs_masked_exact"] < 2e-3, r


def test_nrms_full_size_properties():
    """BASELINE.json configs[1] sizes (batch 512): permutation equivariance and sub-batch consistency hold to fp32
    accumulation-order noise (six titles share one 128-row score tile in the fused front end: which titles are tile mates
    moves a title's keys to other k positions of the P.V MMA; every product with a foreign key is an exact zero)."""
    r = G.check_nrms_full_size_properties()
    assert r["finite"] and r["perm_equivariance_maxabs"] < 2e-6 and r["subbatch_maxabs"] < 2e-6, r


def test_out_of_range_token_id_is_reported():
    import torch
    model, _ = G.nrms_model_and_params(50, 1)
    model.eval()
    ids = torch.randint(1, 50, (4, 20))
    ids[2, 3] = 999
    with torch.no_grad():
        model.get_news_vector({"title": ids})
    with pytest.raises(IndexError):
        model.check_ids()


def test_batched_impression_scoring_matches_per_impression_get_prediction():
    r = G.check_predict_impressions()
    assert r["rel"] < 1e-6 and r["n"] > 1000, r
