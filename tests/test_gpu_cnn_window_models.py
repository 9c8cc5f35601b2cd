"""The drop-in NAML, TANR, LSTUR and Hi-Fi Ark at conv windows other than 3, on the H100, against the window golden cases minted
from the live reference (oracle/make_golden_cnn_window.py) and the oracle, with the bounds of
tests/test_gpu_models.py::test_golden_case:
  * logits within 1e-3 (norm-wise) of the oracle under the bf16 storage contract and of the fp32 oracle on bf16-rounded weights;
  * against the reference's own fp32 logits, no more than 1.25 x the error of the bf16-contract oracle + 1e-4;
  * every parameter gradient: error against the exact fp32 gradient <= 1.5 x the bf16 contract's (floor 2e-3);
  * the padding row of the embedding gradient exactly zero; TANR's topic loss within 1e-3 of the reference's."""
import functools

import pytest
import torch

import cnn_window_util as CW
import gpu_checks as G
import hifiark_oracle as HO
import newsrec_oracle as O
from golden_util import load_case, unique_params

pytestmark = pytest.mark.gpu
DEV = G.DEV


def check_window_golden(case):
    """gpu_checks.check_golden on a window case, in the family's shipped precision mode (LSTUR: accurate, Y_lo)."""
    family = CW.WINDOW_CASES[case][0]
    fused = G.default_nrms_mode("LSTUR") if family.startswith("lstur") else False
    g = load_case(case)
    tw = lambda t: (0.1 * t if t is not None else 0.0)
    p_b = CW.case_params(case, g)
    logits_b, topic_b = CW.oracle_forward(case, g, p_b, O.BF16, bool(fused))
    (O.click_loss(logits_b) + tw(topic_b)).backward()
    p_x = CW.case_params(case, g)
    logits_x, topic_x = CW.oracle_forward(case, g, p_x, O.EXACT)
    (O.click_loss(logits_x) + tw(topic_x)).backward()
    model = CW.build_model(case, DEV, fused=fused)
    model.load_state_dict(CW.state_dict(case, g))
    model.eval()
    cand, clicked = G.golden_inputs(case, g)
    if family.startswith("lstur"):
        out = model(torch.from_numpy(g["user"]), torch.from_numpy(g["clicked_news_length"]).clone(), cand, clicked)
    else:
        out = model(cand, clicked)
    logits, topic = (out if isinstance(out, tuple) else (out, None))
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long, device=DEV))
    (loss + tw(topic)).backward()
    torch.cuda.synchronize()
    with torch.no_grad():
        logits_w, _ = CW.oracle_forward(case, g, CW.case_params(case, g, requires_grad=False), O.WEIGHTS_BF16)
    res = {"logits_vs_oracle_bf16": G.relerr(logits, logits_b), "logits_vs_reference_fp32": G.relerr(logits, torch.from_numpy(g["logits"])),
           "logits_vs_weights_only_oracle": G.relerr(logits, logits_w),
           "oracle_bf16_vs_reference_fp32": G.relerr(logits_b, torch.from_numpy(g["logits"]))}
    if topic is not None:
        res["topic_loss_rel_vs_reference"] = abs(topic.item() - float(g["topic_loss"])) / abs(float(g["topic_loss"]))
    grads = dict(model.named_parameters())
    gscale = max(float(v.grad.norm()) for v in unique_params(p_x).values())
    worst_ratio, worst_key = 0.0, ""
    for k, prm in unique_params(p_x).items():
        if grads[k].grad is None:
            res["missing_grad:" + k] = True
            continue
        if prm.grad.norm() < 1e-4 * gscale:
            continue
        e_kernel = G.relerr(grads[k].grad, prm.grad)
        e_contract = G.relerr(unique_params(p_b)[k].grad, prm.grad)
        ratio = e_kernel / max(e_contract, 2e-3)
        if ratio > worst_ratio:
            worst_ratio, worst_key = ratio, k
    res["worst_grad_ratio_kernel_over_contract"], res["worst_grad_key"] = worst_ratio, worst_key
    w = grads.get("news_encoder.word_embedding.weight", grads.get("news_encoder.text_encoders.title.word_embedding.weight"))
    res["emb_row0_grad_zero"] = bool((w.grad[0] == 0).all())
    return res


@pytest.mark.parametrize("case", ["naml_w4", "tanr_w1", "lstur_ini_w2"])
def test_window_golden_case(case):
    r = check_window_golden(case)
    print(case, r)
    assert r["logits_vs_oracle_bf16"] < 1e-3, r
    assert r["logits_vs_weights_only_oracle"] < 1e-3, r
    assert r["logits_vs_reference_fp32"] < 1.25 * r["oracle_bf16_vs_reference_fp32"] + 1e-4, r
    assert r["worst_grad_ratio_kernel_over_contract"] < 1.5, r
    assert r["emb_row0_grad_zero"], r
    assert not any(k.startswith("missing_grad:") for k in r), r
    if "topic_loss_rel_vs_reference" in r:
        assert r["topic_loss_rel_vs_reference"] < 1e-3, r


@functools.lru_cache(maxsize=None)
def hifiark_window_2_golden():
    """tests/test_gpu_hifiark.py::test_golden_case (eval mode) on hifiark_w2."""
    case = "hifiark_w2"
    g = load_case(case)
    model = CW.build_model(case, DEV)
    model.load_state_dict(CW.state_dict(case, g))
    model.eval()
    ct, ht = torch.from_numpy(g["cand_title"]), torch.from_numpy(g["clicked_title"])
    p_b, p_x = CW.case_params(case, g), CW.case_params(case, g)
    lb = HO.hifiark_forward(ct, ht, p_b, O.BF16)[0]
    O.click_loss(lb).backward()
    lx = HO.hifiark_forward(ct, ht, p_x, O.EXACT)[0]
    O.click_loss(lx).backward()
    with torch.no_grad():
        lw = HO.hifiark_forward(ct, ht, CW.case_params(case, g, requires_grad=False), O.WEIGHTS_BF16, user_c=O.WEIGHTS_BF16)[0]
    cand = [{"title": ct[:, j].contiguous()} for j in range(ct.shape[1])]
    clicked = [{"title": ht[:, j].contiguous()} for j in range(ht.shape[1])]
    logits, reg = model(cand, clicked)
    assert reg is None
    torch.nn.functional.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long, device=DEV)).backward()
    torch.cuda.synchronize()
    ref = torch.from_numpy(g["logits"])
    res = {"contract": G.relerr(logits, lb), "weights_bf16": G.relerr(logits, lw), "reference_fp32": G.relerr(logits, ref),
           "oracle_bf16_vs_reference_fp32": G.relerr(lb, ref)}
    worst = 0.0
    for k, prm in model.named_parameters():
        if k.startswith("news_encoder.abstract_CNN"):  # never read, as in the reference
            assert prm.grad is None, k
            continue
        exact = p_x[k].grad
        if k == "click_predictor.dnn.2.bias":  # analytically zero (test_gpu_hifiark.py): rounding noise everywhere
            assert float(prm.grad.abs().max()) <= 1e-6 and float(exact.abs().max()) <= 1e-6, (k, prm.grad, exact)
            continue
        e_c = float((p_b[k].grad - exact).norm() / exact.norm())
        worst = max(worst, G.relerr(prm.grad, exact) / max(e_c, 2e-3))
    res["worst_grad_ratio_kernel_over_contract"] = worst
    res["emb_row0_grad_zero"] = bool((model.news_encoder.word_embedding.weight.grad[0] == 0).all())
    print(case, res)
    return res


def test_hifiark_window_2_golden_case():
    """The bounds above, except the one against the weights-only oracle (next test)."""
    res = hifiark_window_2_golden()
    assert res["contract"] < 1e-3, res
    assert res["reference_fp32"] < 1.25 * res["oracle_bf16_vs_reference_fp32"] + 1e-4, res
    assert res["worst_grad_ratio_kernel_over_contract"] < 1.5, res
    assert res["emb_row0_grad_zero"], res


@pytest.mark.xfail(strict=True, reason="hifiark_w2 misses the 1e-3 bound against the weights-only oracle: 1.24e-3 on an H100, the "
                                       "kernel 1.8e-7 from its contract (DESIGN.md section 4, Hi-Fi Ark)")
def test_hifiark_window_2_against_weights_only_oracle():
    """The weights-only oracle rounds the user side's weights to bf16 as well, which the kernels keep in fp32: on this case the
    kernels are 4.8e-4 from the reference's fp32 logits and the weights-only oracle 1.06e-3 (CPU, fp32).  Strict: the test
    fails once the bound is met, so that the miss is not kept past its cause."""
    res = hifiark_window_2_golden()
    assert res["weights_bf16"] < 1e-3, res


def test_naml_get_news_vector_eval_at_window_4():
    """get_news_vector in eval mode at an even window (title L = 19, abstract L = 49): the candidates' news vectors against the
    oracle under the bf16 contract and the reference's own fp32 news vectors."""
    case = "naml_w4"
    g = load_case(case)
    model = CW.build_model(case, DEV)
    model.load_state_dict(CW.state_dict(case, g))
    model.eval()
    flat = lambda k: torch.from_numpy(g["cand_" + k]).reshape(-1, *g["cand_" + k].shape[2:])
    news = {k: flat(k) for k in ("title", "abstract", "category", "subcategory")}
    with torch.no_grad():
        got = model.get_news_vector(news)
        want_b = O.naml_news_encoder(news, CW.case_params(case, g, requires_grad=False), O.BF16)
    ref = torch.from_numpy(g["cand_vec"]).reshape(-1, g["cand_vec"].shape[-1])
    res = {"vs_oracle_bf16": G.relerr(got, want_b), "vs_reference_fp32": G.relerr(got, ref), "oracle_bf16_vs_reference_fp32": G.relerr(want_b, ref)}
    print(res)
    assert res["vs_oracle_bf16"] < 1e-3, res
    assert res["vs_reference_fp32"] < 1.25 * res["oracle_bf16_vs_reference_fp32"] + 1e-4, res
