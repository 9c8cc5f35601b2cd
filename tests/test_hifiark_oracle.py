"""Pins the Hi-Fi Ark oracle (oracle/hifiark_oracle.py) against golden vectors minted from the live reference
(oracle/make_golden_hifiark.py), and records the storage contract the kernels ship with.  CPU only."""
import numpy as np
import torch

import hifiark_oracle as HO
import newsrec_oracle as O
from golden_util import V, grad_summary, load_case


def params(g, dtype=torch.float32, requires_grad=True):
    return {k: v.to(dtype).clone().requires_grad_(requires_grad) for k, v in HO.hifiark_state_dict(V, int(g["seed"])).items()}


def titles(g):
    return torch.from_numpy(g["cand_title"]), torch.from_numpy(g["clicked_title"])


def centred(x):
    return x - x.mean(dim=1, keepdim=True)


def test_oracle_matches_reference_fp32():
    g = load_case("hifiark")
    p = params(g)
    logits, _, cv, hv, archive = HO.hifiark_forward(*titles(g), p)
    np.testing.assert_allclose(logits.detach().numpy(), g["logits"], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(cv.detach().numpy(), g["cand_vec"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(hv.detach().numpy(), g["clicked_vec"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(archive.detach().numpy(), g["archive"], rtol=1e-4, atol=1e-5)
    loss = O.click_loss(logits)
    assert abs(loss.item() - float(g["loss"])) < 2e-5 * max(1.0, abs(float(g["loss"])))
    loss.backward()
    for k, prm in p.items():
        if "gsum:" + k not in g:  # abstract_CNN: never read, no gradient in the reference either
            assert k.startswith("news_encoder.abstract_CNN") and prm.grad is None, k
            continue
        s, samp = grad_summary(prm.grad, k)
        ref_s, ref_samp = g["gsum:" + k], g["gsamp:" + k]
        # floor: the gradient of the last bias is analytically zero (each impression's softmax gradient sums to zero), so the
        # golden holds fp32 rounding noise of a few 1e-8 that differs between CPUs
        scale = max(ref_s[0], 5e-2)
        assert abs(s[0] - ref_s[0]) <= 1e-4 * scale, (k, s, ref_s)
        assert abs(s[1] - ref_s[1]) <= 1e-4 * scale, (k, s, ref_s)
        np.testing.assert_allclose(samp, ref_samp, rtol=1e-3, atol=2e-5 * scale)
    assert torch.equal(p["news_encoder.word_embedding.weight"].grad[0], torch.zeros(300))


def test_regularizer_and_1d_prediction_match_reference():
    g = load_case("hifiark")
    p = params(g)
    reg = HO.regularizer(p["omap.W"])
    assert abs(reg.item() - float(g["reg"])) < 1e-5 * float(g["reg"])
    reg.backward()
    s, samp = grad_summary(p["omap.W"].grad, "reg:omap.W")
    np.testing.assert_allclose(s, g["reg_gsum"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(samp, g["reg_gsamp"], rtol=1e-4, atol=1e-7)
    with torch.no_grad():
        cv, a = torch.from_numpy(g["cand_vec"]), torch.from_numpy(g["archive"])
        got = np.array([[HO.get_prediction(cv[b, j], a[b], p).item() for j in range(cv.shape[1])] for b in range(cv.shape[0])])
    np.testing.assert_allclose(got, g["pred1d"], rtol=1e-5, atol=1e-6)


def test_shipped_storage_contract_against_weights_bf16():
    """The contract the drop-in ships with (plain bf16 storage in the news encoder, fp32 after it) against the fp32 oracle on
    bf16-rounded weights: the logits within 1e-3 norm-wise on the golden case.  The centred error (each impression's mean
    logit removed, what the softmax loss sees) is larger because the DNN bias dominates the logits (DESIGN.md section 4)."""
    g = load_case("hifiark")
    p = params(g, requires_grad=False)
    with torch.no_grad():
        want = HO.hifiark_forward(*titles(g), p, O.WEIGHTS_BF16, user_c=O.WEIGHTS_BF16)[0]
        got = HO.hifiark_forward(*titles(g), p, O.BF16, user_c=O.WEIGHTS_BF16)[0]
    assert float((got - want).norm() / want.norm()) < 1e-3
    assert float((centred(got) - centred(want)).norm() / centred(want).norm()) < 5e-2
