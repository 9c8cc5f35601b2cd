"""Pins the DKN oracle (oracle/dkn_oracle.py) against golden vectors minted from the live reference
(oracle/make_golden_dkn.py), checks the collapse of the candidate-aware attention and the storage contract.  CPU only.
Two golden cases: dkn at the default window_sizes [2, 3, 4], dkn_w4133 at [4, 1, 3, 3] (unsorted, a repeated size)."""
import numpy as np
import pytest
import torch

import dkn_oracle as DO
import newsrec_oracle as O
from golden_util import V, grad_summary, load_case

DEAD = ("attention.dnn.0.bias", "attention.dnn.1.bias")  # and the candidate half of attention.dnn.0.weight
CASES = {"dkn": (2, 3, 4), "dkn_w4133": (4, 1, 3, 3)}  # golden case -> config.window_sizes it was minted at


def golden(case):
    g = load_case(case)
    if "window_sizes" in g:  # recorded by the recipe since the second case
        assert tuple(int(x) for x in g["window_sizes"]) == CASES[case]
    return g


def params(g, windows, dtype=torch.float32, requires_grad=True):
    return {k: v.to(dtype).clone().requires_grad_(requires_grad)
            for k, v in DO.dkn_state_dict(V, int(g["num_entities"]), int(g["seed"]), windows=windows).items()}


def ids(g):
    return [torch.from_numpy(g[k]) for k in ("cand_title", "cand_entities", "clicked_title", "clicked_entities")]


def _oracle_matches_reference_fp32(case):
    g, windows = golden(case), CASES[case]
    p = params(g, windows)
    logits, cv, hv, _ = DO.dkn_forward(*ids(g), p, windows=windows)
    assert cv.shape[2] == len(windows) * 50
    np.testing.assert_allclose(logits.detach().numpy(), g["logits"], rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(cv.detach().numpy(), g["cand_vec"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(hv.detach().numpy(), g["clicked_vec"], rtol=1e-4, atol=1e-5)
    O.click_loss(logits).backward()
    Fp = cv.shape[2]
    for k, prm in p.items():
        grad = prm.grad if prm.grad is not None else torch.zeros_like(prm)
        ref_s = g["gsum:" + k]
        if k in DEAD or k == "attention.dnn.0.weight":
            # analytically zero (the softmax over the history cancels them): the reference holds rounding noise there
            live = grad[:, Fp:] if k == "attention.dnn.0.weight" else None
            if live is None:
                assert float(grad.abs().max()) <= 1e-6 and ref_s[0] <= 1e-5, (k, ref_s)
                continue
            assert float(grad[:, :Fp].abs().max()) <= 1e-6, k
        s, samp = grad_summary(grad, k)
        scale = max(ref_s[0], 5e-2)
        assert abs(s[0] - ref_s[0]) <= 1e-4 * scale, (k, s, ref_s)
        np.testing.assert_allclose(samp, g["gsamp:" + k], rtol=1e-3, atol=2e-5 * scale)
    assert torch.equal(p["kcnn.word_embedding.weight"].grad[0], torch.zeros(300))
    assert torch.equal(p["kcnn.entity_embedding.weight"].grad[0], torch.zeros(100))


def test_oracle_matches_reference_fp32():
    _oracle_matches_reference_fp32("dkn")


def test_oracle_matches_reference_fp32_at_windows_4133():
    _oracle_matches_reference_fp32("dkn_w4133")


def _get_prediction_matches_reference(case):
    g, windows = golden(case), CASES[case]
    p = params(g, windows, requires_grad=False)
    cv, hv = torch.from_numpy(g["cand_vec"]), torch.from_numpy(g["clicked_vec"])
    got = np.stack([DO.get_prediction(cv[b], hv[b], p, windows).numpy() for b in range(cv.shape[0])])
    np.testing.assert_allclose(got, g["pred"], rtol=1e-5, atol=1e-6)


def test_get_prediction_matches_reference():
    _get_prediction_matches_reference("dkn")


def test_get_prediction_matches_reference_at_windows_4133():
    _get_prediction_matches_reference("dkn_w4133")


def test_candidate_attention_collapses_to_one_user_vector_fp64():
    """softmax_j(W2 (W1 [c; h_j] + b1) + b2) == softmax_j(beta . h_j): the candidate half and the biases cancel.  Random,
    non-trivial candidate weights and biases, fp64; and their gradients are exactly zero under the collapsed form."""
    B, C, H, Fp = 4, 5, 7, 150
    hv = O.det_uniform((B, H, Fp), 1, -1, 1, torch.float64)
    cand = O.det_uniform((B, C, Fp), 2, -1, 1, torch.float64)
    p = {"attention.dnn.0.weight": O.det_uniform((16, 2 * Fp), 3, -0.5, 0.5, torch.float64),
         "attention.dnn.0.bias": O.det_uniform((16,), 4, -2, 2, torch.float64),
         "attention.dnn.1.weight": O.det_uniform((1, 16), 5, -1, 1, torch.float64),
         "attention.dnn.1.bias": O.det_uniform((1,), 6, -3, 3, torch.float64)}
    full = DO.attention_per_candidate(cand, hv, p)
    u = DO.user_vector(hv, p)
    assert float((full - u.unsqueeze(1)).abs().max()) < 1e-13
    q = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    (DO.attention_per_candidate(cand, hv, q) * O.det_uniform((B, C, Fp), 7, -1, 1, torch.float64)).sum().backward()
    assert float(q["attention.dnn.0.weight"].grad[:, :Fp].abs().max()) < 1e-12
    assert float(q["attention.dnn.0.bias"].grad.abs().max()) < 1e-12
    assert float(q["attention.dnn.1.bias"].grad.abs().max()) < 1e-12


def _shipped_storage_contract_against_weights_bf16(case):
    """Plain bf16 storage in the news encoder, fp32 after it, against the fp32 oracle on bf16-rounded weights: within 1e-3
    norm-wise on the golden case (DESIGN.md section 4)."""
    g, windows = golden(case), CASES[case]
    p = params(g, windows, requires_grad=False)
    with torch.no_grad():
        want = DO.dkn_forward(*ids(g), p, O.WEIGHTS_BF16, windows)[0]
        got = DO.dkn_forward(*ids(g), p, O.BF16, windows)[0]
    assert float((got - want).norm() / want.norm()) < 1e-3


def test_shipped_storage_contract_against_weights_bf16():
    _shipped_storage_contract_against_weights_bf16("dkn")


def test_shipped_storage_contract_against_weights_bf16_at_windows_4133():
    _shipped_storage_contract_against_weights_bf16("dkn_w4133")


def test_window_order_and_repeats_follow_the_config():
    """The oracle runs the windows in config order with repeats kept, as the reference's loop over window_sizes does: the
    sorted, de-duplicated set computes a different function (narrower vectors, other column order), and a reordered list
    permutes the news vector's window blocks."""
    g, windows = golden("dkn_w4133"), CASES["dkn_w4133"]
    p = params(g, windows, requires_grad=False)
    title, ents = ids(g)[:2]
    title, ents = title.reshape(-1, title.shape[-1]), ents.reshape(-1, ents.shape[-1])
    with torch.no_grad():
        got = DO.kcnn(title, ents, p, windows=windows)
        np.testing.assert_allclose(got.view(*g["cand_vec"].shape).numpy(), g["cand_vec"], rtol=1e-4, atol=1e-5)
        srt = DO.kcnn(title, ents, p, windows=tuple(sorted(windows)))
        assert float((srt - got).abs().max()) > 1e-2  # [1, 3, 3, 4] puts other windows in blocks 0, 1 and 3
        uniq = DO.kcnn(title, ents, p, windows=tuple(sorted(set(windows))))
        assert uniq.shape[1] == 3 * 50 != got.shape[1]
        blocks = got.view(got.shape[0], len(windows), 50)
        assert torch.equal(blocks[:, 2], blocks[:, 3])  # the repeated size: the same conv, the same pooled vector
        by_size = {x: blocks[:, i] for i, x in enumerate(windows)}
        assert torch.equal(srt.view_as(blocks), torch.stack([by_size[x] for x in sorted(windows)], 1))
    with pytest.raises(ValueError):  # get_prediction checks the width against the window list
        DO.get_prediction(got[:3], got[3:9], p, (2, 3, 4))
