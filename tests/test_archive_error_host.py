"""The bound of tests/archive_error_ref.py, checked without a GPU on the case list the kernel test runs
(tests/test_gpu_hifiark.py): an fp32 restatement of the kernels stays within a quarter of it on every output element;
TF32- and bf16-rounded operands, and three planted mistakes, miss it by 8x or more."""
import pytest
import torch

import archive_error_ref as R

B = 2
COUNTS = R.SEGMENTS + [2, 2]


def _ratios(fn, ref, *args, **kw):
    out = {}
    for name, ar in (("fp32", R.Arith(torch.float32)), ("tf32", R.Arith(rnd=R.tf32)), ("bf16", R.Arith(rnd=R.bf16))):
        out[name] = R.ratios(R.restate(ar, fn, *args, **kw), ref)
    return out


def _judge(case, res):
    print(case, {m: {k: round(v, 3) for k, v in r.items()} for m, r in res.items()})
    assert max(res["fp32"].values()) <= 0.25, (case, res["fp32"])
    for mode in ("tf32", "bf16"):
        assert max(res[mode].values()) >= 8, (case, mode, res[mode])
        for name in R.PRODUCT_OUTPUTS:
            if name in res[mode]:
                assert res[mode][name] >= 8, (case, mode, name, res[mode][name])


@pytest.mark.parametrize("H,F,P", R.USER_CASES)
def test_user_bound(H, F, P):
    x, W, da = R.user_inputs(B, H, F, P)
    dreg = 0.7
    ref = R.user_ref(R.Arith(probes=R.PROBES), x, W, da, dreg)
    res = _ratios(R.user_ref, ref, x, W, da, dreg)
    for plant in ("no_residual", "q_over_p"):
        got = R.restate(R.Arith(), R.user_ref, x, W, da, dreg, plant=plant)
        res[plant] = R.ratios(got, ref, ["archive"])
        assert res[plant]["archive"] >= 8, (plant, res[plant])
    _judge((H, F, P), res)


def test_user_bound_padded_history_and_peaked_scores():
    F, H = 300, 50
    x, W, da = R.user_inputs(2, H, F, 5, seed=31)
    x = R.f32(x * (0.1 * F ** 0.5 / 3.0))
    x[0, :30] = x[0, 30]                     # a history of identical (padded) news vectors
    x[1] *= 60.0                             # large-norm rows: S up to ~3e3
    ref = R.user_ref(R.Arith(probes=R.PROBES), x, W, da, 0.7)
    _judge("peaked", _ratios(R.user_ref, ref, x, W, da, 0.7))


@pytest.mark.parametrize("F,P,Hd", R.SCORE_CASES)
def test_scorer_bound(F, P, Hd):
    args = R.score_inputs(F, P, Hd, COUNTS)
    ref = R.score_ref(R.Arith(probes=R.PROBES), *args)
    res = _ratios(R.score_ref, ref, *args)
    if P > 1:                                # at P = 1 the mean of the archive rows is the right u
        res["u_mean"] = R.ratios(R.restate(R.Arith(), R.score_ref, *args, plant="u_mean"), ref, ["logits"])
        assert res["u_mean"]["logits"] >= 8, res["u_mean"]
    _judge((F, P, Hd), res)


def test_probes_see_shared_errors():
    """The error of P1 reaches L = Y W as a sum over f: the probed sd of L must exceed the sd that independent
    per-column errors of Y would give when the columns add coherently (every x and W entry positive)."""
    ar = R.Arith(probes=R.PROBES)
    x = R.f32(torch.rand((1, 8, 64), dtype=torch.float64, generator=torch.Generator().manual_seed(3)))
    W = R.f32(torch.rand((64, 2), dtype=torch.float64, generator=torch.Generator().manual_seed(4)))
    X, Wd = ar.input(x), ar.input(W)
    P1, Y, Q = R.user_forward_core(ar, X, Wd)
    L = ar.dot("zbhf,fp->zbhp", Y, Wd, 64)
    indep = ((ar.sd(Y) ** 2).unsqueeze(-1) * Wd.pow(2)).sum(-2).sqrt()
    assert bool((ar.sd(L) > 2 * indep).all())
