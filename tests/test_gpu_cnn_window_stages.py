"""nr_cnn_encoder_fwd / _bwd at conv windows 1 to 4, stage by stage against fp64 references built from the kernels' own stored
Xp, Y and w (tests/cnn_window_util.py), with the bounds of tests/test_gpu_cnn_encoder.py: gather bit exact, conv output within
one bf16 ulp plus an fp32 accumulation allowance, pooling weights and pooled rows, and every gradient row -- dWconv tap by tap,
the bias (column d of tap (w - 1) // 2), dWa, dqv, demb -- within 1.5 x the bf16 contract's error.

Y, w and the backward workspace start as NaN with a guard band behind each: a padded dY row left unzeroed (row T + 1 of a title
at an even window, where L = T - 1) poisons every conv tap's gradient, and a write past the n_seq * L output rows breaks a guard."""
import pytest
import torch

import cnn_window_util as CW
import gpu_checks as G

pytestmark = pytest.mark.gpu

SHORTEST_T = {1: 1, 2: 2, 3: 1, 4: 2}  # T >= w - 2 ((w - 1) // 2)


@pytest.mark.parametrize("accurate", [False, True])
@pytest.mark.parametrize("T", [20, 50, 64, "shortest"])
@pytest.mark.parametrize("window", [1, 2, 3, 4])
def test_cnn_encoder_at_window(window, T, accurate):
    """613 titles (a partial last tile), dropout 0.2 and two out-of-range ids; F = 400 at odd windows, 300 (a partial 32-column
    chunk in every epilogue) at even ones; accurate = the LSTUR mode, Y_lo into the pooled sum."""
    T = SHORTEST_T[window] if T == "shortest" else T
    F = 300 if window % 2 == 0 else 400
    r = CW.check_cnn_window(n_seq=613, T=T, window=window, F=F, accurate=accurate, seed=7 * window + T)
    print(window, T, accurate, {k: v for k, v in r.items() if "ratio" in k or "err" in k})
    CW.assert_cnn_window(r, CW.out_len(T, window))


@pytest.mark.parametrize("window", [2, 4])
def test_cnn_encoder_at_window_training_step_size(window):
    """NAML's title encoder at a training step (512 x 55 titles of 20 words, V = 70976) at the two even windows."""
    r = CW.check_cnn_window(n_seq=512 * 55, T=20, window=window, F=400, V=70976, seed=100 + window)
    CW.assert_cnn_window(r, 19)


def test_cnn_encoder_empty_batch_at_window_4_launches_nothing():
    r = CW.check_cnn_window(n_seq=0, T=20, window=4, V=50)
    assert r["fwd_launches"] == 0 and r["bwd_launches"] == 0 and r["guards_intact"], r


@pytest.mark.parametrize("accurate", [False, True])
def test_window_0_is_window_3(accurate):
    """args.window = 0 (every caller built before the field existed) runs window 3: the same launches, the forward outputs and
    the whole backward workspace (dscore, dPre, the padded dY) bit for bit.  The gradients are split-K fp32 red.add sums, whose
    order differs from run to run: they agree to that reordering."""
    o = CW.cnn_operands(613, 20, 300, 400, 200, 3000, 3, seed=5)
    f0, b0, nf0, nb0 = CW.run_cnn(o, 0.2, accurate, 0)
    f3, b3, nf3, nb3 = CW.run_cnn(o, 0.2, accurate, 3)
    assert (nf0, nb0) == (nf3, nb3), (nf0, nb0, nf3, nb3)
    for k in f0:
        assert G._bits_equal(f0[k].all, f3[k].all), k
    assert G._bits_equal(b0["ws"].all, b3["ws"].all)
    for k in ("dWc", "dWa", "dqv", "demb"):
        a, b = b0[k].body.double(), b3[k].body.double()
        assert torch.isfinite(a).all() and float((a - b).norm() / b.norm()) < 1e-6, k
