"""The CNN text encoder of NAML / LSTUR / TANR (nr_cnn_encoder_fwd / _bwd) and its companion operators (element encoder,
Linear over dense rows, fp32 embeddings), called through the C ABI and compared row by row with fp64 references built from
the kernels' own stored inputs (tests/gpu_checks.py).  Bounds:
  * integer / byte work (gather, masks, ones column, pad rows, untouched pre-fill, guards): bit exact; every output the
    ABI writes with "=" starts as NaN and must end finite, and a NaN in any compared value fails its bound;
  * conv output: every element within one bf16 ulp of fp64 relu(conv + b) * mask, plus 1e-6 x sum |x| |w| for the fp32
    accumulation (the ratio to that bound is <= 1); Y + Y_lo per row within 2^-16 relative;
  * pooling weights within 2e-5 of the fp64 softmax of the kernel's own Y, summing to 1 within 1e-5; the pooled rows within
    2e-6 of sum w |Y| per segment;
  * gradients per row: kernel error against exact fp64 <= 1.5 x the error of the bf16 storage contract (dPre, dY rounded to
    bf16), with the contract's error floored at 2e-3 of the row's norm (one bf16 ulp, 2^-8, at F = 8: see below);
  * fp32 outputs of the companions within 1e-6 x sum |x| |w| per element (per row for the accumulated gradients).

An H100 has 132 SMs; the title case (563,200 tokens, 619,520 padded rows) gives every CTA long runs of 64-row tiles on both
consumer warpgroups, the shapes below put segments across tile edges and partial 32-column chunks in every epilogue."""
import pytest

import gpu_checks as G

pytestmark = pytest.mark.gpu


def assert_cnn(r, T, accurate=False):
    assert r["guards_intact"] and r["fwd_outputs_finite"], r
    assert r["xp_mismatch_rows"] == 0, r                       # masked gather, pad rows, ones column: bit exact
    assert r["y_ratio"] <= 1.0 and r["y_dropped_nonzero"] == 0 and r["y_ones_col_and_pad_exact"], r
    assert 0.3 < r["y_pos_fraction"] < 0.7, r                  # the ReLU sees both signs
    if accurate:
        assert r["ylo_ratio"] <= 1.0, r
    assert r["w_err"] <= 2e-5 and r["w_sum_err"] <= 1e-5 and r["out_ratio"] <= 2e-6, r
    assert r["fwd_deterministic"], r
    assert r["bad_id_flag"] == int(r["bad_ids_planted"] > 0), r
    assert r["dWconv_row_ratio"] <= 1.5 and r["demb_row_ratio"] <= 1.5, r
    assert r["dWconv_pitch_cols_untouched"] and r["dWa_pitch_cols_untouched"] and r["demb_untouched_rows_exact"], r
    if T == 1:  # one token per segment: w = 1, out = Y (+ Y_lo), and dscore = w (dw - w dw) = 0 leaves dqv and dWa alone
        assert r["t1_w_err"] <= 2.0 ** -23 and r["t1_out_ratio"] <= 1.0, r
        assert r["t1_dqv_rel"] <= 1e-6 and r["t1_dWa_rel"] <= 1e-6, r
    else:
        assert r["dWa_row_ratio"] <= 1.5 and r["dqv_ratio"] <= 1.5, r


def test_cnn_encoder_naml_title_full_batch():
    """BASELINE.json configuration 2 (NAML, batch 512 x 55 titles of 20 words, V = 70976): every CTA runs long sequences of
    64-row tiles on both warpgroups, the conv and dY GEMMs take two weight slices, EpiDPoolIn prefetches the next tile."""
    r = G.check_cnn_encoder(n_seq=512 * 55, T=20, d=300, F=400, q=200, V=70976, p_drop=0.2, seed=1)
    assert_cnn(r, 20)


@pytest.mark.parametrize("kw", [
    # NAML abstract: a pooling tile holds one 50-row segment (14 idle rows); 52-row padded segments straddle conv tiles
    dict(n_seq=128 * 55, T=50, F=400, V=5000, seed=2),
    # LSTUR precise mode: Y_lo through the row-mapped put_rows path and into the pooled sum
    dict(n_seq=2000, T=20, F=300, accurate=True, seed=3),
    # TANR in eval mode: no dropout anywhere
    dict(n_seq=2000, T=20, F=400, p_drop=0.0, seed=4),
    # a small vocabulary: every id repeats hundreds of times in the scatter
    dict(n_seq=999, T=20, F=400, V=37, seed=5),
])
def test_cnn_encoder_model_shapes(kw):
    kw = dict(dict(d=300, q=200, V=3000, p_drop=0.2), **kw)
    r = G.check_cnn_encoder(**kw)
    assert_cnn(r, kw["T"], kw.get("accurate", False))


@pytest.mark.parametrize("T,n_seq", [(1, 1), (1, 999), (2, 1), (2, 333), (7, 1), (7, 613), (31, 1), (31, 211), (62, 1), (62, 129),
                                     (64, 1), (64, 97)])
def test_cnn_encoder_segment_lengths(T, n_seq):
    """T + 2 = 64 is one padded segment per conv tile; T = 64 fills a pooling tile; an odd n_seq leaves the last tile partial."""
    r = G.check_cnn_encoder(n_seq=n_seq, T=T, d=300, F=300, q=200, V=3000, p_drop=0.2, seed=10 + T, bad_ids=n_seq > 1)
    assert_cnn(r, T)


@pytest.mark.parametrize("F", [300, 256, 252, 8])
def test_cnn_encoder_filter_counts(F):
    """300 and 252 leave a partial 32-column chunk (the plain-store path of EpiStore and EpiDPoolIn), 256 has none, 8 is the
    smallest F; F % 4 != 0 is rejected before any launch (tests/test_cnn_shape_contract.py).  At F = 8 an embedding-gradient
    row sums 3 x 8 bf16 dY values of which ReLU and dropout often leave one or two, so a single dY that rounds to the
    neighbouring bf16 value moves the row by up to one bf16 ulp (2^-8): the gradient floor is one ulp there."""
    r = G.check_cnn_encoder(n_seq=613, T=20, d=300, F=F, q=200, V=3000, p_drop=0.2, seed=30 + F,
                            grad_floor=2.0 ** -8 if F == 8 else 2e-3)
    assert_cnn(r, 20)


@pytest.mark.parametrize("q", [16, 256])
def test_cnn_encoder_query_dims(q):
    """q < 32 runs EpiDPre without its TMA store; q = 256 is the widest query that fits one weight slice."""
    r = G.check_cnn_encoder(n_seq=613, T=20, d=300, F=400, q=q, V=3000, p_drop=0.2, seed=40 + q)
    assert_cnn(r, 20)


@pytest.mark.parametrize("d,p_drop", [(100, 0.2), (64, 0.5), (300, 0.5)])
def test_cnn_encoder_widths_and_dropout(d, p_drop):
    r = G.check_cnn_encoder(n_seq=613, T=20, d=d, F=400, q=200, V=3000, p_drop=p_drop, seed=50 + d)
    assert_cnn(r, 20)


def test_cnn_encoder_empty_batch_launches_nothing():
    r = G.check_cnn_encoder(n_seq=0, T=20, d=300, F=400, q=200, V=50)
    assert r["fwd_launches"] == 0 and r["bwd_launches"] == 0 and r["guards_intact"], r


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(n=512 * 55, F=400), dict(n=512 * 55, F=300), dict(n=3 * 9, F=400, V=15)])
def test_element_encoder(kw):
    """NAML category / subcategory encoder at B (H + C) = 512 x 55 rows and at the golden case's size."""
    r = G.check_element_encoder(E=100, **kw)
    assert r["gather_exact"] and r["bad_id_flag"] == 1 and r["relu_zero_exact"] and r["dY_relu_mask_exact"], r
    assert r["out_elem_ratio"] <= 1.0 and r["dW_row_ratio"] <= 1e-6 and r["dW_bias_col_ratio"] <= 1e-6, r
    assert r["dtable_row_ratio"] <= 1e-6, r
    assert r["dW_pitch_cols_untouched"] and r["dtable_untouched_rows_exact"] and r["guards_intact"], r


@pytest.mark.parametrize("kw", [
    dict(n=512 * 5, K=300, N=275, relu=0),       # TANR topic predictor
    dict(n=512 * 5, K=300, N=275, relu=1),
    dict(n=777, K=900, N=300, relu=1),           # K + 1 = 901 weight-gradient columns: 512 + 389
    dict(n=1000, K=300, N=275, relu=1, strided=True),
    dict(n=1000, K=900, N=300, relu=0, with_dx=False),
])
def test_linear_rows(kw):
    r = G.check_linear_rows(**kw)
    assert r["x_rows_exact"] and r["dY_exact"] and r["out_elem_ratio"] <= 1.0, r
    assert r["dW_row_ratio"] <= 1e-6 and r["dW_bias_col_ratio"] <= 1e-6 and r["dW_pitch_cols_untouched"], r
    if kw.get("with_dx", True):
        assert r["dx_elem_ratio"] <= 1.0, r
    assert r["guards_intact"], r


@pytest.mark.parametrize("kw", [dict(n=512 * 55, V=300, D=100), dict(n=512, V=50000, D=300), dict(n=27, V=15, D=100)])
def test_embedding_f32(kw):
    """LSTUR category embeddings (B (H + C) lookups into a small table) and user embeddings (B lookups into a large one)."""
    r = G.check_embedding_f32(**kw)
    assert r["fwd_exact"] and r["bad_id_flag"] == 1, r
    assert r["bwd_row_ratio"] <= 1e-6 and r["untouched_rows_exact"] and r["row0_untouched"] and r["guards_intact"], r
