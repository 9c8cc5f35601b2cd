"""The NRMS / Exp1 self-attention encoder (nr_mhsa_encoder_fwd / _bwd) called through the C ABI in its four forward variants
(ids fast, ids accurate, dense fast, dense precise) and their backward, compared stage by stage and row by row with fp64
references built on the device from what the kernels themselves stored for each stage (tests/gpu_checks.py
check_mhsa_encoder).  A stage is judged on its own inputs, so one wrong head, title or row shows up where it happens.

Bounds (bf16 keeps 8 significant bits: one ulp is 2^-7 of the leading bit, so rounding to nearest is within 2^-8 of
the value):
  * integer / byte work: bit exact.  X is bf16(table[id] * gather mask) (out-of-range ids read row 0 and raise the flag) or
    bf16(dense + pos) summed in fp32 first, with the ones column at d and zeros up to the pitch; X_kcat is the [hi | lo]
    pair nr_rows_to_bf16_hilo defines; the section-padding columns of Q|K|V (and of V_lo) are exactly 0; dropped context
    elements are exactly 0 in both planes; the ones column is in C_hi only and every other pitch column of both planes is 0.
    Every "=" output starts as NaN, so a NaN in a compared value fails its bound.
  * Q|K|V stored in bf16: the product of bf16 operands is exact in fp32 and the fp32 sum of d products is within
    d * 2^-24 sum |x||w| of the exact one in the worst case and far less in practice: 1e-6 * sum |x||w| (with |b|) covers
    it, and the one bf16 rounding of the result is within half an ulp, so each element is within one bf16 ulp plus
    1e-6 * sum |x||w|.  V_hi + V_lo keeps about 16 bits: a row within 2^-16 |ref| + 1e-6 |sum |x||w|| (norms per row).
    QKV_f32 (precise) has no output rounding: 1e-6 * sum |x||w| of fp64 (X_hi + X_lo) W^T + b.
  * context against fp64 mask * (A V), A from the stored Q, K (with the reference's +1e-8): in fp32 the scores carry
    an error of about 20 * 2^-24 sum |q||k| / sqrt(d_k) (a few 1e-6 at unit-sized Q, K), the exponentials a few ulps
    (ex2.approx): together well inside 2^-15 of the probabilities, i.e. 2^-15 sum_j A_ij |V_j| on an output element.
      fast: the probabilities enter A V as bf16 (2^-8 each: 2^-8 sum_j A_ij |V_j|), the context is rounded to bf16 once
        (half an ulp) and, under dropout, a second time after the 1/(1 - p) scaling (the kernel rounds before and after):
        one ulp of the output, two where the mask rescales, plus (2^-8 + 2^-15) sum_j A_ij |V_j| * m.
      accurate / precise, on C_hi + C_lo: the probabilities travel as a hi/lo pair (2^-16), A_lo V_lo is dropped
        (2^-16), the output pair keeps 2^-16: 2^-15 sum_j A_ij |V_j| * m + 2^-16 |ref|.
    Discrimination: C_hi alone, and (accurate news) a reference without V_lo, must miss that bound by >= 8x on their
    worst element: one bf16 rounding (up to 2^-8 relative) is ~80x the bound, so the check sees the low planes.
  * pooling: w within 2e-5 of the fp64 softmax of tanh(C_hi Wa^T + ba) qv (the score GEMM reads the hi plane), summing to
    1 within 1e-5; the pooled rows within 2e-6 of sum w |C| per segment of sum w (C_hi [+ C_lo]).
  * the backward's first stages, read from the workspace and judged element by element on their own inputs:
      dscore = w (dw - sum w dw), dw = C_hi . dout: fp32 dot products of d terms, within d 2^-24 sum |c||dout| each, plus
        4 2^-24 of |dw| for the few fp32 operations on w;
      dPre = dscore qv (1 - T^2) from the kernel's own dscore: the epilogue's tanh.approx.f32 is within 2^-10.987 of T
        relatively (PTX ISA) and the fp32 pre-activation within 1e-6 sum |c||wa| (+|ba|), which moves T by (1 - T^2) times
        that; 1 - T^2 then moves by up to 2|T||dT| + dT^2; plus one bf16 ulp of the stored value.  Near saturation the
        tanh approximation alone is as large as dPre's own bf16 rounding (2|T| |dT| against (1 - T^2) 2^-8).
  * gradients per row: kernel error against the exact fp64 chain <= 1.5 x the error of the bf16 contract (the kernels'
    stored dPre, then dC, dS, A as the operand of dV, dQ|dK|dV rounded to bf16, and the recomputed Q|K|V where the backward
    recomputes it), the contract's error floored at 2e-3 of the row's norm; rows of dWqkv_ext (bias column included),
    dWa_ext, dqv, touched demb rows, ddense rows, dpos rows.  The "+=" pre-fill survives bit for bit in the section-padding rows and pitch
    columns of dWqkv_ext, the pitch columns of dWa_ext, demb row 0 and the rows no id touches; every guard is intact.
    Discrimination: a reference without the gather mask pushes the demb ratio above 10, one without the context mask the
    dWqkv ratio.
  * determinism: a second forward is bit-identical.

The grid of the hi/lo title kernel is min(n_seq, SMs), of the plain one min(n_seq, 2 SMs): the SM count comes from the
library, so the uneven last rounds are placed on whatever GPU runs the file."""
import pytest

import gpu_checks as G

pytestmark = pytest.mark.gpu


def _sms():
    from newsrec_b200 import load_library
    return int(load_library().nr_num_sms())


def assert_mhsa(r, level="ids", mode="accurate", pos=False, ddense_rows=True):
    assert r["guards_intact"] and r["fwd_outputs_finite"], r
    assert r["x_mismatch_rows"] == 0 and r["qkv_pad_zero"], r
    assert r["ctx_ratio"] <= 1.0 and r["ctx_dropped_nonzero"] == 0 and r["ctx_ones_col"] and r["ctx_pitch_zero"], r
    if mode == "accurate":
        assert r["ctx_hi_only_ratio"] >= 8.0, r   # the bound sees the low plane of the context
    if level == "ids":
        assert r["bad_id_flag"] == int(r["bad_ids_planted"] > 0), r
        assert r["qkv_ratio"] <= 1.0, r
        if mode == "accurate":
            assert r["vlo_ratio"] <= 1.0 and r["ctx_no_vlo_ratio"] >= 8.0, r
        assert r["demb_row_ratio"] <= 1.5 and r["demb_untouched_rows_exact"] and r["demb_row0_untouched"], r
    else:
        if mode == "accurate":
            assert r["xk_mismatch_rows"] == 0 and r["qkv32_ratio"] <= 1.0, r
        else:
            assert r["qkv_ratio"] <= 1.0, r
        if ddense_rows:
            assert r["ddense_row_ratio"] <= 1.5, r
        if pos:
            assert r["dpos_row_ratio"] <= 1.5, r
    assert r["w_err"] <= 2e-5 and r["w_sum_err"] <= 1e-5 and r["out_ratio"] <= 2e-6, r
    assert r["dscore_ratio"] <= 1.0 and r["dpre_ratio"] <= 1.0, r
    assert r["dWqkv_row_ratio"] <= 1.5 and r["dWa_row_ratio"] <= 1.5 and r["dqv_ratio"] <= 1.5, r
    assert r["dWqkv_padding_untouched"] and r["dWa_pitch_cols_untouched"], r
    if "t1_dWqk_rel" in r:  # T = 1: the Q, K rows of dWqkv_ext are 1e-8 of the V rows (see check_mhsa_encoder)
        assert r["t1_dWqk_rel"] <= 1e-6, r
    assert r["fwd_deterministic"], r


def test_mhsa_encoder_news_bench_shape():
    """bench.py's news level: batch 512 x 55 titles of 20 words, 15 heads, V = 70976, train mode: long per-CTA title loops."""
    r = G.check_mhsa_encoder(n_seq=512 * 55, T=20, d=300, heads=15, q=200, V=70976, p_drop=0.2, mode="accurate", seed=1)
    assert_mhsa(r)


@pytest.mark.parametrize("kw", [
    dict(n_seq=2000, mode="fast", p_drop=0.2, seed=2),       # the plain title kernel template
    dict(n_seq=2000, mode="accurate", p_drop=0.0, seed=3),   # eval mode: no mask anywhere
])
def test_mhsa_encoder_news_modes(kw):
    r = G.check_mhsa_encoder(T=20, d=300, heads=15, q=200, V=3000, **kw)
    assert_mhsa(r, mode=kw["mode"])


@pytest.mark.parametrize("heads", [1, 2, 7, 14])
def test_mhsa_encoder_news_head_counts(heads):
    """The title kernels below 15 warps.  With an odd head count the last head is even and its k8 step runs into the 4
    section-padding columns (d = 20 heads is 4 mod 8); with an even head count the last head is odd.  At d = 20 and 40 the
    V section starts inside a 32-column chunk of the projection GEMM, which emits its low plane by whole chunks: the
    accurate variant does not exist there (nr_mhsa_accurate_supported) and is refused before any launch; the plain title
    kernel runs those head counts."""
    from newsrec_b200 import load_library
    supported = heads >= 3
    assert load_library().nr_mhsa_accurate_supported(20, 20 * heads, heads) == int(supported)
    mode = "accurate" if supported else "fast"
    if not supported:
        r = G.check_mhsa_encoder(n_seq=613, T=20, d=20 * heads, heads=heads, q=200, V=3000, p_drop=0.2, mode="accurate")
        assert "chunk-aligned V section" in r["fwd_rejected"] and r["fwd_launches"] == 0, r
    r = G.check_mhsa_encoder(n_seq=613, T=20, d=20 * heads, heads=heads, q=200, V=3000, p_drop=0.2, mode=mode, seed=10 + heads)
    assert_mhsa(r, mode=mode)


@pytest.mark.parametrize("which", ["1", "sms-1", "sms+1", "2sms+1"])
def test_mhsa_encoder_news_grid_rounds(which):
    """grid = min(n_seq, SMs) for the hi/lo forward and the title backward: one title, one short of a full round, one over,
    and one over two rounds."""
    sms = _sms()
    n_seq = {"1": 1, "sms-1": sms - 1, "sms+1": sms + 1, "2sms+1": 2 * sms + 1}[which]
    r = G.check_mhsa_encoder(n_seq=n_seq, T=20, d=300, heads=15, q=200, V=3000, p_drop=0.2, mode="accurate", seed=20 + n_seq,
                             bad_ids=n_seq > 1)
    assert_mhsa(r)


def test_mhsa_encoder_news_head_level_kernels():
    """T = 30, d_k = 30: no title-level kernel applies (the accurate variant does not exist for the shape), the head-level
    forward and backward run with the context dropout."""
    from newsrec_b200 import load_library
    assert load_library().nr_mhsa_accurate_supported(30, 300, 10) == 0
    r = G.check_mhsa_encoder(n_seq=613, T=30, d=300, heads=10, q=200, V=3000, p_drop=0.2, mode="fast", seed=30)
    assert_mhsa(r, mode="fast")


def test_mhsa_encoder_news_scatter_contention_and_masks():
    """37 words: every id repeats hundreds of times in the scatter; p = 0.5 drops half of everything.  The references without
    the gather mask and without the context mask must fail by far: the masks the backward regenerates are the forward's."""
    r = G.check_mhsa_encoder(n_seq=999, T=20, d=300, heads=15, q=200, V=37, p_drop=0.5, mode="accurate", seed=31, discriminate=True)
    assert_mhsa(r)
    assert r["demb_ratio_without_gather_mask"] > 10 and r["dWqkv_ratio_without_ctx_mask"] > 10, r


@pytest.mark.parametrize("q", [16, 256])
def test_mhsa_encoder_news_query_dims(q):
    """The narrowest and the widest query the pooling GEMMs take."""
    r = G.check_mhsa_encoder(n_seq=613, T=20, d=300, heads=15, q=q, V=3000, p_drop=0.2, mode="accurate", seed=40 + q)
    assert_mhsa(r)


@pytest.mark.parametrize("mode", ["accurate", "fast"])
@pytest.mark.parametrize("pos", [False, True])
def test_mhsa_encoder_user_bench_shape(mode, pos):
    """bench.py's history level (512 users x 50 clicked news, NRMS) and Exp1's positional history embedding."""
    r = G.check_mhsa_encoder(n_seq=512, T=50, d=300, heads=15, q=200, level="dense", mode=mode, pos=pos, p_drop=0.0, seed=50)
    # the input-gradient rows of the precise variant with the positional addend: test_mhsa_encoder_user_exp1_input_gradient_rows
    assert_mhsa(r, level="dense", mode=mode, pos=pos, ddense_rows=not (mode == "accurate" and pos))


@pytest.mark.xfail(strict=True, reason="open finding: on an H100 80GB HBM3 (400 W) the worst of the 25,600 input-gradient "
                                      "rows of this case has a kernel error of 4.4e-3 against the bf16 contract's 2.8e-3 "
                                      "(ratio 1.54 > 1.5); every other row and stage of the case meets its bound")
def test_mhsa_encoder_user_exp1_input_gradient_rows():
    r = G.check_mhsa_encoder(n_seq=512, T=50, d=300, heads=15, q=200, level="dense", mode="accurate", pos=True, p_drop=0.0, seed=50)
    assert r["ddense_row_ratio"] <= 1.5, r


@pytest.mark.parametrize("kw", [
    dict(heads=10, T=50),                        # d_k = 30: the scalar mhsa_f32_fwd_kernel
    dict(heads=20, T=50),                        # d_k = 15
    dict(heads=15, T=1),                         # one clicked news: w = 1
    dict(heads=15, T=64),                        # the longest sequence
    dict(heads=15, T=50, noncontig=True),        # a (B, H, d) view: dense_s_* strides
])
def test_mhsa_encoder_user_precise_shapes(kw):
    r = G.check_mhsa_encoder(n_seq=97, d=300, q=200, level="dense", mode="accurate", p_drop=0.0, seed=60 + kw["heads"] + kw["T"], **kw)
    assert_mhsa(r, level="dense", mode="accurate")


@pytest.mark.parametrize("level", ["ids", "dense"])
def test_mhsa_encoder_empty_batch_launches_nothing(level):
    r = G.check_mhsa_encoder(n_seq=0, T=20 if level == "ids" else 50, level=level, mode="accurate", V=50)
    assert r["fwd_launches"] == 0 and r["bwd_launches"] == 0 and r["guards_intact"], r
