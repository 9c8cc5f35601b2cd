"""The self-attention core (nr_mhsa_core_fwd / _bwd) called through the C ABI across its kernel dispatch (csrc/attn.cu
dispatch(): the title kernels, and mhsa_mma_{fwd,bwd}_kernel over the d_k class NTD 2/3/4, the per-lane copy plan or the copy
loops, the fixed head shape or the run-time one, per-warp tasks or cooperative CTAs), and the standalone
MultiHeadSelfAttention built on it (ops.MhsaFn), compared element by element with fp64 references built on the device from
the same bf16 Q|K|V and dCtx the kernels read (tests/mhsa_core_ref.py, itself checked by tests/test_mhsa_core_host.py).

Inputs: every column the kernels must not read holds NaN (the section padding [d, sec), the columns [3 sec, ld_qkv) and the
dCtx columns [d, ld_dctx)); every "=" output starts as NaN; every buffer is followed by a guard.

Bounds (bf16 keeps 8 significant bits: rounding to nearest is within 2^-8 relatively, half an ulp absolutely; one fp32 ulp is
2^-23 relatively, allowed per accumulation step because tensor-core sums may truncate):
  * the probabilities.  The scores are fp32 sums of d_k exact bf16 products, within d_k 2^-23 sum |q||k| / sqrt(d_k); the
    scale (rsqrt) and the max-subtracted exponent argument add 2^-21 of |S| and of |S - max S|.  An error dS_j in one score
    moves A_ij by dS_j relatively, the normalisation by at most the row's largest dS; exp2 (ex2.approx), the fp32 row sum of
    T terms and the reciprocal add 2^-20 + T 2^-23.  That is eps_ij; probabilities below the fp32 normal range flush to 0,
    so A_k is within eps A + 2^-100 of A.
  * context against fp64 m * (A V), A = exp(S) / (sum exp(S) + 1e-8) in its stable form: A enters A V as bf16 (2^-8), plus
    eps and the fp32 sum; the context is rounded to bf16 once, and a second time after the 1/(1 - p) scaling where the mask
    rescales: one ulp of the output (two where m > 1) + sum_j (2^-8 + eps_ij) A_ij |V_j| m.
  * dV = bf16(A)^T dC: the kernel's bf16(A_k) differs from bf16(A) only where a rounding boundary lies within eps A of A
    (flip(A), one bf16 ulp of A there, 0 elsewhere): half an ulp + sum_i (flip(A_ij) + T 2^-23 A_ij) |dC_i|.
  * dQ = bf16(dS) K, dK = bf16(dS)^T Q, dS = A (dA - sum A dA) / sqrt(d_k) the gradient of the unscaled product (fp64):
    half an ulp + sum_j (flip(dS_ij) + T 2^-23 |dS_ij|) |K_j| (|Q_i| for dK), where flip(dS) is the bf16 rounding change over
    the kernel's fp32 error of dS: eps of A in A (dA - sum A dA), the fp32 sums of dA = dC V^T (d_k 2^-23 sum |dC||V|) and of
    sum A dA (T 2^-23), and 2^-21 of |dS| for the scaling.
  * bit exact: dropped context elements are 0 where dropout_mask_dev(seed, p, rows, d, ld_ctx) is 0 (the library's hash of
    row * ld_ctx + col); the ones column at d and zeros in (d, ld_ctx); zeros in the dQ|dK|dV section padding; the columns
    [3 sec, ld_dqkv) are not written (they keep their NaN pre-fill); a second call of each direction is bit-identical (no
    atomics).
  * every score below -88.7: exp2f(-max) overflows in the kernels' 1e-8 exp2(-max) term, so the context and every gradient
    are exactly 0 (the reference's are below 1e-30).  That is the kernels' documented range, asserted exactly.
  * discrimination: the neighbouring head's context, the context without the last key row, the neighbouring row's dropout
    mask and dV with unrounded A must miss their bound by >= 8x on their worst element.
  * MhsaFn: the context within the context bound on the Q|K|V the forward stored; every gradient per row ([W | b] rows of each
    projection, input rows) within 1.5 x the error of the bf16 contract (oracle.multihead_self_attention under Contract(bf16))
    against the exact chain on the same bf16 operands, the contract's error floored at 2e-3 of the row's norm.  At T = 1 the
    W_Q, W_K gradients are 1e-8 of W_V's (A = 1 / (1 + 1e-8): dS is below fp32 resolution) and are held to that scale.
    Measured on an H100 80GB HBM3 (700 W power limit), the worst ratios at bench.py's user shape (512 x T 50 x 15 heads) are
    ctx 0.55, dQ 0.997, dK 0.997, dV 0.997; in the negative-score regime at that shape 0.56 / 0.997 / 0.996 / 0.997.  The
    gradients' worst elements sit at half an ulp: their bound is one output rounding plus a spread that is 0 wherever no bf16
    flip is possible.

Grid rounds follow launch_mma's rule (restated in gpu_checks.core_launch_grid) on whatever GPU runs the file: nr_num_sms()."""
import pytest

import gpu_checks as G

pytestmark = pytest.mark.gpu


def _sms():
    from newsrec_b200 import load_library
    return int(load_library().nr_num_sms())


def assert_core(r, p_drop=0.0, regime="unit"):
    assert r["fwd_rc"] == 0 and r["bwd_rc"] == 0, r
    assert r["guards_intact"] and r["ctx_ones_col"] and r["ctx_tail_zero"], r
    assert r["dqkv_section_pad_zero"] and r["dqkv_tail_prefill_kept"], r
    assert r["ctx_dropped_nonzero"] == 0 and (r["ctx_dropped"] > 0) == (p_drop > 0), r
    assert r["fwd_deterministic"] and r["bwd_deterministic"], r
    if regime == "flush":
        assert r["flushed_to_zero"], r
        return
    assert r["outputs_finite"], r
    for k in ("ctx_ratio", "dQ_ratio", "dK_ratio", "dV_ratio"):
        assert r[k] <= 1.0, (k, r)


def assert_discriminates(r, heads, T, p_drop):
    if heads > 1:
        assert r["ctx_neighbour_head_ratio"] >= 8, r
    if T > 1:
        assert r["ctx_no_last_key_ratio"] >= 8, r
    if p_drop > 0:
        assert r["ctx_neighbour_row_mask_ratio"] >= 8, r
    assert r["dV_unrounded_A_ratio"] >= 8, r


# ---- the dispatch matrix ----------------------------------------------------------------------------------------------------
# (n_seq, T, heads, d_k, sec): sec None = round_up(d, 8) (the encoders' sections), "dense" = d, or an explicit stride
_DK = [(2, "dense"), (3, None), (8, "dense"), (9, None), (15, "dense"), (16, None), (17, "dense"), (24, None), (25, "dense"),
       (31, None), (32, "dense")]
_CASES = (
    # NTD 2 / 3 / 4 over d_k at a per-warp length; odd d_k: 2-byte pieces, d_k = 2 (mod 4): 4-byte pieces
    [dict(n_seq=9, T=17, heads=3, dk=dk, sec=s) for dk, s in _DK]
    + [dict(n_seq=9, T=12, heads=5, dk=18, sec="dense"), dict(n_seq=9, T=12, heads=5, dk=10, sec=None),
       dict(n_seq=9, T=12, heads=3, dk=8, sec=25),                  # odd dense section stride: 2-byte pieces at d_k 8
       # the copy-plan limit T * d_k / (piece / 2) <= 128: T = 32 at d_k 16 (128: plan) and 20 (160: loops), T = 24 at 20 (120)
       dict(n_seq=7, T=32, heads=4, dk=16, sec="dense"), dict(n_seq=7, T=32, heads=4, dk=20, sec="dense"),
       dict(n_seq=7, T=24, heads=4, dk=20, sec=None)]
    # per-warp lengths, cooperative lengths
    + [dict(n_seq=11, T=T, heads=4, dk=12, sec=None if T % 2 else "dense") for T in (1, 2, 15, 16, 17, 31, 32)]
    + [dict(n_seq=5, T=T, heads=3, dk=20, sec=None if T % 2 else "dense") for T in (33, 48, 49, 63, 64)]
    # the fixed-shape kernels: T = 20 on dense sections of 300 (MhsaFn's path), T = 50 (the user level, both layouts)
    + [dict(n_seq=13, T=20, heads=15, dk=20, sec="dense"), dict(n_seq=5, T=50, heads=15, dk=20, sec=None),
       dict(n_seq=5, T=50, heads=15, dk=20, sec="dense")]
    # the title kernels through the raw ABI (sectioned)
    + [dict(n_seq=7, T=20, heads=h, dk=20, sec=None) for h in (1, 2, 7, 15)]
    # the former whole-tensor cases, at the encoders' natural pitches (no extra columns)
    + [dict(n_seq=2000, T=20, heads=15, dk=20, sec="dense", pad=0), dict(n_seq=5, T=16, heads=30, dk=10, sec="dense", pad=0),
       dict(n_seq=5, T=33, heads=20, dk=15, sec="dense", pad=0), dict(n_seq=4, T=64, heads=10, dk=30, sec="dense", pad=0),
       dict(n_seq=9, T=7, heads=12, dk=25, sec="dense", pad=0), dict(n_seq=9, T=7, heads=12, dk=25, sec=None, pad=0),
       dict(n_seq=3, T=40, heads=6, dk=20, sec="dense", pad=0), dict(n_seq=301, T=20, heads=4, dk=20, sec=None, pad=0),
       dict(n_seq=40, T=20, heads=9, dk=20, sec=None, pad=0), dict(n_seq=9, T=12, heads=8, dk=9, sec="dense", pad=0),
       dict(n_seq=5, T=24, heads=15, dk=20, sec="dense", pad=0), dict(n_seq=5, T=20, heads=5, dk=18, sec="dense", pad=0),
       dict(n_seq=6, T=8, heads=4, dk=32, sec="dense", pad=0), dict(n_seq=1, T=20, heads=15, dk=20, sec=None, pad=0),
       dict(n_seq=2000, T=20, heads=15, dk=20, sec=None, pad=0), dict(n_seq=3, T=50, heads=15, dk=20, sec=None, pad=0)]
)


def _kw(c):
    c = dict(c)
    s = c.pop("sec")
    if s == "dense":
        c["sec"] = c["heads"] * c["dk"]
    elif s is None:
        c["sectioned"] = True
    else:
        c["sec"] = s
    return c


def _id(c):
    s = {"dense": "dense", None: "sect"}.get(c["sec"], f"sec{c['sec']}")
    return f"n{c['n_seq']}-T{c['T']}-h{c['heads']}-dk{c['dk']}-{s}" + ("-pad0" if c.get("pad") == 0 else "")


@pytest.mark.parametrize("p_drop", [0.0, 0.2])
@pytest.mark.parametrize("case", _CASES, ids=[_id(c) for c in _CASES])
def test_core_dispatch_matrix(case, p_drop):
    r = G.check_mhsa_core(p_drop=p_drop, seed=case["T"] + case["dk"], **_kw(case))
    assert_core(r, p_drop)


# ---- score regimes ----------------------------------------------------------------------------------------------------------
_REGIME_SHAPES = [dict(n_seq=9, T=17, heads=3, dk=16, sec="dense"), dict(n_seq=9, T=20, heads=15, dk=20, sec=None),
                  dict(n_seq=5, T=50, heads=15, dk=20, sec=None), dict(n_seq=5, T=64, heads=2, dk=32, sec="dense"),
                  dict(n_seq=9, T=23, heads=4, dk=3, sec=None)]


@pytest.mark.parametrize("regime", ["saturated", "negative", "flush"])
@pytest.mark.parametrize("case", _REGIME_SHAPES, ids=[_id(c) for c in _REGIME_SHAPES])
def test_core_score_regimes(case, regime):
    """saturated: |S| up to about 60, A nearly one-hot; negative: every score in [-58, -25], where the +1e-8 of the
    denominator dominates and the context shrinks by orders of magnitude (only there would a kernel without the
    1e-8 exp2(-max) correction be wrong); flush: every score below -95, the context and the gradients are exactly 0."""
    r = G.check_mhsa_core(p_drop=0.2, regime=regime, seed=7, **_kw(case))
    assert_core(r, 0.2, regime)


# ---- discrimination ---------------------------------------------------------------------------------------------------------
_DISC = [dict(n_seq=9, T=17, heads=3, dk=16, sec="dense"), dict(n_seq=7, T=32, heads=4, dk=20, sec="dense"),
         dict(n_seq=5, T=50, heads=15, dk=20, sec=None), dict(n_seq=13, T=20, heads=15, dk=20, sec="dense"),
         dict(n_seq=7, T=20, heads=7, dk=20, sec=None), dict(n_seq=5, T=63, heads=3, dk=9, sec="dense")]


@pytest.mark.parametrize("regime", ["unit", "negative"])
@pytest.mark.parametrize("case", _DISC, ids=[_id(c) for c in _DISC])
def test_core_bounds_discriminate(case, regime):
    """One shape per kernel family: the references a subtly wrong kernel would match miss the bound by >= 8x."""
    r = G.check_mhsa_core(p_drop=0.2, regime=regime, seed=11, **_kw(case))
    assert_core(r, 0.2, regime)
    assert_discriminates(r, case["heads"], case["T"], 0.2)


# ---- grid rounds ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["1", "W-1", "W", "W+1", "2W+1", "3W+2"])
@pytest.mark.parametrize("direction", ["fwd", "bwd"])
@pytest.mark.parametrize("T", [20, 40])
def test_core_grid_rounds(T, direction, which):
    """One head per sequence, so that tasks = n_seq: a single task, one short of a full round of W tasks, exactly one, one
    over, and several rounds in which some warps (CTAs) run an odd and others an even number of tasks through the two-stage
    copy ring.  W is the round of the direction named (per-warp at T = 20, cooperative at T = 40)."""
    W = G.core_launch_grid(T, 16, 1, direction == "bwd", _sms())
    n_seq = {"1": 1, "W-1": W - 1, "W": W, "W+1": W + 1, "2W+1": 2 * W + 1, "3W+2": 3 * W + 2}[which]
    r = G.check_mhsa_core(n_seq=n_seq, T=T, heads=1, dk=16, sec=16, p_drop=0.2, seed=n_seq)
    assert_core(r, 0.2)


# ---- bench points -----------------------------------------------------------------------------------------------------------
def test_core_user_bench_shape():
    """bench.py's history level: 512 users x 50 clicked news x 15 heads (the fixed-shape cooperative kernels, both ways)."""
    r = G.check_mhsa_core(n_seq=512, T=50, heads=15, dk=20, sectioned=True, pad=0, p_drop=0.0, seed=50)
    assert_core(r, 0.0)
    assert_discriminates(r, 15, 50, 0.0)


def test_core_title_mid_size():
    """The title kernels over 3000 titles: many titles per CTA."""
    r = G.check_mhsa_core(n_seq=3000, T=20, heads=15, dk=20, sectioned=True, pad=0, p_drop=0.2, seed=51)
    assert_core(r, 0.2)


# ---- the shape contract -----------------------------------------------------------------------------------------------------
_BAD = [
    (dict(T=0), "sequence length"), (dict(T=65), "sequence length"), (dict(dk=1), "head size"), (dict(dk=33), "head size"),
    (dict(heads=0), "heads=0"), (dict(n_seq=-1), "n_seq=-1"), (dict(sec=31), "section stride"),
    (dict(ld_qkv=100), "Q|K|V pitch 100 is not a multiple of 8"),
]
_BAD_FWD = [(dict(ld_ctx=32), "ones column"), (dict(ld_ctx=34), "context pitch 34 is not a multiple of 8"),
            (dict(p_drop=-0.1), "dropout p"), (dict(p_drop=1.0), "dropout p"), (dict(p_drop=float("nan")), "dropout p")]
_BAD_BWD = [(dict(ld_dctx=34), "not a multiple of 8"), (dict(ld_dqkv=100), "not a multiple of 8"), (dict(ld_dqkv=88), "too small"),
            (dict(ld_dctx=24), "too small")]


@pytest.mark.parametrize("which,args,rule", [("fwd", a, m) for a, m in _BAD + _BAD_FWD] + [("bwd", a, m) for a, m in _BAD + _BAD_BWD],
                         ids=lambda v: v if isinstance(v, str) else None)
def test_core_rejects_bad_shapes_before_launch(which, args, rule):
    rc, msg, launches, untouched = G.mhsa_core_contract_call(which, **args)
    assert rc == -1 and rule in msg and launches == 0 and untouched, (rc, msg, launches, untouched)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
def test_core_accepts_the_valid_base_shape_and_empty_batches(which):
    """The base shape of the contract calls runs (so each rejection above is its one argument's doing); n_seq = 0 launches
    nothing and writes nothing."""
    rc, msg, launches, _ = G.mhsa_core_contract_call(which)
    assert rc == 0 and launches == 1, (rc, msg, launches)
    rc, msg, launches, untouched = G.mhsa_core_contract_call(which, n_seq=0)
    assert rc == 0 and launches == 0 and untouched, (rc, msg, launches, untouched)


# ---- the standalone MultiHeadSelfAttention ----------------------------------------------------------------------------------
def assert_module(r):
    assert r["ctx_ratio"] <= 1.0, r
    for k in ("dx", "dW_Q", "dW_K", "dW_V"):
        if f"{k}_row_ratio" in r:
            assert r[f"{k}_row_ratio"] <= 1.5, (k, r)
    if "t1_dWqk_rel" in r:  # T = 1: the W_Q, W_K gradients are 1e-8 of W_V's (see check_mhsa_module)
        assert r["t1_dWqk_rel"] <= 1e-6, r


@pytest.mark.parametrize("kw", [
    dict(N=37, T=20, d=300, heads=15),                   # the fixed-shape per-warp kernel on dense sections
    dict(N=13, T=50, d=300, heads=15),                   # the fixed-shape cooperative kernel
    dict(N=29, T=20, d=64, heads=4),                     # d_k 16: NTD 2, copy plan
    dict(N=41, T=1, d=300, heads=15),                    # one token: A = 1 / (1 + 1e-8)
    dict(N=17, T=20, d=300, heads=15, noncontig=True),   # a (T, N, d) tensor seen as (N, T, d)
    dict(N=9, T=20, d=512, heads=16),                    # d + 1 > 512: the weight gradient in two launches
], ids=["d300-T20", "d300-T50", "d64-h4", "T1", "noncontig", "d512-h16"])
def test_multihead_self_attention_module(kw):
    assert_module(G.check_mhsa_module(**kw))


def test_multihead_self_attention_module_after_optimizer_step():
    """After optimizer.step() the next call reads the new weights through the operand cache."""
    r = G.check_mhsa_module(N=11, T=20, d=300, heads=15, step=True)
    assert_module(r)
    assert r["ctx_old_weights_ratio"] >= 8, r
