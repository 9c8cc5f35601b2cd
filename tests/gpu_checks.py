"""Kernel-vs-oracle checks, written as plain functions returning error metrics so that both the pytest
wrappers (tests/test_gpu_*.py) and the triage ladder (tools/gpu_ladder.py) can run them.

Everything goes through the C ABI (ctypes) or through the drop-in model package that calls it.
The oracle (oracle/newsrec_oracle.py) runs on the CPU; it is the checker, never the thing measured.
"""
from __future__ import annotations

import ctypes as C
import math

import torch

import newsrec_oracle as O
from newsrec_b200 import check, load_library
from newsrec_b200.ops import _p, _stream, cast_pad, ru8, ru16

DEV = "cuda"


def relerr(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / max(b.norm().item(), 1e-30))


def maxabs(a, b) -> float:
    return float((a.detach().double().cpu() - b.detach().double().cpu()).abs().max())


def bf16r(x):
    return x.to(torch.bfloat16).to(torch.float32)


# ------------------------------------------------------------------------------------------------
def check_prep_and_gather():
    lib = load_library()
    V, D, T, n_seq = 97, 300, 20, 13
    ld = ru8(D + 1)
    w = O.det_uniform((V, D), 5)
    table = cast_pad(w.to(DEV), ld)
    ref = torch.zeros(V, ld)
    ref[:, :D] = bf16r(w)
    out = {"cast_pad_exact": bool(torch.equal(table.float().cpu(), ref))}
    wt = cast_pad(w.to(DEV), ru8(V), transpose=True)
    reft = torch.zeros(D, ru8(V))
    reft[:, :V] = bf16r(w).t()
    out["cast_pad_T_exact"] = bool(torch.equal(wt.float().cpu(), reft))
    ids = O.synth_titles(n_seq, T, V, 77).to(DEV)
    X = torch.full((n_seq * T, ld), 7.0, dtype=torch.bfloat16, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    check(lib.nr_gather_rows(_p(ids), n_seq * T, T, _p(table), V, D, ld, _p(X), 0, 0.0, 0, _p(flag), _stream()), "gather")
    expect = ref[ids.cpu().reshape(-1)]
    expect[:, D] = 1.0
    out["gather_exact"] = bool(torch.equal(X.float().cpu(), expect)) and int(flag.item()) == 0
    # padded CNN layout
    Xp = torch.full((n_seq * (T + 2), ld), 7.0, dtype=torch.bfloat16, device=DEV)
    check(lib.nr_gather_rows(_p(ids), n_seq * T, T, _p(table), V, D, ld, _p(Xp), 1, 0.0, 0, _p(flag), _stream()), "gather")
    Xp3 = Xp.float().cpu().view(n_seq, T + 2, ld)
    out["gather_padded_exact"] = bool(torch.equal(Xp3[:, 1:T + 1].reshape(-1, ld), expect)) and \
        float(Xp3[:, 0].abs().sum() + Xp3[:, T + 1].abs().sum()) == 0.0
    # out-of-range id sets the flag
    bad = ids.clone()
    bad[0, 0] = V + 5
    check(lib.nr_gather_rows(_p(bad), n_seq * T, T, _p(table), V, D, ld, _p(X), 0, 0.0, 0, _p(flag), _stream()), "gather")
    out["bad_id_flag"] = int(flag.item()) == 1
    # dropout: keep-rate and scaling
    big = O.synth_titles(2000, T, V, 78, min_len=T).to(DEV)
    Xd = torch.empty((2000 * T, ld), dtype=torch.bfloat16, device=DEV)
    flag.zero_()
    check(lib.nr_gather_rows(_p(big), 2000 * T, T, _p(table), V, D, ld, _p(Xd), 0, 0.2, 1234, _p(flag), _stream()), "gather")
    e = ref[big.cpu().reshape(-1)][:, :D]
    got = Xd.float().cpu()[:, :D]
    kept = got != 0
    out["dropout_keep_rate"] = float(kept.float().mean() / (e != 0).float().mean())
    ratio = (got[kept] / e[kept])
    out["dropout_scale_err"] = float((ratio - 1.25).abs().max())
    out["dropout_ones_col_intact"] = bool((Xd[:, D].float() == 1).all())
    return out


# ------------------------------------------------------------------------------------------------
def _rand_bf16(shape, seed, scale=1.0):
    return bf16r(O.det_uniform(shape, seed, -scale, scale))


def check_linear(M=300, N=900, K=300, taps=1, seg=0, relu=0, out_bf16=1):
    """nr_linear (wgmma gemm_nt + store epilogue) against an fp64 matmul of the same bf16 operands: the norm-wise error and
    the worst element against its bound (gemm_elem_ratio, <= 1)."""
    lib = load_library()
    lda, ldw = ru8(K + 1), ru8(K + 1)
    if taps == 1:
        A = _rand_bf16((M, K), 1)
        W = _rand_bf16((N, K), 2, 0.1)
        bias = O.det_uniform((N,), 3, -0.5, 0.5)
        Ad = torch.zeros(M, lda)
        Ad[:, :K] = A
        Wd = torch.zeros(N, ldw)
        Wd[:, :K] = W
        rpt, w_tap_rows = 128, 0
    else:  # window-3 conv over the padded layout: seg tokens per segment, M = n_seg*(seg+2) rows
        n_seg = M
        Mrows = n_seg * (seg + 2)
        X = _rand_bf16((n_seg, seg, K), 1)
        W = _rand_bf16((N, taps, K), 2, 0.1)
        bias = O.det_uniform((N,), 3, -0.5, 0.5)
        Xp = torch.zeros(n_seg, seg + 2, K)
        Xp[:, 1:seg + 1] = X
        Ad = torch.zeros(Mrows, lda)
        Ad[:, :K] = Xp.view(Mrows, K)
        Wd = torch.zeros(taps * N, ldw)
        for s in range(taps):
            Wd[s * N:(s + 1) * N, :K] = W[:, s]
        M = Mrows
        rpt, w_tap_rows = (128 // (seg + 2)) * (seg + 2), N
    ld_out = ru8(N) if out_bf16 else (N + 3) // 4 * 4
    out = torch.full((M, ld_out), float("nan"), dtype=torch.bfloat16 if out_bf16 else torch.float32, device=DEV)
    Ad, Wd, bd = Ad.to(torch.bfloat16).to(DEV), Wd.to(torch.bfloat16).to(DEV), bias.to(DEV)
    check(lib.nr_linear(_p(Ad), M, lda, _p(Wd), N, ldw, K, taps, w_tap_rows, rpt, _p(bd), relu, _p(out), ld_out, out_bf16,
                        _stream()), "nr_linear")
    torch.cuda.synchronize()
    pre, absum = linear_ref(Ad[:, :K].double(), Wd[:, :K].double(), bd.double(), N, taps, w_tap_rows)
    got = out[:, :N]
    ratio, zero_exact = gemm_elem_ratio(got, pre, absum, taps * -(-K // 16), out_bf16, relu)
    ref = pre.clamp_min(0) if relu else pre
    if taps > 1:  # pad rows of the padded layout are not part of the result
        keep = torch.ones(M, dtype=torch.bool, device=DEV).view(-1, seg + 2)
        keep[:, 0] = keep[:, -1] = False
        keep = keep.view(-1)
        got, ref = got[keep], ref[keep]
    got = got.float()
    return {"rel": relerr(got, ref), "maxabs": maxabs(got, ref), "nan": int(torch.isnan(got).sum()), "elem_ratio": ratio,
            "relu_zero_exact": zero_exact}


def linear_ref(A, W, bias, N, taps=1, w_tap_rows=0, tap_origin=None):
    """fp64 pre-activation of nr_linear and the sum of |products| + |bias| per element: tap s reads A shifted by s - tap_origin
    rows (tap_origin None: taps // 2; zero outside A) against weight rows [s * w_tap_rows, + N).  A [M][K], W [rows][K], bias [N]
    or None (fp64 device)."""
    M = A.shape[0]
    pre = torch.zeros(M, N, dtype=torch.float64, device=A.device)
    absum = torch.zeros_like(pre)
    for s in range(taps):
        d = s - (taps // 2 if tap_origin is None else tap_origin)
        As = torch.zeros_like(A)
        lo, hi = max(0, -d), min(M, M - d)
        if hi > lo:
            As[lo:hi] = A[lo + d:hi + d]
        Ws = W[s * w_tap_rows:s * w_tap_rows + N]
        pre += As @ Ws.t()
        absum += As.abs() @ Ws.abs().t()
    if bias is not None:
        pre += bias
        absum += bias.abs()
    return pre, absum


def check_gemm_tn(Kr=1000, Ma=900, Nb=301, shift=0):
    """nr_gemm_tn (+= onto ones) against an fp64 evaluation of the same bf16 operands: the norm-wise error and the worst element
    against its bound (gemm_elem_ratio with n_acc = ceil(Kr/16) + the k-ranges' red.add, <= 1)."""
    import gemm_plan_ref as P
    lib = load_library()
    lda, ldb = ru8(Ma), ru8(Nb)
    A = _rand_bf16((Kr, Ma), 11, 0.5)
    B = _rand_bf16((Kr, Nb), 12, 0.5)
    Ad = torch.zeros(Kr, lda)
    Ad[:, :Ma] = A
    Bd = torch.zeros(Kr, ldb)
    Bd[:, :Nb] = B
    ldd = ru8(Nb)
    D = torch.full((Ma, ldd), 1.0, dtype=torch.float32, device=DEV)  # accumulate on top of ones
    Ad, Bd = Ad.to(torch.bfloat16).to(DEV), Bd.to(torch.bfloat16).to(DEV)
    check(lib.nr_gemm_tn(_p(Ad), Kr, Ma, lda, _p(Bd), Kr, Nb, ldb, 0, Nb, shift, _p(D), ldd, _stream()), "nr_gemm_tn")
    torch.cuda.synchronize()
    ref, absum = gemm_tn_ref(Ad[:, :Ma].double(), Bd[:, :Nb].double(), shift)
    got = D[:, :Nb] - 1.0
    n_acc = -(-Kr // 16) + P.plan_tn(Kr, Ma, Nb, sms=int(lib.nr_num_sms()))["k_slices_max"]
    ratio, _ = gemm_elem_ratio(D[:, :Nb], ref + 1.0, absum + 1.0, n_acc, 0)
    return {"rel": relerr(got, ref), "maxabs": maxabs(got, ref), "nan": int(torch.isnan(got).sum()), "elem_ratio": ratio}


def gemm_tn_ref(A, B, shift):
    """fp64 A^T . B[rows + shift] (rows of B outside [0, rows) are zero) and the sum of |products|; A [Kr][Ma], B [b_rows][Nb]."""
    Kr, rows = A.shape[0], B.shape[0]
    Bs = torch.zeros(Kr, B.shape[1], dtype=B.dtype, device=B.device)
    lo, hi = max(0, -shift), min(Kr, rows - shift)
    if hi > lo:
        Bs[lo:hi] = B[lo + shift:hi + shift]
    return A.t() @ Bs, A.abs().t() @ Bs.abs()


# ------------------------------------------------------------------------------------------------
def mhsa_core_inputs(n, T, heads, dk, regime, seed, device=DEV):
    """Q, K, V, dC (n, T, d) as fp64 tensors of bf16 values in one of the score regimes of tests/test_gpu_mhsa_core.py:
    "unit" (scores of standard deviation 1), "saturated" (standard deviation 16, |S| up to about 60: A nearly one-hot),
    "negative" (every score in [-58, -25]: the +1e-8 dominates the softmax denominator) and "flush" (every score below -95:
    the kernels' exp2(-max) overflows and the context flushes to zero)."""
    d = heads * dk
    u = lambda s, lo, hi: O.det_uniform((n, T, d), seed + s, lo, hi).to(device).double()
    if regime in ("unit", "saturated"):
        a = math.sqrt(3.0) if regime == "unit" else 7.0
        Q, K = u(1, -a, a), u(2, -a, a)
    else:  # S = -(c / d_k) sum_c u_c v_c with u, v in [0.8, 1.2]: S in -c [0.64, 1.44]
        c = 40.0 if regime == "negative" else 150.0
        a = math.sqrt(c / math.sqrt(dk))
        Q, K = -a * u(1, 0.8, 1.2), a * u(2, 0.8, 1.2)
    r = lambda t: t.to(torch.bfloat16).double()
    return r(Q), r(K), r(u(3, -1.0, 1.0)), r(u(4, -1.0, 1.0))


def core_launch_grid(T, dk, heads, bwd, sms, fixed=False):
    """Tasks per full grid round of the head-level kernels (attn.cu launch_mma: per_sm from the tile sets' shared memory, the
    grid capped at SMs x per_sm CTAs of kWarps = 4 per-warp tasks, or one task per cooperative CTA)."""
    coop = T > 32
    TP, PT = (64 if coop else 32), (24 if fixed else 40)
    tile = 2 * T * PT
    sets = 1 if coop else 4
    smem = sets * (2 * 4 * tile + 2 * 2 * TP * (TP + 8)) if bwd else sets * 2 * 3 * tile + 2 * (TP - T) * PT
    per_sm = max(1, min(3 if coop else (6 if bwd else 8), (224 * 1024) // (smem + 1024)))
    return sms * per_sm * (1 if coop else 4)


def check_mhsa_core(n_seq=7, T=20, heads=15, dk=20, sectioned=False, sec=None, pad=8, p_drop=0.0, regime="unit", seed=1,
                    extra=True):
    """nr_mhsa_core_fwd / _bwd through the C ABI against the fp64 references of tests/mhsa_core_ref.py, element by element.
    Q | K | V at columns 0, sec, 2 sec of rows of pitch ld3 (sec = round_up(d, 8) when sectioned, else d, or as given);
    pad = extra columns behind the natural pitches (ld3 = round_up(3 sec, 16), ldx = round_up(d + 1, 8), dCtx round_up(d, 8)).
    Every input column the kernels must not read holds NaN (section padding, [3 sec, ld3), dCtx [d, ld_dctx)), every "="
    output starts as NaN, every buffer is followed by a guard.  extra: discrimination references and the determinism reruns.
    Bounds: tests/test_gpu_mhsa_core.py."""
    import mhsa_core_ref as R
    lib = load_library()
    d = heads * dk
    if sec is None:
        sec = ru8(d) if sectioned else d
    ld3, ldx, ldc = ru16(3 * sec) + pad, ru8(d + 1) + pad, ru8(d) + pad
    n_tok = n_seq * T
    nan = float("nan")
    Q, K, V, dC = mhsa_core_inputs(max(n_seq, 1), T, heads, dk, regime, seed)
    qkv = _Guarded(n_tok * ld3, torch.bfloat16, nan)
    dct = _Guarded(n_tok * ldc, torch.bfloat16, nan)
    if n_seq:
        q2 = qkv.body.view(n_tok, ld3)
        for i, t in enumerate((Q, K, V)):
            q2[:, i * sec:i * sec + d] = t.reshape(n_tok, d).to(torch.bfloat16)
        dct.body.view(n_tok, ldc)[:, :d] = dC.reshape(n_tok, d).to(torch.bfloat16)
    kseed = (0x9E3779B97F4A7C15 * (seed + 17)) & 0xFFFFFFFFFFFFFFFF

    def fwd():
        out = _Guarded(n_tok * ldx, torch.bfloat16, nan)
        n0 = int(lib.nr_launch_count())
        rc = lib.nr_mhsa_core_fwd(_p(qkv.all), ld3, sec, n_seq, T, heads, dk, _p(out.all), ldx, float(p_drop), kseed, _stream())
        return out, rc, int(lib.nr_launch_count()) - n0

    def bwd():
        out = _Guarded(n_tok * ld3, torch.bfloat16, nan)
        n0 = int(lib.nr_launch_count())
        rc = lib.nr_mhsa_core_bwd(_p(qkv.all), ld3, sec, _p(dct.all), ldc, n_seq, T, heads, dk, _p(out.all), ld3, _stream())
        return out, rc, int(lib.nr_launch_count()) - n0

    cb, rcf, lf = fwd()
    db, rcb, lb = bwd()
    torch.cuda.synchronize()
    res = {"fwd_rc": rcf, "bwd_rc": rcb, "fwd_launches": lf, "bwd_launches": lb,
           "msg": lib.nr_last_error().decode() if (rcf or rcb) else ""}
    if rcf or rcb or n_seq == 0:
        res["guards_intact"] = all(g.guard_ok() for g in (qkv, dct, cb, db))
        return res
    C2, D2 = cb.body.view(n_seq, T, ldx), db.body.view(n_seq, T, ld3)
    got_c = C2[..., :d].double()
    got = {k: D2[..., i * sec:i * sec + d].double() for i, k in enumerate(("dQ", "dK", "dV"))}
    rows = torch.arange(n_tok, device=DEV)
    cm = dropout_mask_dev(kseed, p_drop, rows, d, ldx).double().view(n_seq, T, d)
    # ---- exact outputs
    res["ctx_ones_col"] = bool((C2[..., d] == 1).all())
    res["ctx_tail_zero"] = bool((C2[..., d + 1:] == 0).all())
    res["ctx_dropped_nonzero"] = int(((cm == 0) & (got_c != 0)).sum())
    res["ctx_dropped"] = int((cm == 0).sum())
    res["dqkv_section_pad_zero"] = all(bool((D2[..., i * sec + d:(i + 1) * sec] == 0).all()) for i in range(3))
    res["dqkv_tail_prefill_kept"] = bool(torch.isnan(D2[..., 3 * sec:].float()).all())
    res["guards_intact"] = all(g.guard_ok() for g in (qkv, dct, cb, db))
    res["outputs_finite"] = bool(torch.isfinite(got_c).all()) and all(bool(torch.isfinite(g).all()) for g in got.values())
    if regime == "flush":  # every exp2(-max) overflows: the context and every gradient are exactly zero
        res["flushed_to_zero"] = bool((got_c == 0).all()) and all(bool((g == 0).all()) for g in got.values())
    # ---- element bounds, a chunk of sequences at a time
    acc = {k: 0.0 for k in ("ctx_ratio", "dQ_ratio", "dK_ratio", "dV_ratio", "ctx_neighbour_head_ratio", "ctx_no_last_key_ratio",
                            "ctx_neighbour_row_mask_ratio", "dV_unrounded_A_ratio")}
    worst = {}

    def note(k, t, s0):
        v = _worst(t)
        if v >= acc[k]:
            acc[k] = v
            i = int(torch.nan_to_num(t, nan=float("inf")).reshape(-1).argmax())
            worst[k] = [s0 + i // (T * d), (i // d) % T, i % d]

    cm_next = dropout_mask_dev(kseed, p_drop, rows + 1, d, ldx).double().view(n_seq, T, d) if p_drop > 0 else None
    cs = max(1, (1 << 22) // (heads * T * T))
    for s0 in range(0, n_seq, cs):
        s = slice(s0, min(n_seq, s0 + cs))
        q, k, v, g, m = Q[s], K[s], V[s], dC[s], cm[s]
        ref_c, spread_c = R.context_bound(q, k, v, heads, m)
        note("ctx_ratio", R.judge_context(got_c[s], ref_c, spread_c, m), s0)
        refs, spread = R.grad_bounds(q, k, v, g, heads)
        for key in ("dQ", "dK", "dV"):
            note(key + "_ratio", R.judge_grad(got[key][s], refs[key], spread[key]), s0)
        if extra:  # discrimination: references a subtly wrong kernel would match instead
            if heads > 1:
                note("ctx_neighbour_head_ratio", R.judge_context(got_c[s], R.neighbour_head(ref_c, heads), spread_c, m), s0)
            if T > 1:
                ref_nl = R.forward(q, k, v, heads, keys=T - 1)[0] * m
                note("ctx_no_last_key_ratio", R.judge_context(got_c[s], ref_nl, spread_c, m), s0)
            if cm_next is not None:
                ref_nm = R.forward(q, k, v, heads)[0] * cm_next[s]
                note("ctx_neighbour_row_mask_ratio", R.judge_context(got_c[s], ref_nm, spread_c, m), s0)
            ref_ua = R.backward(q, k, v, g, heads)["dV"]
            note("dV_unrounded_A_ratio", R.judge_grad(got["dV"][s], ref_ua, spread["dV"]), s0)
        del ref_c, spread_c, refs, spread
    res.update(acc)
    res["worst_at"] = worst
    if extra:  # determinism: the core has no atomics
        cb2, _, _ = fwd()
        db2, _, _ = bwd()
        torch.cuda.synchronize()
        res["fwd_deterministic"] = _bits_equal(cb.body, cb2.body)
        res["bwd_deterministic"] = _bits_equal(db.body, db2.body)
    return res


def mhsa_core_contract_call(which, **args):
    """nr_mhsa_core_fwd / _bwd with the given arguments and a valid small shape for the others (2 sequences of 20 rows, 2 heads
    of d_k 16), on real guarded buffers large enough for any shape the contract tests pass (2 x 65 rows of 256 columns).
    Returns the return code, the message, the launches and whether every buffer (and its guard) is untouched."""
    lib = load_library()
    a = dict(n_seq=2, T=20, heads=2, dk=16, sec=32, ld_qkv=104, ld_ctx=40, ld_dctx=40, ld_dqkv=104, p_drop=0.0)
    a.update(args)
    n = 2 * 65 * 256
    src = O.det_uniform((n,), 5).to(DEV)
    bufs = [_Guarded(n, torch.bfloat16, src) for _ in range(3)]
    n0 = int(lib.nr_launch_count())
    if which == "fwd":
        rc = lib.nr_mhsa_core_fwd(_p(bufs[0].all), a["ld_qkv"], a["sec"], a["n_seq"], a["T"], a["heads"], a["dk"], _p(bufs[1].all),
                                  a["ld_ctx"], float(a["p_drop"]), 7, _stream())
    else:
        rc = lib.nr_mhsa_core_bwd(_p(bufs[0].all), a["ld_qkv"], a["sec"], _p(bufs[1].all), a["ld_dctx"], a["n_seq"], a["T"], a["heads"],
                                  a["dk"], _p(bufs[2].all), a["ld_dqkv"], _stream())
    launches = int(lib.nr_launch_count()) - n0
    msg = lib.nr_last_error().decode() if rc else ""
    torch.cuda.synchronize()
    untouched = all(b.guard_ok() and b.unchanged(torch.ones(n, dtype=torch.bool, device=DEV)) for b in bufs)
    return rc, msg, launches, untouched


def check_mhsa_module(N=37, T=20, d=300, heads=15, seed=3, noncontig=False, step=False, grad_floor=2e-3):
    """The standalone MultiHeadSelfAttention (ops.MhsaFn: bf16 rows, the Q|K|V projection, the dense-section core, and back)
    against oracle.multihead_self_attention in fp64 on the module's bf16 operands: the context element by element from the
    Q|K|V the forward stored, every gradient per row ([W | b] rows, input rows) against the exact chain next to the bf16
    contract's error.  step: an SGD step first, then the same checks on the next call (the operand cache must rebuild), and
    the context against the old weights' reference as a discrimination."""
    import mhsa_core_ref as R
    from model.general.attention.multihead_self import MultiHeadSelfAttention
    torch.manual_seed(seed)
    m = MultiHeadSelfAttention(d, heads).to(DEV)
    base = O.det_uniform((T, N, d), seed + 1, -2.0, 2.0).to(DEV)
    x = base.transpose(0, 1) if noncontig else base.transpose(0, 1).contiguous()
    dout = O.det_uniform((N, T, d), seed + 2).to(DEV)
    names = [f"W_{k}" for k in "QKV"]

    def params64():
        p = {}
        for n in names:
            lin = getattr(m, n)
            p[f"m.{n}.weight"] = lin.weight.detach().to(torch.bfloat16).double().requires_grad_(True)
            p[f"m.{n}.bias"] = lin.bias.detach().double().requires_grad_(True)
        return p

    def run():
        m.zero_grad(set_to_none=True)
        xi = x.detach().clone().requires_grad_(True) if not noncontig else x.detach().requires_grad_(True)
        out = m(xi)
        QKV = out.grad_fn.saved_tensors[1].double()
        out.backward(dout)
        return xi, out.detach().double(), QKV

    res = {}
    if step:
        run()
        old = params64()
        # a step of up to 30 % of each weight (the backward's own gradients would move the scores past what the oracle's
        # exp without max-subtraction can hold in fp64)
        for i, t in enumerate(m.parameters()):
            t.grad = 0.3 * t.detach() * O.det_uniform(tuple(t.shape), seed + 10 + i).to(DEV)
        torch.optim.SGD(m.parameters(), lr=1.0).step()
    xi, got, QKV = run()
    xb = x.detach().to(torch.bfloat16).double()
    Q, K, V = (QKV[:, i * d:(i + 1) * d].reshape(N, T, d) for i in range(3))
    ones = torch.ones(N, T, d, dtype=torch.float64, device=DEV)
    ref, spread = R.context_bound(Q, K, V, heads, ones)
    res["ctx_ratio"] = _worst(R.judge_context(got, ref, spread, ones))
    grads = {}
    for v, c in (("exact", O.EXACT), ("contract", O.BF16)):
        p = params64()
        xr = xb.clone().requires_grad_(True)
        O.multihead_self_attention(xr, p, "m", heads, c).backward(dout.double())
        grads[v] = dict(x=xr.grad.reshape(N * T, d), **{n: torch.cat([p[f"m.{n}.weight"].grad, p[f"m.{n}.bias"].grad.view(-1, 1)], 1)
                                                        for n in names})
    kern = dict(x=xi.grad.double().reshape(N * T, d),
                **{n: torch.cat([getattr(m, n).weight.grad, getattr(m, n).bias.grad.view(-1, 1)], 1).double() for n in names})
    # T = 1: A = 1 / (1 + 1e-8), so dS = A (dA - A dA) / sqrt(d_k) is 1e-8 of dA -- below fp32 resolution, the kernels' dQ, dK
    # are 0 -- and the W_Q, W_K gradients are 1e-8 of W_V's: they are held to that scale, the rest to the rule
    judged = [k for k in kern if not (T == 1 and k in ("W_Q", "W_K"))]
    for k in judged:
        res[f"d{k}_row_ratio"], res[f"d{k}_ek"], res[f"d{k}_ec"] = _row_ratio(kern[k], grads["exact"][k], grads["contract"][k],
                                                                              floor=grad_floor)
    if T == 1:
        res["t1_dWqk_rel"] = max(_worst(kern[k].abs()) for k in ("W_Q", "W_K")) / max(_worst(grads["exact"]["W_V"].abs()), 1e-300)
    if step:  # the context of the old weights must be far from what the new call computed
        with torch.no_grad():
            old_ctx = O.multihead_self_attention(xb, old, "m", heads, O.EXACT)
        res["ctx_old_weights_ratio"] = _worst(R.judge_context(got, old_ctx, spread, ones))
    return res


def check_additive(N=37, S=20, D=300, q=200, precision="fast"):
    """precision "accurate": fp32 rows that are not bf16 values enter as hi/lo planes (nr_additive_attention_fwd_hilo, as
    NAML's view fusion and Exp1's final attention run it).  The forward is compared with the oracle's hi/lo contract (scores
    on the hi plane, the pooled sum on the fp32 rows); the backward reads the hi plane in both modes, so its gradients are
    compared with the bf16 contract's gradients at the hi plane bf16(x)."""
    from newsrec_b200.ops import AdditiveAttentionFn, OperandCache
    accurate = precision == "accurate"
    xf = O.det_uniform((N, S, D), 31) if accurate else _rand_bf16((N, S, D), 31)
    x = bf16r(xf).requires_grad_(True)  # the leaf of the gradient reference: the plane the backward reads
    p = {"a.linear.weight": O.det_uniform((q, D), 32, -0.1, 0.1).requires_grad_(True),
         "a.linear.bias": O.det_uniform((q,), 33, -0.05, 0.05).requires_grad_(True),
         "a.attention_query_vector": O.det_uniform((q,), 34, -0.1, 0.1).requires_grad_(True)}
    g = O.det_uniform((N, D), 35)
    O.additive_attention(x, p, "a", O.BF16).backward(g)
    with torch.no_grad():
        ref = O.additive_attention(xf, p, "a", O.BF16_FUSED if accurate else O.BF16)
    xd = xf.to(DEV).requires_grad_(True)
    pd = {k: v.detach().to(DEV).requires_grad_(True) for k, v in p.items()}
    out = AdditiveAttentionFn.apply(xd, pd["a.linear.weight"], pd["a.linear.bias"], pd["a.attention_query_vector"],
                                    OperandCache(), "t", precision)
    out.backward(g.to(DEV))
    torch.cuda.synchronize()
    # the forward element by element (additive_fwd_judge) from the operands it read: bf16(x) (and bf16(x - bf16(x)) in
    # accurate mode), bf16(Wa), fp32 ba and qv
    hi = bf16r(xf).to(DEV)
    lo = bf16r(xf.to(DEV) - hi).double().reshape(N * S, D) if accurate else None
    j = additive_fwd_judge(hi.double().reshape(N * S, D), bf16r(p["a.linear.weight"].detach()).double().to(DEV),
                           p["a.linear.bias"].detach().double().to(DEV), p["a.attention_query_vector"].detach().double().to(DEV),
                           S, out.detach(), X_lo=lo)
    return {"fwd_rel": relerr(out, ref), "fwd_elem_ratio": j["out_ratio"], "dx_rel": relerr(xd.grad, x.grad),
            "dW_rel": relerr(pd["a.linear.weight"].grad, p["a.linear.weight"].grad),
            "db_rel": relerr(pd["a.linear.bias"].grad, p["a.linear.bias"].grad),
            "dq_rel": relerr(pd["a.attention_query_vector"].grad, p["a.attention_query_vector"].grad)}


def check_dot_score(B=9, Cn=5, D=300):
    from newsrec_b200.ops import DotScoreFn
    c = O.det_uniform((B, Cn, D), 41).requires_grad_(True)
    u = O.det_uniform((B, D), 42).requires_grad_(True)
    ref = O.dot_product_click_predictor(c, u)
    g = O.det_uniform((B, Cn), 43)
    ref.backward(g)
    cd, ud = c.detach().to(DEV).requires_grad_(True), u.detach().to(DEV).requires_grad_(True)
    out = DotScoreFn.apply(cd, ud)
    out.backward(g.to(DEV))
    return {"fwd_rel": relerr(out, ref), "dc_rel": relerr(cd.grad, c.grad), "du_rel": relerr(ud.grad, u.grad)}


# ------------------------------------------------------------------------------------------------
def nrms_model_and_params(V, seed, heads=15, dropout=0.2, fused=False):
    import config as cfgmod
    from model.NRMS import NRMS
    # fused: False = fast mode, "accurate" = hi/lo pairs (V / probabilities / context) on the unfused kernels
    cfg = type("Cfg", (cfgmod.NRMSConfig,), dict(num_words=V, num_attention_heads=heads, dropout_probability=dropout,
                                                 precision="accurate" if fused == "accurate" else "fast"))
    sd = O.det_state_dict(O.nrms_shapes(V), seed)
    model = NRMS(cfg)
    model.load_state_dict(sd)
    return model.to(DEV), sd


def slots(t):
    return [{"title": t[:, j].contiguous()} for j in range(t.shape[1])]


def check_nrms_golden():
    """The committed golden case (minted from the live reference): CUDA path vs reference fp32 outputs and
    vs the oracle under the bf16 storage contract, forward and all parameter gradients."""
    from golden_util import case_params, load_case, oracle_forward, unique_params
    g = load_case("nrms")
    cand_t, clicked_t = torch.from_numpy(g["cand_title"]), torch.from_numpy(g["clicked_title"])
    p = case_params("nrms", g)
    logits_o, _ = oracle_forward("nrms", g, p, O.BF16)
    O.click_loss(logits_o).backward()
    model, _ = nrms_model_and_params(120, int(g["seed"]))
    model.eval()
    logits = model(slots(cand_t), slots(clicked_t))
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long, device=DEV))
    loss.backward()
    torch.cuda.synchronize()
    out = {"logits_vs_oracle_bf16": relerr(logits, logits_o), "logits_vs_reference_fp32": relerr(logits, torch.from_numpy(g["logits"])),
           "loss_abs_vs_reference": abs(loss.item() - float(g["loss"]))}
    grads = dict(model.named_parameters())
    worst, worst_key = 0.0, ""
    for k, prm in unique_params(p).items():
        if prm.grad.norm() < 1e-5:  # analytically ~0 gradients (W_K.bias) carry only rounding noise
            continue
        e = relerr(grads[k].grad, prm.grad)
        if e > worst:
            worst, worst_key = e, k
        out["grad:" + k] = e
    out["worst_grad_rel"] = worst
    out["worst_grad_key"] = worst_key
    out["emb_row0_grad_zero"] = bool((grads["news_encoder.word_embedding.weight"].grad[0] == 0).all())
    model.check_ids()
    return out


def check_nrms_random(B=8, Cn=5, H=50, T=20, V=500, seed=5, fused=False):
    """A MIND-shaped batch (K=4, history 50, left padded) vs the oracle under the bf16 contract."""
    cand_t, clicked_t, _ = O.synth_batch(B, Cn, H, T, V, seed * 100)
    model, sd = nrms_model_and_params(V, seed, fused=fused)
    model.eval()
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    logits_o = O.nrms_forward(cand_t, clicked_t, p, 15, O.WEIGHTS_BF16 if fused else O.BF16, c_news=O.BF16_FUSED if fused else O.BF16)
    O.click_loss(logits_o).backward()
    with torch.no_grad():
        logits_x = O.nrms_forward(cand_t, clicked_t, {k: v.detach() for k, v in p.items()}, 15, O.EXACT)
    logits = model(slots(cand_t), slots(clicked_t))
    torch.nn.functional.cross_entropy(logits, torch.zeros(B, dtype=torch.long, device=DEV)).backward()
    torch.cuda.synchronize()
    out = {"logits_vs_oracle_bf16": relerr(logits, logits_o), "logits_vs_exact_fp32": relerr(logits, logits_x),
           "oracle_bf16_vs_exact": relerr(logits_o, logits_x)}
    grads = dict(model.named_parameters())
    worst = 0.0
    for k, prm in p.items():
        if prm.grad.norm() < 1e-5:
            continue
        e = relerr(grads[k].grad, prm.grad)
        out["grad:" + k] = e
        worst = max(worst, e)
    out["worst_grad_rel"] = worst
    return out


def check_nrms_direct_grad_accumulation(B=8, Cn=5, H=50, T=20, V=500, seed=6):
    """Parameters with pre-allocated .grad storage (ddp.FlatGradients) are accumulated in place by the kernels; the
    result must equal the allocate-and-return path, also when two backward passes accumulate."""
    from newsrec_b200 import ddp
    cand_t, clicked_t, _ = O.synth_batch(B, Cn, H, T, V, seed * 100)
    label = torch.zeros(B, dtype=torch.long, device=DEV)
    model_a, _ = nrms_model_and_params(V, seed)
    model_b, _ = nrms_model_and_params(V, seed)
    model_a.eval()
    model_b.eval()
    flat = ddp.FlatGradients(model_b.parameters(), 1)
    flat.zero()
    for _ in range(2):  # two accumulating backward passes
        torch.nn.functional.cross_entropy(model_a(slots(cand_t), slots(clicked_t)), label).backward()
        torch.nn.functional.cross_entropy(model_b(slots(cand_t), slots(clicked_t)), label).backward()
    torch.cuda.synchronize()
    def worst_rel(ma, mb):
        # W_K.bias has an analytically zero gradient (softmax shift invariance): what both paths hold there is fp32
        # accumulation noise in atomic order.  Every difference is therefore measured against the tensor's own scale
        # floored at 1e-3 of the largest gradient in the model.
        floor = 1e-3 * max(float(p.grad.abs().max()) for p in ma.parameters())
        w = 0.0
        for (k, pa), (_, pb) in zip(ma.named_parameters(), mb.named_parameters()):
            scale = max(float(pa.grad.abs().max()), floor)
            w = max(w, float((pa.grad - pb.grad).abs().max()) / scale)
        return w

    worst = worst_rel(model_a, model_b)
    # a third backward with the persistent workspaces must start from cleared accumulators
    flat.zero()
    model_a.zero_grad(set_to_none=True)
    torch.nn.functional.cross_entropy(model_a(slots(cand_t), slots(clicked_t)), label).backward()
    torch.nn.functional.cross_entropy(model_b(slots(cand_t), slots(clicked_t)), label).backward()
    torch.cuda.synchronize()
    again = worst_rel(model_a, model_b)
    return {"direct_vs_returned_rel_maxabs": worst, "after_zero_rel_maxabs": again,
            "grads_are_flat_views": all(p.grad.data_ptr() >= flat.flat.data_ptr() for p in model_b.parameters())}


def check_nrms_prefetch_equals_direct(B=8, Cn=5, H=50, T=20, V=500, seed=7):
    """NRMS.prefetch (copy stream) + forward(PackedBatch) gives bit-identical logits to forward(lists)."""
    cand_t, clicked_t, _ = O.synth_batch(B, Cn, H, T, V, seed * 100)
    model, _ = nrms_model_and_params(V, seed)
    model.eval()
    with torch.no_grad():
        a = model(slots(cand_t), slots(clicked_t))
        pb = model.prefetch(slots(cand_t), slots(clicked_t))
        b = model(pb)
        pb2 = model.prefetch(slots(cand_t), slots(clicked_t))  # a second staged batch while the first is alive
        c = model(pb2)
    torch.cuda.synchronize()
    return {"maxabs": float((a - b).abs().max()), "maxabs_second": float((a - c).abs().max())}


def check_nrms_eval_api(V=300, seed=9):
    """get_news_vector / get_user_vector (non-contiguous input, evaluate.py:220-224) / get_prediction."""
    model, sd = nrms_model_and_params(V, seed)
    model.eval()
    p = {k: v for k, v in sd.items()}
    titles = O.synth_titles(40, 20, V, 3)
    with torch.no_grad():
        nv = model.get_news_vector({"title": titles, "id": ["N%d" % i for i in range(40)]})
        nv_o = O.nrms_news_encoder(titles, p, 15, O.BF16)
        B, H = 4, 10
        stacked = torch.stack([nv[i * 4:(i + 1) * 4] for i in range(H)], dim=0).transpose(0, 1)  # (B,H,d) non-contiguous
        uv = model.get_user_vector(stacked)
        uv_o = O.nrms_user_encoder(stacked.cpu(), p, 15, O.BF16)
        pred = model.get_prediction(nv[:7], uv[0])
        pred_o = (nv[:7].cpu() @ uv[0].cpu())
    return {"news_vec_rel": relerr(nv, nv_o), "user_vec_rel": relerr(uv, uv_o), "pred_rel": relerr(pred, pred_o),
            "user_input_noncontig": not stacked.is_contiguous(), "pred_tolist_len": len(pred.tolist())}


def check_nrms_train_mode(B=16, V=400, seed=4):
    """Training mode: dropout masks come from the in-kernel counter RNG, so parity is statistical:
    the mean logits over many seeds approach the eval logits, gradients are finite, row 0 grad is zero,
    and the backward regenerates exactly the forward masks (grad check against finite differences of the
    SAME masked function is implied by the eval-mode parity of the identical kernels with p=0)."""
    cand_t, clicked_t, _ = O.synth_batch(B, 5, 50, 20, V, seed * 100)
    model, _ = nrms_model_and_params(V, seed)
    model.eval()
    with torch.no_grad():
        ref = model(slots(cand_t), slots(clicked_t))
    model.train()
    acc = torch.zeros_like(ref)
    n = 24
    for _ in range(n):
        with torch.no_grad():
            acc += model(slots(cand_t), slots(clicked_t))
    mean = acc / n
    logits = model(slots(cand_t), slots(clicked_t))
    torch.nn.functional.cross_entropy(logits, torch.zeros(B, dtype=torch.long, device=DEV)).backward()
    g = model.news_encoder.word_embedding.weight.grad
    return {"mean_train_vs_eval_rel": relerr(mean, ref), "train_differs_from_eval": relerr(logits, ref) > 1e-3,
            "grads_finite": bool(torch.isfinite(g).all()), "emb_row0_grad_zero": bool((g[0] == 0).all())}


def check_nrms_train_masked(B=6, Cn=5, H=50, T=20, V=500, seed=8, p_drop=0.2, fused=False):
    """TRAIN mode -- the configuration bench.py times -- forward AND backward against the oracle under the SAME dropout
    masks: the kernels draw their masks from a counter hash of (seed, row, column); the test reads the seed the next
    forward will use (ops.peek_seeds) and hands it to the oracle, which rebuilds the masks with the NumPy restatement of
    that hash (oracle.dropout_mask) at both dropout sites (after the embedding, news_encoder.py:38, and after the
    self-attention, :43).  A backward that regenerated a different mask than its forward would fail every gradient."""
    from newsrec_b200 import ops
    cand_t, clicked_t, _ = O.synth_batch(B, Cn, H, T, V, seed * 100)
    model, sd = nrms_model_and_params(V, seed, dropout=p_drop, fused=fused)
    model.train()
    kseed = ops.peek_seeds(1)[0]  # the news encoder draws the only seed of a forward pass (the user encoder has no dropout)
    drop = dict(p=p_drop, seed=kseed, ld=ru8(300 + 1))
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    logits_o = O.nrms_forward(cand_t, clicked_t, p, 15, O.WEIGHTS_BF16 if fused else O.BF16, c_news=O.BF16_FUSED if fused else O.BF16,
                              drop=drop)
    O.click_loss(logits_o).backward()
    px = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    logits_x = O.nrms_forward(cand_t, clicked_t, px, 15, O.EXACT, drop=drop)  # exact arithmetic, same masks
    O.click_loss(logits_x).backward()
    with torch.no_grad():
        logits_eval = O.nrms_forward(cand_t, clicked_t, {k: v.detach() for k, v in px.items()}, 15, O.EXACT)
    logits = model(slots(cand_t), slots(clicked_t))
    torch.nn.functional.cross_entropy(logits, torch.zeros(B, dtype=torch.long, device=DEV)).backward()
    torch.cuda.synchronize()
    out = {"logits_vs_masked_oracle": relerr(logits, logits_o), "logits_vs_masked_exact_fp32": relerr(logits, logits_x),
           "masked_oracle_vs_masked_exact": relerr(logits_o, logits_x), "masks_matter": relerr(logits_x, logits_eval)}
    grads = dict(model.named_parameters())
    gscale = max(float(v.grad.norm()) for v in px.values())
    worst_ratio, worst_key = 0.0, ""
    for k, prm in px.items():
        if prm.grad.norm() < 1e-4 * gscale:
            continue
        e_kernel = relerr(grads[k].grad, prm.grad)
        e_contract = relerr(p[k].grad, prm.grad)
        out["grad:" + k] = [e_kernel, e_contract]
        ratio = e_kernel / max(e_contract, 2e-3)
        if ratio > worst_ratio:
            worst_ratio, worst_key = ratio, k
    out["worst_grad_ratio_kernel_over_contract"] = worst_ratio
    out["worst_grad_key"] = worst_key
    out["emb_row0_grad_zero"] = bool((grads["news_encoder.word_embedding.weight"].grad[0] == 0).all())
    return out


def check_nrms_full_size_properties(B=512):
    """BASELINE.json config[1] sizes (B=512, K=4, H=50, T=20, d=300, 15 heads, V=70976): size-independent
    properties -- (1) permuting the impressions permutes the logits, (2) the logits of a sub-batch equal the
    corresponding rows of the full batch, (3) sum of the embedding gradient over rows == a probe identity:
    d(sum logits)/d(emb) summed over the vocabulary equals the gradient w.r.t. a shared additive shift."""
    V = 70976
    cand_t, clicked_t, _ = O.synth_batch(B, 5, 50, 20, V, 4242)
    model, _ = nrms_model_and_params(V, 3)
    model.eval()
    with torch.no_grad():
        full = model(slots(cand_t), slots(clicked_t))
        perm = torch.from_numpy(__import__("numpy").random.RandomState(0).permutation(B))
        permd = model(slots(cand_t[perm]), slots(clicked_t[perm]))
        sub = model(slots(cand_t[:16]), slots(clicked_t[:16]))
    return {"perm_equivariance_maxabs": maxabs(permd, full[perm.to(DEV)]), "subbatch_maxabs": maxabs(sub, full[:16]),
            "finite": bool(torch.isfinite(full).all())}


# ------------------------------------------------------------------------------------------------
def check_backend_agreement(M=8800, N=900, K=300):
    """wgmma accumulators vs the SIMT triage backend on identical operands (fp32 output): locates
    pipeline bugs (which tile / row / column disagrees) that bf16 output rounding would hide."""
    lib = load_library()
    lda = ldw = ru8(K + 1)
    A = torch.zeros(M, lda)
    A[:, :K] = _rand_bf16((M, K), 1)
    W = torch.zeros(N, ldw)
    W[:, :K] = _rand_bf16((N, K), 2, 0.1)
    bias = O.det_uniform((N,), 3, -0.5, 0.5).to(DEV)
    ref = (A[:, :K].double() @ W[:, :K].double().t() + bias.cpu().double())
    Ad, Wd = A.to(torch.bfloat16).to(DEV), W.to(torch.bfloat16).to(DEV)
    ld_out = (N + 3) // 4 * 4
    outs = []
    for simt in (0, 1, 0):
        lib.nr_debug_set_simt_gemm(simt)
        out = torch.full((M, ld_out), float("nan"), dtype=torch.float32, device=DEV)
        check(lib.nr_linear(_p(Ad), M, lda, _p(Wd), N, ldw, K, 1, 0, 128, _p(bias), 0, _p(out), ld_out, 0, _stream()), "nr_linear")
        torch.cuda.synchronize()
        outs.append(out[:, :N].cpu().double())
    lib.nr_debug_set_simt_gemm(0)
    t, s, t2 = outs
    diff = (t - s).abs()
    bad = (diff > 1e-4).nonzero()
    res = {"tc_vs_ref_rel": relerr(t, ref), "simt_vs_ref_rel": relerr(s, ref), "tc_vs_simt_maxabs": float(diff.max()),
           "tc_rerun_maxabs": float((t - t2).abs().max()), "n_bad": int(bad.shape[0])}
    if bad.shape[0]:
        rows, cols = bad[:, 0], bad[:, 1]
        res["bad_rows_sample"] = rows[:12].tolist()
        res["bad_cols_sample"] = cols[:12].tolist()
        res["bad_tiles"] = sorted(set((rows // 128).tolist()))[:40]
        res["bad_col_range"] = [int(cols.min()), int(cols.max())]
        res["bad_row_in_tile_range"] = [int((rows % 128).min()), int((rows % 128).max())]
    return res


def _encoder_fwd_raw(ids, dense, sd, prefix, heads, V, p_drop=0.0, seed=0):
    """Direct nr_mhsa_encoder_fwd call returning every intermediate buffer (for differential triage)."""
    from newsrec_b200 import MhsaEncoderFwdArgs
    from newsrec_b200.ops import qkv_pitches, stack_qkv
    lib = load_library()
    d, q = 300, 200
    ldx, ld3 = ru8(d + 1), qkv_pitches(d)[1]
    g = lambda k: sd[f"{prefix}.{k}"].to(DEV)
    wqkv = stack_qkv(*[g(f"multihead_self_attention.W_{n}.weight") for n in "QKV"])
    ops = dict(wqkv=cast_pad(wqkv, ldx), bqkv=stack_qkv(*[g(f"multihead_self_attention.W_{n}.bias") for n in "QKV"]).contiguous(),
               wa=cast_pad(g("additive_attention.linear.weight"), ldx), ba=g("additive_attention.linear.bias").contiguous(),
               qv=g("additive_attention.attention_query_vector").contiguous())
    a = MhsaEncoderFwdArgs()
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    if ids is not None:
        n_seq, T = ids.shape
        table = cast_pad(sd["news_encoder.word_embedding.weight"].to(DEV), ldx)
        a.ids, a.table_bf16, a.V = _p(ids), _p(table), V
    else:
        n_seq, T, _ = dense.shape
        a.dense = _p(dense)
        a.dense_s_seq, a.dense_s_tok, a.dense_s_col = dense.stride()
    n_tok = n_seq * T
    bufs = dict(X=torch.zeros((n_tok, ldx), dtype=torch.bfloat16, device=DEV),
                QKV=torch.zeros((n_tok, ld3), dtype=torch.bfloat16, device=DEV),
                C=torch.zeros((n_tok, ldx), dtype=torch.bfloat16, device=DEV), w=torch.zeros((n_tok,), device=DEV),
                out=torch.zeros((n_seq, d), device=DEV))
    a.n_seq, a.T, a.d, a.heads, a.q, a.ldx, a.ld3 = n_seq, T, d, heads, q, ldx, ld3
    a.wqkv_bf16, a.bqkv, a.wa_bf16, a.ba, a.qv = _p(ops["wqkv"]), _p(ops["bqkv"]), _p(ops["wa"]), _p(ops["ba"]), _p(ops["qv"])
    a.p_drop, a.seed = float(p_drop), int(seed)
    a.X_bf16, a.QKV_bf16, a.C_bf16, a.w, a.out = _p(bufs["X"]), _p(bufs["QKV"]), _p(bufs["C"]), _p(bufs["w"]), _p(bufs["out"])
    a.bad_id_flag = _p(flag)
    check(lib.nr_mhsa_encoder_fwd(C.byref(a), _stream()), "nr_mhsa_encoder_fwd")
    torch.cuda.synchronize()
    out = {k: v.float().cpu() for k, v in bufs.items() if v is not None}
    out["bad_flag"] = int(flag.item())
    return out


def check_encoder_backend_diff(B=8, V=500, seed=5):
    """Every intermediate of the news and user encoders, wgmma vs SIMT triage backend, same inputs."""
    lib = load_library()
    cand_t, clicked_t, _ = O.synth_batch(B, 5, 50, 20, V, seed * 100)
    sd = O.det_state_dict(O.nrms_shapes(V), seed)
    ids = torch.cat((clicked_t.reshape(-1, 20), cand_t.reshape(-1, 20)), 0).to(DEV)
    res = {}
    runs = {}
    for name, simt in (("tc", 0), ("simt", 1)):
        lib.nr_debug_set_simt_gemm(simt)
        news = _encoder_fwd_raw(ids, None, sd, "news_encoder", 15, V)
        dense = news["out"][:B * 50].view(B, 50, 300).to(DEV).contiguous()
        user = _encoder_fwd_raw(None, dense, sd, "user_encoder", 15, V)
        runs[name] = (news, user)
    lib.nr_debug_set_simt_gemm(0)
    for lvl, i in (("news", 0), ("user", 1)):
        for k in ("X", "QKV", "C", "w", "out"):
            a, b = runs["tc"][i][k], runs["simt"][i][k]
            d = (a - b).abs()
            res[f"{lvl}.{k}.maxabs"] = float(d.max())
            res[f"{lvl}.{k}.n_diff"] = int((d > 0).sum())
            res[f"{lvl}.{k}.rel"] = relerr(a, b)
            if k in ("w", "out") and d.max() > 0:
                idx = d.reshape(d.shape[0], -1).max(dim=1).values.topk(min(5, d.shape[0]))
                res[f"{lvl}.{k}.worst_rows"] = idx.indices.tolist()
                res[f"{lvl}.{k}.worst_vals"] = [float(v) for v in idx.values]
    # and against the oracle
    p = {k: v for k, v in sd.items()}
    with torch.no_grad():
        nv_o = O.nrms_news_encoder(ids.cpu(), p, 15, O.BF16)
    res["news.out.tc_vs_oracle"] = relerr(runs["tc"][0]["out"], nv_o)
    res["news.out.simt_vs_oracle"] = relerr(runs["simt"][0]["out"], nv_o)
    dn = (runs["tc"][0]["out"] - nv_o).abs().max(dim=1).values
    res["news.out.tc_vs_oracle_worst_rows"] = dn.topk(5).indices.tolist()
    res["news.out.tc_vs_oracle_worst_vals"] = [float(v) for v in dn.topk(5).values]
    return res


# ------------------------------------------------------------------------------------------------
def build_model(case, V=120, ncat=15, nusers=40, H=6, dropout=0.2, fused=False):
    """Drop-in model + deterministic state_dict for a golden case name (see oracle/make_golden.py)."""
    import importlib
    import config as cfgmod
    from golden_util import case_shapes
    name = {"nrms": "NRMS", "naml": "NAML", "naml_f400": "NAML", "tanr": "TANR", "lstur_ini": "LSTUR", "lstur_con": "LSTUR"}[case]
    over = dict(num_words=V, num_categories=ncat, num_users=nusers, num_clicked_news_a_user=H, dropout_probability=dropout)
    if name == "NRMS":
        over["precision"] = "accurate" if fused == "accurate" else "fast"
    if name == "LSTUR":
        over["precision"] = "accurate" if fused else "fast"
    if case == "naml_f400":
        over["num_filters"] = 400
    if case.startswith("lstur"):
        over["long_short_term_method"] = case.split("_")[1]
    cfg = type("Cfg", (getattr(cfgmod, name + "Config"),), over)
    Model = getattr(importlib.import_module("model." + name), name)
    return Model(cfg).to(DEV), cfg


def golden_inputs(case, g):
    """Reference-style slot lists for a golden case."""
    t = lambda k: torch.from_numpy(g[k])
    keys = {"title": "title", "abstract": "abstract", "category": "category", "subcategory": "subcategory"}
    def mk(prefix):
        n = g[prefix + "_title"].shape[1]
        out = []
        for j in range(n):
            dct = {}
            for k in keys:
                if f"{prefix}_{k}" in g:
                    dct[k] = t(f"{prefix}_{k}")[:, j].contiguous()
            out.append(dct)
        return out
    return mk("cand"), mk("clicked")


def default_nrms_mode(name="NRMS"):
    """False ("fast") or "accurate": what the NRMS / LSTUR drop-in does when the config says nothing (config.py / NEWSREC_PRECISION)."""
    import config as cfgmod
    return "accurate" if getattr(getattr(cfgmod, name + "Config"), "precision", "fast") == "accurate" else False


def check_golden(case, fused=None):
    """A committed golden case (minted from the live reference): CUDA drop-in vs the reference's fp32 outputs, vs the
    oracle under the bf16 storage contract, and -- per gradient -- against the exact fp32 oracle next to the error the
    bf16 contract itself has (kernel_err <= ~1.5 x contract_err is the pass criterion)."""
    from golden_util import case_params, load_case, oracle_forward, unique_params
    if fused is None:  # the shipped default
        fused = default_nrms_mode() if case == "nrms" else (default_nrms_mode("LSTUR") if case.startswith("lstur") else False)
    g = load_case(case)
    p_b = case_params(case, g)
    logits_b, topic_b = oracle_forward(case, g, p_b, O.BF16, bool(fused))
    (O.click_loss(logits_b) + (0.1 * topic_b if topic_b is not None else 0.0)).backward()
    p_x = case_params(case, g)
    logits_x, topic_x = oracle_forward(case, g, p_x, O.EXACT)
    (O.click_loss(logits_x) + (0.1 * topic_x if topic_x is not None else 0.0)).backward()
    model, _ = build_model(case, fused=fused)
    sd = O.tie_shared(O.det_state_dict(__import__("golden_util").case_shapes(case), int(g["seed"])))
    model.load_state_dict(sd)
    model.eval()
    cand, clicked = golden_inputs(case, g)
    if case.startswith("lstur"):
        out = model(torch.from_numpy(g["user"]), torch.from_numpy(g["clicked_news_length"]).clone(), cand, clicked)
    else:
        out = model(cand, clicked)
    logits, topic = (out if isinstance(out, tuple) else (out, None))
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long, device=DEV))
    (loss + (0.1 * topic if topic is not None else 0.0)).backward()
    torch.cuda.synchronize()
    with torch.no_grad():  # the blueprint's tolerance definition (SURVEY.md 7.3-5): fp32 oracle on bf16-rounded weights / embeddings
        logits_w, _ = oracle_forward(case, g, case_params(case, g, requires_grad=False), O.WEIGHTS_BF16)
    res = {"logits_vs_oracle_bf16": relerr(logits, logits_b), "logits_vs_reference_fp32": relerr(logits, torch.from_numpy(g["logits"])),
           "logits_vs_weights_only_oracle": relerr(logits, logits_w),
           "oracle_bf16_vs_reference_fp32": relerr(logits_b, torch.from_numpy(g["logits"])),
           "loss_abs_vs_reference": abs(loss.item() - float(g["loss"]))}
    if topic is not None:
        res["topic_loss_rel_vs_reference"] = abs(topic.item() - float(g["topic_loss"])) / abs(float(g["topic_loss"]))
    grads = dict(model.named_parameters())
    worst_ratio, worst_key, worst_vs_b = 0.0, "", 0.0
    gscale = max(float(v.grad.norm()) for v in unique_params(p_x).values())
    for k, prm in unique_params(p_x).items():
        gk = grads[k].grad
        if gk is None:
            res["missing_grad:" + k] = True
            continue
        if prm.grad.norm() < 1e-4 * gscale:  # analytically ~0 gradients (W_K.bias): rounding noise only
            continue
        e_kernel = relerr(gk, prm.grad)
        e_contract = relerr(unique_params(p_b)[k].grad, prm.grad)
        e_vs_b = relerr(gk, unique_params(p_b)[k].grad)
        res["grad:" + k] = [e_kernel, e_contract, e_vs_b]
        ratio = e_kernel / max(e_contract, 2e-3)
        if ratio > worst_ratio:
            worst_ratio, worst_key = ratio, k
        worst_vs_b = max(worst_vs_b, e_vs_b)
    res["worst_grad_ratio_kernel_over_contract"] = worst_ratio
    res["worst_grad_key"] = worst_key
    res["worst_grad_vs_oracle_bf16"] = worst_vs_b
    w = grads.get("news_encoder.word_embedding.weight", grads.get("news_encoder.text_encoders.title.word_embedding.weight"))
    res["emb_row0_grad_zero"] = bool((w.grad[0] == 0).all())
    return res


def check_train_masked(case, p_drop=0.2, mask_p=0.5, fused=None):
    """TRAIN mode of a CNN family (NAML / TANR / LSTUR) on its golden inputs, forward AND backward, against the oracle under
    the SAME dropout masks (see check_nrms_train_masked): one seed per text-encoder call (NAML: title, then abstract), masks
    over the zero-padded gather layout and the compact conv-output layout.  LSTUR's user masking (F.dropout2d on the
    (1, B, dim) user embedding, LSTUR/__init__.py:74-77) is drawn by torch.rand on the device generator: the test seeds it,
    reads the draw the model is going to make, re-seeds and hands the same keep-multipliers to the oracle."""
    from golden_util import case_params, case_shapes, load_case, oracle_forward, unique_params
    from newsrec_b200 import ops
    g = load_case(case)
    if fused is None:  # the shipped default of the family (LSTUR: accurate = conv output / GRU input as hi/lo pairs)
        fused = default_nrms_mode("LSTUR") if case.startswith("lstur") else False
    model, cfg = build_model(case, dropout=p_drop, fused=fused)
    sd = O.tie_shared(O.det_state_dict(case_shapes(case), int(g["seed"])))
    model.load_state_dict(sd)
    model.train()
    cand, clicked = golden_inputs(case, g)
    B = g["cand_title"].shape[0]
    user_keep = None
    if case.startswith("lstur"):
        cfg.masking_probability = mask_p
        torch.cuda.manual_seed(1234)
        user_keep = ((torch.rand(B, 1, device=DEV) >= mask_p).float() / (1.0 - mask_p)).cpu()
        torch.cuda.manual_seed(1234)
    if case.startswith("naml"):
        s1, s2 = ops.peek_seeds(2)
        drop = dict(p=p_drop, seeds={"title": s1, "abstract": s2})
    else:
        drop = dict(p=p_drop, seed=ops.peek_seeds(1)[0])
    tw = lambda t: (0.1 * t if t is not None else 0.0)
    p_b = case_params(case, g)
    logits_b, topic_b = oracle_forward(case, g, p_b, O.BF16, bool(fused), drop=drop, user_keep=user_keep)
    (O.click_loss(logits_b) + tw(topic_b)).backward()
    p_x = case_params(case, g)
    logits_x, topic_x = oracle_forward(case, g, p_x, O.EXACT, drop=drop, user_keep=user_keep)
    (O.click_loss(logits_x) + tw(topic_x)).backward()
    with torch.no_grad():
        logits_eval, _ = oracle_forward(case, g, case_params(case, g, requires_grad=False), O.EXACT)
    if case.startswith("lstur"):
        out = model(torch.from_numpy(g["user"]), torch.from_numpy(g["clicked_news_length"]).clone(), cand, clicked)
    else:
        out = model(cand, clicked)
    logits, topic = (out if isinstance(out, tuple) else (out, None))
    loss = torch.nn.functional.cross_entropy(logits, torch.zeros(logits.shape[0], dtype=torch.long, device=DEV))
    (loss + tw(topic)).backward()
    torch.cuda.synchronize()
    res = {"logits_vs_masked_oracle": relerr(logits, logits_b), "logits_vs_masked_exact_fp32": relerr(logits, logits_x),
           "masked_oracle_vs_masked_exact": relerr(logits_b, logits_x), "masks_matter": relerr(logits_x, logits_eval)}
    if topic is not None:
        res["topic_loss_rel_vs_masked_exact"] = abs(topic.item() - float(topic_x)) / abs(float(topic_x))
    grads = dict(model.named_parameters())
    gscale = max(float(v.grad.norm()) for v in unique_params(p_x).values())
    worst_ratio, worst_key = 0.0, ""
    for k, prm in unique_params(p_x).items():
        if grads[k].grad is None:
            res["missing_grad:" + k] = True
            continue
        if prm.grad.norm() < 1e-4 * gscale:
            continue
        e_kernel = relerr(grads[k].grad, prm.grad)
        e_contract = relerr(unique_params(p_b)[k].grad, prm.grad)
        res["grad:" + k] = [e_kernel, e_contract]
        ratio = e_kernel / max(e_contract, 2e-3)
        if ratio > worst_ratio:
            worst_ratio, worst_key = ratio, k
    res["worst_grad_ratio_kernel_over_contract"] = worst_ratio
    res["worst_grad_key"] = worst_key
    return res


def check_predict_impressions(n_news=500, D=300, n_imp=200, seed=3):
    """Batched evaluation scoring (ops.predict_impressions) against the evaluator's per-impression get_prediction loop."""
    from newsrec_b200.ops import predict_impressions
    model, _ = nrms_model_and_params(50, 1)
    news = O.det_uniform((n_news, D), seed).to(DEV)
    users = O.det_uniform((n_imp, D), seed + 1).to(DEV)
    counts = O.det_randint((n_imp,), seed + 2, 1, 40)
    offs = torch.zeros(n_imp + 1, dtype=torch.int64)
    offs[1:] = counts.cumsum(0)
    cand = O.det_randint((int(offs[-1]),), seed + 3, 0, n_news)
    got = predict_impressions(news, cand, offs, users)
    ref = []
    for s in range(n_imp):  # evaluate.py:245-260
        idx = cand[offs[s]:offs[s + 1]].to(DEV)
        ref.append(model.get_prediction(news[idx], users[s]))
    ref = torch.cat(ref)
    return {"rel": relerr(got, ref), "n": int(got.numel())}


def check_pack_slots(B=37, H=50, Cn=5, tail=(20,), where="pinned"):
    """SlotPacker.pack through the one-launch batch feed (nr_pack_slots) against the stack / transpose / cat it replaces."""
    from newsrec_b200.pack import SlotPacker
    gen = torch.Generator().manual_seed(B * 131 + H)
    mk = lambda: torch.randint(0, 70000, (B,) + tuple(tail), generator=gen, dtype=torch.int64)
    place = {"pinned": lambda t: t.pin_memory(), "device": lambda t: t.to(DEV), "pageable": lambda t: t}[where]
    clicked = [{"f": place(mk())} for _ in range(H)]
    cand = [{"f": place(mk())} for _ in range(Cn)]
    pk = SlotPacker()
    direct = pk._pack_direct([x["f"] for x in clicked], [x["f"] for x in cand], DEV)
    ids, Bo = pk.pack(clicked, cand, "f", DEV)
    torch.cuda.synchronize()
    ref = torch.cat((torch.stack([x["f"].cpu() for x in clicked], 1).reshape(B * H, *tail),
                     torch.stack([x["f"].cpu() for x in cand], 1).reshape(B * Cn, *tail)), 0)
    return {"equal": bool(torch.equal(ids.cpu(), ref)), "B": Bo, "direct": direct is not None,
            "direct_equal": direct is None or bool(torch.equal(direct[0].cpu(), ref))}


# ------------------------------------------------------------------------------------------------
# The CNN text encoder (nr_cnn_encoder_fwd / _bwd) and its companion operators, called through the C ABI with every output
# pre-filled (NaN where the ABI writes "=", a known pattern where it accumulates "+=") and followed by a guard of sentinel
# values, then compared ROW BY ROW with fp64 evaluations on the device built from the kernels' own stored inputs.  A norm
# over a whole tensor of 600k rows cannot see one wrong row; a per-row or per-segment measure can.
# ------------------------------------------------------------------------------------------------
_GUARD = 2048
_M32 = 0xFFFFFFFF
_INT_VIEW = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int32: torch.int32, torch.uint8: torch.uint8,
             torch.int64: torch.int64}


class _Guarded:
    """Flat device buffer of n elements pre-filled with `fill` (a scalar, or a tensor of n elements kept as `prefill` for the
    "+=" outputs), followed by _GUARD sentinel elements.  Only the guard is copied: the bodies can be hundreds of MB."""

    def __init__(self, n, dtype, fill, sentinel=-1234.5):
        self.n = int(n)
        self.all = torch.empty(self.n + _GUARD, dtype=dtype, device=DEV)
        self.prefill = None
        if isinstance(fill, torch.Tensor):
            self.prefill = fill.reshape(-1).to(dtype)
            self.all[:self.n] = self.prefill
        else:
            self.all[:self.n].fill_(fill)
        self.all[self.n:].fill_(sentinel)
        self.guard = self.all[self.n:].clone()

    @property
    def body(self):
        return self.all[:self.n]

    def guard_ok(self):
        iv = _INT_VIEW[self.all.dtype]
        return bool(torch.equal(self.all[self.n:].view(iv), self.guard.view(iv)))

    def unchanged(self, mask):
        """Elements selected by the boolean mask over the body still hold their pre-fill, bit for bit."""
        iv = _INT_VIEW[self.all.dtype]
        return bool(torch.equal(self.body.view(iv)[mask.reshape(-1)], self.prefill.view(iv)[mask.reshape(-1)]))


def _bits_equal(a, b):
    iv = _INT_VIEW[a.dtype]
    return bool(torch.equal(a.contiguous().view(iv), b.contiguous().view(iv)))


def _mul32(a, b):
    """(a * b) mod 2^32 for an int64 tensor a < 2^32 and a constant b < 2^32, without int64 overflow."""
    return (a * (b & 0xFFFF) + (((a * (b >> 16)) & 0xFFFF) << 16)) & _M32


def dropout_mask_dev(seed, p, rows, n_cols, ld):
    """Device restatement of oracle.dropout_mask (the kernels' counter hash): fp32 multipliers of the given rows (int64
    device tensor) and columns [0, n_cols) of a matrix with pitch ld."""
    import numpy as np
    if p <= 0.0:
        return torch.ones(rows.numel(), n_cols, device=rows.device)
    thresh = int(np.float32(p) * np.float32(65536.0) + np.float32(0.5))
    scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
    flat = rows.reshape(-1, 1).long() * ld + torch.arange(n_cols, device=rows.device).view(1, -1)
    group = flat >> 2
    s_lo, s_hi = seed & _M32, (seed >> 32) & _M32
    x = ((group & _M32) ^ s_lo) + _mul32(group >> 32, 0x85EBCA6B) + ((s_hi * 0x165667B1) & _M32)
    x = _mul32(x & _M32, 0x9E3779B1)
    x ^= x >> 15
    x = _mul32(x, 0x85EBCA77)
    x ^= x >> 13
    y = (_mul32(x, 0xC2B2AE3D) + s_hi) & _M32
    y ^= y >> 16
    y = _mul32(y, 0x27D4EB2F)
    y ^= y >> 15
    lane = flat & 3
    half = torch.where(lane < 2, x, y)
    bits = torch.where((lane & 1) == 0, half & 0xFFFF, half >> 16)
    return torch.where(bits >= thresh, torch.tensor(scale, device=rows.device), torch.tensor(0.0, device=rows.device))


def _bf16_ulp(v):
    """One bf16 ulp at |v| (fp64 tensor); 0 where v == 0."""
    _, e = torch.frexp(v.abs())
    return torch.where(v == 0, torch.zeros_like(v), torch.ldexp(torch.ones_like(v), e - 8))


def _safe_div(num, den):
    return torch.where(num == 0, torch.zeros_like(num), num / den.clamp_min(1e-300))


def _worst(t):
    """Largest element of a metric tensor, +inf if any element is NaN (an output the kernels never wrote keeps its NaN
    pre-fill: it must fail every bound, never drop out of a max)."""
    return float(torch.nan_to_num(t, nan=float("inf")).max()) if t.numel() else 0.0


def _row_ratio(kern, exact, contract, floor=2e-3):
    """The project's gradient rule applied to each row of 2-D tensors: (|kernel - exact| / |exact|) divided by
    max(|contract - exact| / |exact|, floor), which must stay <= 1.5.  Returns (worst ratio, relative kernel and contract
    error of that row); a NaN anywhere makes the ratio +inf."""
    nx = exact.norm(dim=1)
    ek = _safe_div((kern - exact).norm(dim=1), nx)
    ec = _safe_div((contract - exact).norm(dim=1), nx)
    r = torch.nan_to_num(ek / ec.clamp_min(floor), nan=float("inf"))
    i = int(r.argmax())
    return float(r[i]), float(ek[i]), float(ec[i])


def _cnn_ids(n_seq, T, V, seed, bad_ids):
    """MIND-like right-padded titles with ids 0 and V-1 present; bad_ids plants two out-of-range ids (V + 5 and -1)."""
    ids = O.synth_titles(n_seq, T, V, seed, min_len=1).reshape(-1)
    n = ids.numel()
    if n == 0:  # a one-element buffer, so that the ABI sees a valid pointer
        return torch.zeros(1, dtype=torch.int64, device=DEV)
    ids[0] = V - 1
    if n > 2:
        ids[n - 1] = V - 1
        ids[n // 2] = 0
    if bad_ids and n >= 8:
        ids[n // 3] = V + 5
        ids[(2 * n) // 3 + 1] = -1
    return ids.view(n_seq, T).to(DEV)


def check_cnn_encoder(n_seq=37, T=20, d=300, F=400, q=200, V=500, p_drop=0.2, accurate=False, seed=1, bad_ids=True, grad_floor=2e-3):
    """nr_cnn_encoder_fwd / _bwd stage by stage against fp64 references built from the kernels' own stored Xp, Y, w:
    exact gather, per-element conv output within one bf16 ulp plus an fp32-accumulation allowance, per-segment pooling,
    per-row gradients under the project's gradient rule (kernel error <= 1.5 x the bf16 contract's, floor grad_floor), every
    "=" output finite (nothing left at its NaN pre-fill), the pre-fill of every "+=" output outside the rows / columns the
    kernels own, and the guard behind every buffer."""
    from newsrec_b200 import CnnEncoderBwdArgs, CnnEncoderFwdArgs
    lib = load_library()
    T_p = T + 2
    ldx, ldf, ldq = ru8(d + 1), ru8(F + 1), ru16(q)
    n_tok, Mp = n_seq * T, n_seq * T_p
    # ---- operands, built the way CnnPoolEncoderFn.build does (tap-major conv weight rows, transposed taps for dX)
    a_w = 0.5 * math.sqrt(3.0 / d)  # pre-activation std ~0.5: with a small centred bias about half of it is positive
    Wc = _rand_bf16((F, 3, d), seed + 1, a_w).to(DEV)
    bc = O.det_uniform((F,), seed + 2, -0.05, 0.05).to(DEV)
    Wa = _rand_bf16((q, F), seed + 3, math.sqrt(3.0 / F)).to(DEV)
    ba = O.det_uniform((q,), seed + 4, -0.1, 0.1).to(DEV)
    qv = O.det_uniform((q,), seed + 5, -1.0, 1.0).to(DEV)
    table_f = _rand_bf16((V, d), seed + 6).to(DEV)
    wconv = cast_pad(Wc.permute(1, 0, 2).reshape(3 * F, d), ldx)
    wconvT = cast_pad(torch.cat([Wc[:, 2 - s, :].t() for s in range(3)], 0), ldf)
    wa, waT, table = cast_pad(Wa, ldf), cast_pad(Wa, ldq, transpose=True), cast_pad(table_f, ldx)
    ids = _cnn_ids(n_seq, T, V, seed + 7, bad_ids)
    kseed = (0x9E3779B97F4A7C15 * (seed + 11)) & 0xFFFFFFFFFFFFFFFF

    def forward():
        bufs = dict(Xp=_Guarded(Mp * ldx, torch.bfloat16, float("nan")), Y=_Guarded(n_tok * ldf, torch.bfloat16, float("nan")),
                    w=_Guarded(n_tok, torch.float32, float("nan")), out=_Guarded(n_seq * F, torch.float32, float("nan")),
                    flag=_Guarded(1, torch.int32, 0, sentinel=-7))
        if accurate:
            bufs["Ylo"] = _Guarded(n_tok * ldf, torch.bfloat16, float("nan"))
        a = CnnEncoderFwdArgs()
        a.n_seq, a.T, a.d, a.F, a.q, a.ldx, a.ldf = n_seq, T, d, F, q, ldx, ldf
        a.ids, a.table_bf16, a.V = _p(ids), _p(table), V
        a.wconv_bf16, a.bconv, a.wa_bf16, a.ba, a.qv = _p(wconv), _p(bc), _p(wa), _p(ba), _p(qv)
        a.p_drop, a.seed = float(p_drop), kseed
        a.Xp_bf16, a.Y_bf16, a.w, a.out = _p(bufs["Xp"].all), _p(bufs["Y"].all), _p(bufs["w"].all), _p(bufs["out"].all)
        a.bad_id_flag = _p(bufs["flag"].all)
        if accurate:
            a.Y_lo_bf16 = _p(bufs["Ylo"].all)
        n0 = int(lib.nr_launch_count())
        check(lib.nr_cnn_encoder_fwd(C.byref(a), _stream()), "nr_cnn_encoder_fwd")
        return bufs, int(lib.nr_launch_count()) - n0

    fb, fwd_launches = forward()
    dout = O.det_uniform((max(n_seq, 1), F), seed + 8).to(DEV)
    pat = lambda n, s: O.det_uniform((n,), s, 0.5, 1.0).to(DEV) * 2.0 ** -16  # small non-zero "+=" pre-fill
    bb = dict(dWc=_Guarded(3 * F * ldx, torch.float32, pat(3 * F * ldx, seed + 20)),
              dWa=_Guarded(q * ldf, torch.float32, pat(q * ldf, seed + 21)),
              dqv=_Guarded(q, torch.float32, pat(q, seed + 22)), demb=_Guarded(V * d, torch.float32, pat(V * d, seed + 23)))
    ws_bytes = int(lib.nr_cnn_encoder_bwd_workspace(n_seq, T, F, q))
    ws = _Guarded(ws_bytes, torch.uint8, 0xFF, sentinel=0xA5)  # 0xFFFF.. = NaN in bf16 and fp32: unwritten rows poison results
    b = CnnEncoderBwdArgs()
    b.n_seq, b.T, b.d, b.F, b.q, b.ldx, b.ldf, b.ldq = n_seq, T, d, F, q, ldx, ldf, ldq
    b.ids, b.V = _p(ids), V
    b.wconvT_bf16, b.wa_bf16, b.waT_bf16, b.ba, b.qv = _p(wconvT), _p(wa), _p(waT), _p(ba), _p(qv)
    b.p_drop, b.seed = float(p_drop), kseed
    b.Xp_bf16, b.Y_bf16, b.w, b.dout = _p(fb["Xp"].all), _p(fb["Y"].all), _p(fb["w"].all), _p(dout)
    b.dWconv_ext, b.dWa_ext, b.dqv, b.demb = _p(bb["dWc"].all), _p(bb["dWa"].all), _p(bb["dqv"].all), _p(bb["demb"].all)
    b.workspace, b.workspace_bytes = _p(ws.all), ws_bytes
    n0 = int(lib.nr_launch_count())
    check(lib.nr_cnn_encoder_bwd(C.byref(b), _stream()), "nr_cnn_encoder_bwd")
    bwd_launches = int(lib.nr_launch_count()) - n0
    torch.cuda.synchronize()
    res = {"fwd_launches": fwd_launches, "bwd_launches": bwd_launches,
           "guards_intact": all(g.guard_ok() for g in list(fb.values()) + list(bb.values()) + [ws])}
    del ws
    if n_seq == 0:
        return res
    res["bad_id_flag"] = int(fb["flag"].body.item())
    ids_flat = ids.reshape(-1)
    bad = (ids_flat < 0) | (ids_flat >= V)
    res["bad_ids_planted"] = int(bad.sum())
    # every "=" output is written where the ABI says it is (Y_lo: columns [0, F))
    res["fwd_outputs_finite"] = all(bool(torch.isfinite(fb[k].body.float()).all()) for k in ("Xp", "Y", "w", "out")) and \
        (not accurate or bool(torch.isfinite(fb["Ylo"].body.view(n_tok, ldf)[:, :F].float()).all()))

    # ---- fp64 references, a chunk of about 8k padded rows at a time (a few hundred MB of fp64 temporaries at any n_seq)
    Xp3 = fb["Xp"].body.view(n_seq, T_p, ldx)
    Y2 = fb["Y"].body.view(n_tok, ldf)
    Ylo2 = fb["Ylo"].body.view(n_tok, ldf) if accurate else None
    w1, out2 = fb["w"].body, fb["out"].body.view(n_seq, F)
    W64 = Wc.double().permute(1, 0, 2).contiguous()  # (3, F, d)
    Wa64, ba64, qv64, bc64 = Wa.double(), ba.double(), qv.double(), bc.double()
    scale = float(1.0 / (1.0 - torch.tensor(p_drop, dtype=torch.float32))) if p_drop > 0 else 1.0  # the kernels' fp32 1/(1-p)
    ids_safe = torch.where(bad, torch.zeros_like(ids_flat), ids_flat)
    scat = (ids_flat >= 1) & (ids_flat < V)
    acc = {k: 0.0 for k in ("y_ratio", "ylo_ratio", "w_err", "w_sum_err", "out_ratio", "t1_w_err", "t1_out_ratio")}
    worst = lambda k, t: acc.__setitem__(k, max(acc[k], _worst(t)))
    cnt = dict(xp_mismatch_rows=0, y_dropped_nonzero=0, y_pos=0, y_n=0)
    ones_ok = True
    grads = {v: dict(dWc=torch.zeros(3, F, d + 1, dtype=torch.float64, device=DEV),
                     dWa=torch.zeros(q, F + 1, dtype=torch.float64, device=DEV),
                     dqv=torch.zeros(q, dtype=torch.float64, device=DEV),
                     demb=torch.zeros(V, d, dtype=torch.float64, device=DEV)) for v in ("exact", "contract")}
    cs = max(1, 8192 // T_p)
    for s0 in range(0, n_seq, cs):
        s1 = min(n_seq, s0 + cs)
        ns = s1 - s0
        r0, r1 = s0 * T, s1 * T
        seg = torch.arange(s0, s1, device=DEV)
        tok_rows = (seg.view(-1, 1) * T_p + 1 + torch.arange(T, device=DEV).view(1, -1)).reshape(-1)  # padded rows of tokens
        # Xp: masked gather of the bf16 table rows, ones column at d, zeros behind it, zero pad rows -- bit exact
        mx = dropout_mask_dev(kseed, p_drop, tok_rows, d, ldx)
        exp_x = torch.zeros(ns, T_p, ldx, dtype=torch.float32, device=DEV)
        exp_x[:, 1:T + 1, :d] = ((table_f[ids_safe[r0:r1]] * mx).to(torch.bfloat16).float()).view(ns, T, d)
        exp_x[:, 1:T + 1, d] = 1.0
        got_x = Xp3[s0:s1]
        cnt["xp_mismatch_rows"] += int((got_x.view(torch.int16) != exp_x.to(torch.bfloat16).view(torch.int16)).any(dim=2).sum())
        X64 = got_x.double()
        # conv: pre[s, t] = sum_k Xp[s, t + k] . W_k + b, and the sum of |products| for the accumulation allowance
        pre = torch.zeros(ns * T, F, dtype=torch.float64, device=DEV) + bc64
        absum = torch.zeros(ns * T, F, dtype=torch.float64, device=DEV) + bc64.abs()
        for k in range(3):
            xk = X64[:, k:k + T, :d].reshape(-1, d)
            pre += xk @ W64[k].t()
            absum += xk.abs() @ W64[k].abs().t()
        my = dropout_mask_dev(kseed ^ 0x5BD1E995, p_drop, torch.arange(r0, r1, device=DEV), F, ldf).double()
        ref_y = pre.clamp_min(0) * my
        y = Y2[r0:r1]
        y64 = y[:, :F].double()
        bound = _bf16_ulp(torch.maximum(ref_y.abs(), y64.abs())) + 1e-6 * absum * my.clamp_min(1.0)
        worst("y_ratio", _safe_div((y64 - ref_y).abs(), bound))
        cnt["y_dropped_nonzero"] += int(((my == 0) & (y64 != 0)).sum())
        cnt["y_pos"] += int((pre > 0).sum())
        cnt["y_n"] += pre.numel()
        ones_ok &= bool((y[:, F] == 1).all()) and bool((y[:, F + 1:] == 0).all())
        yy = y64
        if accurate:
            yy = y64 + Ylo2[r0:r1, :F].double()
            rb = 2.0 ** -16 * ref_y.norm(dim=1) + 1e-6 * (absum * my).norm(dim=1)
            worst("ylo_ratio", _safe_div((yy - ref_y).norm(dim=1), rb))
        # pooling from the kernel's own Y: fp64 tanh scores, softmax per segment, weighted sum of Y (+ Y_lo)
        score = torch.tanh(y64 @ Wa64.t() + ba64) @ qv64
        w_ref = torch.softmax(score.view(ns, T), dim=1)
        wk = w1[r0:r1].double().view(ns, T)
        worst("w_err", (wk - w_ref).abs())
        worst("w_sum_err", (wk.sum(1) - 1).abs())
        yy3 = yy.view(ns, T, F)
        o_ref = (wk.unsqueeze(2) * yy3).sum(1)
        o_abs = (wk.unsqueeze(2) * yy3.abs()).sum(1)
        o_got = out2[s0:s1].double()
        worst("out_ratio", _safe_div((o_got - o_ref).norm(dim=1), o_abs.norm(dim=1)))
        if T == 1:
            worst("t1_w_err", (wk - 1).abs())
            worst("t1_out_ratio", _safe_div((o_got - yy).abs(), yy.abs() * 2.0 ** -23))
        # ---- backward, exact and under the bf16 contract (dPre and dY stored in bf16)
        do = dout[s0:s1].double()
        dw = (y64.view(ns, T, F) * do.unsqueeze(1)).sum(2)
        dscore = wk * (dw - (wk * dw).sum(1, keepdim=True))
        th = torch.tanh(y64 @ Wa64.t() + ba64)
        dpre = dscore.reshape(-1, 1) * qv64 * (1 - th * th)
        dqv_c = (dscore.reshape(-1, 1) * th).sum(0)
        relu_keep = (y64 > 0).double() * scale
        xs = X64[:, :, :d + 1].reshape(-1, d + 1)
        y1 = torch.cat([y64, torch.ones(ns * T, 1, dtype=torch.float64, device=DEV)], 1)
        sc_ids = ids_flat[r0:r1][scat[r0:r1]]
        for v in ("exact", "contract"):
            dp = dpre if v == "exact" else bf16r(dpre.float()).double()
            dyc = (dp @ Wa64 + wk.reshape(-1, 1) * do.repeat_interleave(T, 0)) * relu_keep
            if v == "contract":
                dyc = bf16r(dyc.float()).double()
            g = grads[v]
            g["dqv"] += dqv_c
            g["dWa"] += dp.t() @ y1
            dyp = torch.zeros(ns, T_p, F, dtype=torch.float64, device=DEV)
            dyp[:, 1:T + 1] = dyc.view(ns, T, F)
            dyp = dyp.view(-1, F)
            n_p = dyp.shape[0]
            for k in range(3):  # dW_k += dY^T . X[rows + k - 1]; dX[r] += dY[r - k + 1] . W_k
                sh = k - 1
                xsh = torch.zeros_like(xs)
                dys = torch.zeros_like(dyp)
                if sh >= 0:
                    xsh[:n_p - sh] = xs[sh:]
                    dys[sh:] = dyp[:n_p - sh]
                else:
                    xsh[-sh:] = xs[:n_p + sh]
                    dys[:n_p + sh] = dyp[-sh:]
                g["dWc"][k] += dyp.t() @ xsh
                dX = dys @ W64[k] if k == 0 else dX + dys @ W64[k]
            dXt = dX.view(ns, T_p, d)[:, 1:T + 1].reshape(-1, d) * mx.double()
            g["demb"].index_add_(0, sc_ids, dXt[scat[r0:r1]])
    res.update({k: v for k, v in acc.items()})
    res.update(cnt)
    res["y_pos_fraction"] = cnt["y_pos"] / max(1, cnt["y_n"])
    res["y_ones_col_and_pad_exact"] = ones_ok
    # ---- gradients: per row, kernel vs exact against contract vs exact
    ex, co = grads["exact"], grads["contract"]
    dWc_k = (bb["dWc"].body.double() - bb["dWc"].prefill.double()).view(3, F, ldx)[:, :, :d + 1]
    dWa_k = (bb["dWa"].body.double() - bb["dWa"].prefill.double()).view(q, ldf)[:, :F + 1]
    dqv_k = bb["dqv"].body.double() - bb["dqv"].prefill.double()
    demb_k = (bb["demb"].body.double() - bb["demb"].prefill.double()).view(V, d)
    res["dWconv_row_ratio"], res["dWconv_ek"], res["dWconv_ec"] = _row_ratio(*[t.reshape(3 * F, -1) for t in (dWc_k, ex["dWc"], co["dWc"])],
                                                                            floor=grad_floor)
    res["dWa_row_ratio"], res["dWa_ek"], res["dWa_ec"] = _row_ratio(dWa_k, ex["dWa"], co["dWa"], floor=grad_floor)
    res["dqv_ratio"], res["dqv_ek"], res["dqv_ec"] = _row_ratio(*[t.view(1, -1) for t in (dqv_k, ex["dqv"], co["dqv"])], floor=grad_floor)
    touched = torch.zeros(V, dtype=torch.bool, device=DEV)
    touched[ids_flat[scat]] = True
    res["demb_rows_touched"] = int(touched.sum())
    res["demb_row_ratio"], res["demb_ek"], res["demb_ec"] = _row_ratio(demb_k[touched], ex["demb"][touched], co["demb"][touched],
                                                                       floor=grad_floor)
    # what a whole-tensor norm would have said about the same outputs (for comparison only)
    res["dWconv_tensor_relerr"] = relerr(dWc_k, ex["dWc"])
    res["demb_tensor_relerr"] = relerr(demb_k, ex["demb"])
    # ---- the pre-fill outside what the kernels own: pitch columns, untouched embedding rows (row 0, unused ids)
    colmask = torch.zeros(3, F, ldx, dtype=torch.bool, device=DEV)
    colmask[:, :, d + 1:] = True
    res["dWconv_pitch_cols_untouched"] = bb["dWc"].unchanged(colmask)
    colmask = torch.zeros(q, ldf, dtype=torch.bool, device=DEV)
    colmask[:, F + 1:] = True
    res["dWa_pitch_cols_untouched"] = bb["dWa"].unchanged(colmask)
    res["demb_untouched_rows_exact"] = bb["demb"].unchanged((~touched).view(V, 1).expand(V, d))
    if T == 1:  # dscore = w (dw - w dw) vanishes: dqv and dWa_ext keep their pre-fill
        res["t1_dqv_rel"] = _worst(dqv_k.abs() / bb["dqv"].prefill.double())
        res["t1_dWa_rel"] = _worst(dWa_k.abs() / bb["dWa"].prefill.double().view(q, ldf)[:, :F + 1])
    del grads, ex, co, dWc_k, dWa_k, dqv_k, demb_k, bb

    # ---- determinism: a second forward is bit-identical (run last, when the references are freed)
    fb2, _ = forward()
    torch.cuda.synchronize()
    res["fwd_deterministic"] = all(_bits_equal(fb[k].body, fb2[k].body) for k in fb if k != "flag")
    return res


# ------------------------------------------------------------------------------------------------
def _abs_allow_rows(got, ref, absref):
    """max over rows of |got - ref| / |absref| (row norms): fp32 accumulation error against the sum of |products|."""
    return _worst(_safe_div((got - ref).norm(dim=1), absref.norm(dim=1)))


# ------------------------------------------------------------------------------------------------
# Element bounds of the wgmma GEMMs and of the additive-attention forward (tests/test_gpu_gemm_elements.py,
# tests/test_gpu_additive_fwd.py): each output element against an fp64 evaluation of the operands the kernel read.
# ------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24  # unit roundoff of fp32
TANH_ERR = 2e-7   # absolute error of fast_tanh (nr_common.cuh): ex2.approx, one division, one subtraction


def gemm_elem_ratio(got, pre, absum, n_acc, out_bf16, relu=False):
    """The GEMM element judge.  An element may miss its fp64 value ref (pre, after the ReLU) by e = 4u (n_acc + 2) S, with
    S = sum of |products| + |bias| (+ |pre-fill| for a "+=" output) and n_acc the fp32 accumulations it went through (a
    worst-case gamma_n, doubled because the tensor core's internal rounding is not documented); a bf16 output by e + half a
    bf16 ulp of |ref| + e.  Returns the worst (|got - ref| - rounding allowance) / e, clamped at 0 -- the share of the
    accumulation allowance used, <= 1 exactly when every element is inside its bound (+inf for a NaN) -- and whether every
    element whose pre-activation lies below -e came out exactly 0 under a ReLU (True without one)."""
    ref = pre.clamp_min(0) if relu else pre
    e = 4 * U32 * (n_acc + 2) * absum
    err = (got.double() - ref).abs()
    if out_bf16:
        err = (err - 0.5 * _bf16_ulp(ref.abs() + e)).clamp_min(0)
    ratio = _worst(_safe_div(err, e))
    zero_exact = bool((got[pre + e < 0] == 0).all()) if relu else True
    return ratio, zero_exact


def additive_fwd_judge(X, Wa, ba, qv, seg, out, w=None, X_lo=None):
    """The pooling forward out_s = sum_r w_r X_r, w = softmax over the segment of score_r = sum_c qv_c tanh(X_r . Wa_c + ba_c),
    judged element by element.  X [rows][D] (the plane the scores read), X_lo (or None) the low plane, Wa [q][D], ba and qv [q]:
    the kernel's own operands as fp64 device tensors; out [n_seg][D] and w [rows] (or None) are the kernel's results.
    The bound is carried stage by stage:
      pre   e_rc = the GEMM bound (fp32 accumulation of ceil(D/16) k-steps, then the bias)
      tanh  e_rc + TANH_ERR
      score ds_r = sum_c |qv_c| (e_rc + TANH_ERR) + q u sum_c |qv_c t_rc|
      w     |dw_r| <= w_r (2 max_seg ds + x_r + sum_t w_t x_t + (seg + 2) u) + 2^-126, with x_r = (2 |s_r - max| + 4) u the
            error of __expf on the shifted score (the subtraction, the scaling by log2(e), ex2.approx), seg u the fp32 sum
            and 2u the division; ex2.approx flushes results below 2^-126 to zero
      out   |dout_d| <= sum_r |dw_r| |X_rd| + (n + 1) u sum_r w_r |X_rd|, n = seg fma steps (2 seg with the low plane, whose
            rows enter |X| too)
    Returns {"out_ratio", "w_ratio"}: the worst |kernel - ref| / bound of out, and of w the worst (|kernel - ref| - 2^-126) /
    (the relative part of its bound), clamped at 0 -- both <= 1 exactly when every element is inside its bound (+inf for a
    NaN); a weight that underflows to 0 in the kernel uses the flush allowance, not the relative one."""
    rows, D = X.shape
    q, n_seg = Wa.shape[0], rows // seg
    pre = X @ Wa.t() + ba
    e = 4 * U32 * (-(-D // 16) + 2) * (X.abs() @ Wa.abs().t() + ba.abs())
    t = torch.tanh(pre)
    s = (t @ qv).view(n_seg, seg)
    ds = ((e + TANH_ERR) @ qv.abs() + q * U32 * (t.abs() @ qv.abs())).view(n_seg, seg)
    wr = torch.softmax(s, dim=1)
    xe = (2 * (s - s.max(dim=1, keepdim=True).values).abs() + 4) * U32
    dw_rel = wr * (2 * ds.max(dim=1, keepdim=True).values + xe + (wr * xe).sum(dim=1, keepdim=True) + (seg + 2) * U32)
    dw = dw_rel + 2.0 ** -126
    Xs, Xa = X, X.abs()
    if X_lo is not None:
        Xs, Xa = X + X_lo, Xa + X_lo.abs()
    n = 2 * seg if X_lo is not None else seg
    ref = torch.einsum("ns,nsd->nd", wr, Xs.view(n_seg, seg, D))
    bound = torch.einsum("ns,nsd->nd", dw, Xa.view(n_seg, seg, D)) + (n + 1) * U32 * torch.einsum("ns,nsd->nd", wr, Xa.view(n_seg, seg, D))
    res = {"out_ratio": _worst(_safe_div((out.double() - ref).abs(), bound))}
    if w is not None:
        # like the bf16 rounding of the GEMM judge: the share of the relative allowance used beyond the flush to zero
        res["w_ratio"] = _worst(_safe_div(((w.double().view(n_seg, seg) - wr).abs() - 2.0 ** -126).clamp_min(0), dw_rel))
    return res


def check_element_encoder(n=512 * 55, E=100, F=400, V=300, seed=3):
    """NAML category / subcategory encoder relu(Linear(embedding(id))) through nr_element_encoder_fwd / _bwd: exact gather,
    fp32 output per element, the ReLU mask the backward takes from the fp32 output (bit-exact dY), the bias column of dW_ext
    and the dtable scatter (row 0 and out-of-range ids skipped, repeated ids summed) per row."""
    lib = load_library()
    lde, ldf = ru8(E + 1), ru8(F + 1)
    table_f = _rand_bf16((V, E), seed).to(DEV)
    W = _rand_bf16((F, E), seed + 1, math.sqrt(3.0 / E)).to(DEV)
    bias = O.det_uniform((F,), seed + 2, -0.3, 0.3).to(DEV)
    ids = O.det_randint((n,), seed + 3, 0, V)
    ids[0], ids[-1] = 0, V - 1
    if n >= 8:
        ids[n // 3], ids[n // 2] = V + 5, -1
    ids = ids.to(DEV)
    table, w, wT = cast_pad(table_f, lde), cast_pad(W, lde), cast_pad(W, ldf, transpose=True)
    Eb = _Guarded(n * lde, torch.bfloat16, float("nan"))
    out = _Guarded(n * F, torch.float32, float("nan"))
    flag = _Guarded(1, torch.int32, 0, sentinel=-7)
    check(lib.nr_element_encoder_fwd(_p(ids), n, _p(table), V, E, lde, _p(Eb.all), _p(w), F, _p(bias), _p(out.all), _p(flag.all),
                                     _stream()), "nr_element_encoder_fwd")
    bad = (ids < 0) | (ids >= V)
    safe = torch.where(bad, torch.zeros_like(ids), ids)
    exp_e = torch.zeros(n, lde, device=DEV)
    exp_e[:, :E] = table_f[safe]
    exp_e[:, E] = 1.0
    e64 = Eb.body.view(n, lde)[:, :E].double()
    pre = e64 @ W.double().t() + bias.double()
    ref = pre.clamp_min(0)
    absum = e64.abs() @ W.double().abs().t() + bias.double().abs()
    o = out.body.view(n, F)
    res = {"gather_exact": _bits_equal(Eb.body.view(n, lde), exp_e.to(torch.bfloat16)), "bad_id_flag": int(flag.body.item()),
           "out_elem_ratio": _worst(_safe_div((o.double() - ref).abs(), 1e-6 * absum)),
           "relu_zero_exact": bool((o[pre < -1e-5 * absum] == 0).all())}
    dout = O.det_uniform((n, F), seed + 4).to(DEV)
    dY = _Guarded(n * ldf, torch.bfloat16, float("nan"))
    pat = lambda m, s: O.det_uniform((m,), s, 0.5, 1.0).to(DEV) * 2.0 ** -16
    dW = _Guarded(F * lde, torch.float32, pat(F * lde, seed + 5))
    dt = _Guarded(V * E, torch.float32, pat(V * E, seed + 6))
    check(lib.nr_element_encoder_bwd(_p(ids), n, _p(dout), _p(out.all), F, _p(dY.all), ldf, _p(Eb.all), E, lde, _p(wT), _p(dW.all),
                                     _p(dt.all), V, _stream()), "nr_element_encoder_bwd")
    torch.cuda.synchronize()
    exp_dy = torch.zeros(n, ldf, device=DEV)
    exp_dy[:, :F] = torch.where(o > 0, dout, torch.zeros_like(dout))  # the kernel writes +0 where the ReLU was off
    res["dY_relu_mask_exact"] = _bits_equal(dY.body.view(n, ldf), exp_dy.to(torch.bfloat16))
    dy64 = dY.body.view(n, ldf)[:, :F].double()
    e1 = torch.cat([e64, torch.ones(n, 1, dtype=torch.float64, device=DEV)], 1)
    dW_k = dW.body.view(F, lde)[:, :E + 1].double() - dW.prefill.view(F, lde)[:, :E + 1].double()
    res["dW_row_ratio"] = _abs_allow_rows(dW_k, dy64.t() @ e1, dy64.abs().t() @ e1.abs())
    res["dW_bias_col_ratio"] = _worst(_safe_div((dW_k[:, E] - dy64.sum(0)).abs(), dy64.abs().sum(0)))
    colmask = torch.zeros(F, lde, dtype=torch.bool, device=DEV)
    colmask[:, E + 1:] = True
    res["dW_pitch_cols_untouched"] = dW.unchanged(colmask)
    scat = (ids >= 1) & (ids < V)
    dX = dy64 @ W.double()
    ref_t = torch.zeros(V, E, dtype=torch.float64, device=DEV).index_add_(0, ids[scat], dX[scat])
    abs_t = torch.zeros(V, E, dtype=torch.float64, device=DEV).index_add_(0, ids[scat], (dy64.abs() @ W.double().abs())[scat])
    touched = torch.zeros(V, dtype=torch.bool, device=DEV)
    touched[ids[scat]] = True
    dt_k = dt.body.view(V, E).double() - dt.prefill.view(V, E).double()
    res["dtable_row_ratio"] = _abs_allow_rows(dt_k[touched], ref_t[touched], abs_t[touched])
    res["dtable_untouched_rows_exact"] = dt.unchanged((~touched).view(V, 1).expand(V, E))
    res["guards_intact"] = all(g.guard_ok() for g in (Eb, out, flag, dY, dW, dt))
    return res


def check_linear_rows(n=4000, K=300, N=275, relu=1, strided=False, with_dx=True, seed=5):
    """nr_linear_rows_fwd / _bwd (TANR topic predictor, GRU projections): bf16 operand rows (exact), fp32 output per element,
    masked bf16 dY (exact), dW_ext per row with its bias column (K + 1 > 512 columns are split across two weight-gradient
    calls), dx per element, or dx = NULL."""
    lib = load_library()
    ldx, ldn = ru8(K + 1), ru8(N + 1)
    ld_out = (N + 3) // 4 * 4
    base = O.det_uniform((n, 2 * K if strided else K), seed).to(DEV)
    x = base[:, ::2] if strided else base  # strided: element stride 2 inside a row
    W = _rand_bf16((N, K), seed + 1, math.sqrt(3.0 / K)).to(DEV)
    bias = O.det_uniform((N,), seed + 2, -0.2, 0.2).to(DEV)
    w, wT = cast_pad(W, ldx), cast_pad(W, ldn, transpose=True)
    X = _Guarded(n * ldx, torch.bfloat16, float("nan"))
    out = _Guarded(n * ld_out, torch.float32, float("nan"))
    check(lib.nr_linear_rows_fwd(_p(x), n, K, x.stride(0), x.stride(1), _p(X.all), ldx, _p(w), N, ldx, _p(bias), relu, _p(out.all),
                                 ld_out, _stream()), "nr_linear_rows_fwd")
    exp_x = torch.zeros(n, ldx, device=DEV)
    exp_x[:, :K] = x
    exp_x[:, K] = 1.0
    x64 = X.body.view(n, ldx)[:, :K].double()
    pre = x64 @ W.double().t() + bias.double()
    ref = pre.clamp_min(0) if relu else pre
    absum = x64.abs() @ W.double().abs().t() + bias.double().abs()
    o = out.body.view(n, ld_out)[:, :N]
    res = {"x_rows_exact": _bits_equal(X.body.view(n, ldx), exp_x.to(torch.bfloat16)),
           "out_elem_ratio": _worst(_safe_div((o.double() - ref).abs(), 1e-6 * absum))}
    dy = _Guarded(n * ld_out, torch.float32, 0.0)
    dy.body.view(n, ld_out)[:, :N] = O.det_uniform((n, N), seed + 3).to(DEV)
    dY = _Guarded(n * ldn, torch.bfloat16, float("nan"))
    dW = _Guarded(N * ldx, torch.float32, O.det_uniform((N * ldx,), seed + 4, 0.5, 1.0).to(DEV) * 2.0 ** -16)
    ld_dx = (K + 3) // 4 * 4
    dx = _Guarded(n * ld_dx, torch.float32, float("nan")) if with_dx else None
    check(lib.nr_linear_rows_bwd(_p(dy.all), _p(out.all) if relu else None, n, N, ld_out, _p(dY.all), ldn, _p(X.all), K, ldx, _p(wT),
                                 ldn, _p(dW.all), _p(dx.all) if with_dx else None, ld_dx, _stream()), "nr_linear_rows_bwd")
    torch.cuda.synchronize()
    g = dy.body.view(n, ld_out)[:, :N]
    exp_dy = torch.zeros(n, ldn, device=DEV)
    exp_dy[:, :N] = torch.where(o > 0, g, torch.zeros_like(g)) if relu else g
    res["dY_exact"] = _bits_equal(dY.body.view(n, ldn), exp_dy.to(torch.bfloat16))
    dy64 = dY.body.view(n, ldn)[:, :N].double()
    x1 = torch.cat([x64, torch.ones(n, 1, dtype=torch.float64, device=DEV)], 1)
    dW_k = dW.body.view(N, ldx)[:, :K + 1].double() - dW.prefill.view(N, ldx)[:, :K + 1].double()
    res["dW_row_ratio"] = _abs_allow_rows(dW_k, dy64.t() @ x1, dy64.abs().t() @ x1.abs())
    res["dW_bias_col_ratio"] = _worst(_safe_div((dW_k[:, K] - dy64.sum(0)).abs(), dy64.abs().sum(0)))
    colmask = torch.zeros(N, ldx, dtype=torch.bool, device=DEV)
    colmask[:, K + 1:] = True
    res["dW_pitch_cols_untouched"] = dW.unchanged(colmask)
    if with_dx:
        dxk = dx.body.view(n, ld_dx)[:, :K].double()
        res["dx_elem_ratio"] = _worst(_safe_div((dxk - dy64 @ W.double()).abs(), 1e-6 * (dy64.abs() @ W.double().abs())))
    res["guards_intact"] = all(b.guard_ok() for b in (X, out, dy, dY, dW) + ((dx,) if with_dx else ()))
    return res


def check_embedding_f32(n=512 * 55, V=300, D=100, seed=7):
    """nr_embedding_f32_fwd / _bwd (LSTUR category and user embeddings): the lookup is bit exact (out-of-range ids read row 0
    and raise the flag); the backward adds each touched row's fp64 sum, leaves row 0 and unused rows bit-identical."""
    lib = load_library()
    table = O.det_uniform((V, D), seed).to(DEV)
    ids = O.det_randint((n,), seed + 1, 0, V)
    ids[0], ids[-1] = 0, V - 1
    if n >= 8:
        ids[n // 3], ids[n // 2] = V + 5, -1
    ids = ids.to(DEV)
    out = _Guarded(n * D, torch.float32, float("nan"))
    flag = _Guarded(1, torch.int32, 0, sentinel=-7)
    check(lib.nr_embedding_f32_fwd(_p(ids), n, _p(table), V, D, _p(out.all), _p(flag.all), _stream()), "nr_embedding_f32_fwd")
    bad = (ids < 0) | (ids >= V)
    safe = torch.where(bad, torch.zeros_like(ids), ids)
    res = {"fwd_exact": _bits_equal(out.body.view(n, D), table[safe]), "bad_id_flag": int(flag.body.item())}
    dout = O.det_uniform((n, D), seed + 2).to(DEV)
    dt = _Guarded(V * D, torch.float32, O.det_uniform((V * D,), seed + 3, 0.5, 1.0).to(DEV) * 2.0 ** -16)
    check(lib.nr_embedding_f32_bwd(_p(ids), n, _p(dout), V, D, _p(dt.all), _stream()), "nr_embedding_f32_bwd")
    torch.cuda.synchronize()
    scat = (ids >= 1) & (ids < V)
    ref = torch.zeros(V, D, dtype=torch.float64, device=DEV).index_add_(0, ids[scat], dout[scat].double())
    absr = torch.zeros(V, D, dtype=torch.float64, device=DEV).index_add_(0, ids[scat], dout[scat].double().abs())
    touched = torch.zeros(V, dtype=torch.bool, device=DEV)
    touched[ids[scat]] = True
    dk = dt.body.view(V, D).double() - dt.prefill.view(V, D).double()
    res["bwd_row_ratio"] = _abs_allow_rows(dk[touched], ref[touched], absr[touched])
    res["untouched_rows_exact"] = dt.unchanged((~touched).view(V, 1).expand(V, D))
    res["row0_untouched"] = not bool(touched[0])
    res["guards_intact"] = all(b.guard_ok() for b in (out, flag, dt))
    return res


# ------------------------------------------------------------------------------------------------
# The NRMS / Exp1 self-attention encoder (nr_mhsa_encoder_fwd / _bwd): the same treatment as the CNN encoder above, stage by
# stage, for the four forward variants and their backward.  The fp64 backward chain is a plain function of tensors so that
# tests/test_mhsa_encoder_host.py can check it against torch.autograd through the oracle on the CPU.
# ------------------------------------------------------------------------------------------------
def _bf16_round(t):
    return t.to(torch.bfloat16).to(t.dtype)


def mhsa_attention_probs(Q, K, heads):
    """A = exp(S) / (sum_j exp(S) + 1e-8) with S = Q_h K_h^T / sqrt(d_k) per head (multihead_self.py:15-23), in its
    max-subtracted form, in the inputs' dtype: Q, K (n, T, d) -> (n, heads, T, T)."""
    n, T, d = Q.shape
    dk = d // heads
    sp = lambda t: t.reshape(n, T, heads, dk).transpose(1, 2)
    S = sp(Q) @ sp(K).transpose(-1, -2) / math.sqrt(dk)
    m = S.amax(-1, keepdim=True)
    e = torch.exp(S - m)
    return e / (e.sum(-1, keepdim=True) + 1e-8 * torch.exp(-m))


def mhsa_pool_bwd_chain(X, Q, K, V, C, w, W3, Wa, ba, qv, dout, heads, ctx_mask=None, contract=False, dpre=None):
    """The backward of one self-attention + additive-pooling encoder written out stage by stage, in the inputs' dtype, from
    the forward values the kernels stored: X (n, T, d) the projection's input rows, Q, K, V (n, T, d), C (n, T, d) the
    context the pooling read, w (n, T), W3 (3, d, d) = W_Q | W_K | W_V, Wa (q, d), ba, qv (q,), dout (n, d) and ctx_mask
    (n, T, d) the context-dropout multipliers (None: no dropout).  contract=True rounds to bf16 where the kernels store bf16:
    dPre, dC, dS (the gradient w.r.t. the unscaled product Q K^T, as oracle.scaled_dot_product_attention does), A as the
    operand of dV, and dQ | dK | dV.  dpre (n T, q), if given, is used as the stored dPre instead (the kernels' own, which a
    separate element bound judges).  Returns dqv (q,), dWa_ext (q, d + 1), dW3_ext (3, d, d + 1) (column d: the bias) and
    dX (n, T, d), the gradient of the projection's input rows."""
    r = _bf16_round if contract else (lambda t: t)
    n, T, d = X.shape
    dk = d // heads
    one = torch.ones(n * T, 1, dtype=X.dtype, device=X.device)
    C2 = C.reshape(n * T, d)
    # additive pooling (additive.py:35-53): dscore -> dPre -> dqv, dWa_ext; dC = (dPre Wa + w dout) * context mask
    dw = (C * dout.unsqueeze(1)).sum(2)
    dscore = w * (dw - (w * dw).sum(1, keepdim=True))
    th = torch.tanh(C2 @ Wa.t() + ba)
    if dpre is None:
        dpre = r(dscore.reshape(-1, 1) * qv * (1 - th * th))
    dqv = (dscore.reshape(-1, 1) * th).sum(0)
    dWa = dpre.t() @ torch.cat([C2, one], 1)
    dC = dpre @ Wa + w.reshape(-1, 1) * dout.repeat_interleave(T, 0)
    if ctx_mask is not None:
        dC = dC * ctx_mask.reshape(n * T, d)
    dC = r(dC)
    # attention: A recomputed; dV = A^T dC, dA = dC V^T, dS = A (dA - sum A dA) / sqrt(d_k), dQ = dS K, dK = dS^T Q
    sp = lambda t: t.reshape(n, T, heads, dk).transpose(1, 2)
    mg = lambda t: t.transpose(1, 2).reshape(n * T, d)
    A = mhsa_attention_probs(Q, K, heads)
    G = sp(dC)
    dV = r(A).transpose(-1, -2) @ G
    dA = G @ sp(V).transpose(-1, -2)
    dS = r(A * (dA - (A * dA).sum(-1, keepdim=True)) / math.sqrt(dk))
    dQKV = [r(mg(t)) for t in (dS @ sp(K), dS.transpose(-1, -2) @ sp(Q), dV)]
    # projection (multihead_self.py:53-58): dX = dQ|dK|dV . W_Q|W_K|W_V, dW_ext = dQKV^T [X, 1]
    X1 = torch.cat([X.reshape(n * T, d), one], 1)
    dX = dQKV[0] @ W3[0] + dQKV[1] @ W3[1] + dQKV[2] @ W3[2]
    return dict(dqv=dqv, dWa=dWa, dW3=torch.stack([g.t() @ X1 for g in dQKV]), dX=dX.view(n, T, d))


def check_mhsa_encoder(n_seq=37, T=20, d=300, heads=15, q=200, V=500, p_drop=0.2, level="ids", mode="accurate", pos=False,
                       noncontig=False, seed=1, bad_ids=True, discriminate=False, grad_floor=2e-3):
    """nr_mhsa_encoder_fwd / _bwd stage by stage against fp64 references built from the kernels' own stored X, Q|K|V, C, w.
    level "ids" (news encoder: masked gather, context dropout, embedding scatter) or "dense" (user encoder: fp32 rows
    [+ pos], input and positional gradient); mode "fast" or "accurate" (ids: V / probabilities / context as hi/lo pairs;
    dense: the precise variant, fp32 Q|K|V and attention, hi/lo context).  Every "=" output starts as NaN, every "+=" output
    with a small pattern, the workspace with 0xFF; every buffer, the packed operands included, is followed by a guard, and
    the packed Q|K|V operands and dWqkv_ext are sized 3*sec rows (include/newsrec_b200.h).  Bounds: tests/test_gpu_mhsa_encoder.py."""
    from newsrec_b200 import MhsaEncoderBwdArgs, MhsaEncoderFwdArgs
    from newsrec_b200.ops import qkv_pitches, stack_qkv
    lib = load_library()
    ids_level = level == "ids"
    accurate = mode == "accurate"
    precise = accurate and not ids_level
    ldx, ldq = ru8(d + 1), ru16(q)
    sec, ld3 = qkv_pitches(d)
    n_tok = n_seq * T
    p_ctx = p_drop if ids_level else 0.0  # the dense (user-level) variant has no dropout
    # ---- operands, built the way ops.mhsa_operands / MhsaPoolEncoderFn do; Q, K entries of about unit size
    a_w = 3.0 / math.sqrt(d)
    Wqkv = [_rand_bf16((d, d), seed + 1 + i, a_w).to(DEV) for i in range(3)]
    bqkv_l = [O.det_uniform((d,), seed + 4 + i, -0.1, 0.1).to(DEV) for i in range(3)]
    Wa = _rand_bf16((q, d), seed + 7, math.sqrt(3.0 / d)).to(DEV)
    ba = O.det_uniform((q,), seed + 8, -0.1, 0.1).to(DEV)
    qv = O.det_uniform((q,), seed + 9, -1.0, 1.0).to(DEV)
    wqkv_f = stack_qkv(*Wqkv)
    G_ = lambda t: _Guarded(t.numel(), t.dtype, t)  # a read-only operand followed by its guard
    ops = dict(wqkv=G_(cast_pad(wqkv_f, ldx)), wqkvT=G_(cast_pad(wqkv_f, ld3, transpose=True)), bqkv=G_(stack_qkv(*bqkv_l)),
               wa=G_(cast_pad(Wa, ldx)), waT=G_(cast_pad(Wa, ldq, transpose=True)), ba=G_(ba), qv=G_(qv))
    assert ops["wqkv"].n == 3 * sec * ldx and ops["bqkv"].n == 3 * sec
    if precise:
        kc = torch.nn.functional.pad(wqkv_f, (0, ldx - d))
        ops["kcat"] = G_(cast_pad(torch.cat((kc, kc), 1), 2 * ldx))
    ids = table_f = dense = posv = None
    if ids_level:
        table_f = _rand_bf16((V, d), seed + 10).to(DEV)
        ops["table"] = G_(cast_pad(table_f, ldx))
        ids = _cnn_ids(n_seq, T, V, seed + 11, bad_ids)
    else:
        base = O.det_uniform((T, max(n_seq, 1), d), seed + 12).to(DEV)
        dense = base.transpose(0, 1) if noncontig else base.transpose(0, 1).contiguous()  # (n, T, d)
        if pos:
            posv = O.det_uniform((T, d), seed + 13, -0.1, 0.1).to(DEV)
    kseed = (0x9E3779B97F4A7C15 * (seed + 17)) & 0xFFFFFFFFFFFFFFFF

    def forward():
        nan = float("nan")
        fb = dict(X=_Guarded(n_tok * ldx, torch.bfloat16, nan), C=_Guarded(n_tok * ldx, torch.bfloat16, nan),
                  w=_Guarded(n_tok, torch.float32, nan), out=_Guarded(n_seq * d, torch.float32, nan),
                  flag=_Guarded(1, torch.int32, 0, sentinel=-7))
        if not precise:
            fb["QKV"] = _Guarded(n_tok * ld3, torch.bfloat16, nan)
        if accurate:
            fb["Clo"] = _Guarded(n_tok * ldx, torch.bfloat16, nan)
        if accurate and ids_level:
            fb["Vlo"] = _Guarded(n_tok * sec, torch.bfloat16, nan)
        if precise:
            fb["Xk"] = _Guarded(n_tok * 2 * ldx, torch.bfloat16, nan)
            fb["Q32"] = _Guarded(n_tok * 3 * sec, torch.float32, nan)
        a = MhsaEncoderFwdArgs()
        a.n_seq, a.T, a.d, a.heads, a.q, a.ldx, a.ld3 = n_seq, T, d, heads, q, ldx, ld3
        if ids_level:
            a.ids, a.table_bf16, a.V = _p(ids), _p(ops["table"].all), V
        else:
            a.dense = _p(dense)
            a.dense_s_seq, a.dense_s_tok, a.dense_s_col = dense.stride()
            a.dense_pos = _p(posv)
        a.wqkv_bf16, a.bqkv, a.wa_bf16 = _p(ops["wqkv"].all), _p(ops["bqkv"].all), _p(ops["wa"].all)
        a.ba, a.qv = _p(ops["ba"].all), _p(ops["qv"].all)
        a.p_drop, a.seed = float(p_drop), kseed
        a.X_bf16, a.C_bf16, a.w, a.out = _p(fb["X"].all), _p(fb["C"].all), _p(fb["w"].all), _p(fb["out"].all)
        a.QKV_bf16 = _p(fb["QKV"].all) if "QKV" in fb else None
        a.bad_id_flag = _p(fb["flag"].all)
        if accurate:
            a.C_lo_bf16 = _p(fb["Clo"].all)
        if "Vlo" in fb:
            a.V_lo_bf16 = _p(fb["Vlo"].all)
        if precise:
            a.wqkv_kcat_bf16, a.X_kcat_bf16, a.QKV_f32 = _p(ops["kcat"].all), _p(fb["Xk"].all), _p(fb["Q32"].all)
        n0 = int(lib.nr_launch_count())
        rc = lib.nr_mhsa_encoder_fwd(C.byref(a), _stream())
        launches = int(lib.nr_launch_count()) - n0
        if rc != 0:  # a refused shape: what the library said and how much it launched before saying it
            return None, {"fwd_rejected": lib.nr_last_error().decode(), "fwd_launches": launches}
        return fb, launches

    fb, fwd_launches = forward()
    if fb is None:
        return fwd_launches
    dout = O.det_uniform((max(n_seq, 1), d), seed + 14).to(DEV)
    pat = lambda n, s: O.det_uniform((n,), s, 0.5, 1.0).to(DEV) * 2.0 ** -16  # small non-zero "+=" pre-fill
    bb = dict(dW3=_Guarded(3 * sec * ldx, torch.float32, pat(3 * sec * ldx, seed + 20)),
              dWa=_Guarded(q * ldx, torch.float32, pat(q * ldx, seed + 21)), dqv=_Guarded(q, torch.float32, pat(q, seed + 22)))
    if ids_level:
        bb["demb"] = _Guarded(V * d, torch.float32, pat(V * d, seed + 23))
    else:
        bb["ddense"] = _Guarded(n_tok * d, torch.float32, float("nan"))
        if pos:
            bb["dpos"] = _Guarded(T * d, torch.float32, pat(T * d, seed + 24))
    ws_bytes = int(lib.nr_mhsa_encoder_bwd_workspace(n_seq, T, d, q))
    ws = _Guarded(ws_bytes, torch.uint8, 0xFF, sentinel=0xA5)  # 0xFFFF.. = NaN in bf16 and fp32: unwritten rows poison results
    b = MhsaEncoderBwdArgs()
    b.n_seq, b.T, b.d, b.heads, b.q, b.ldx, b.ld3, b.ldq = n_seq, T, d, heads, q, ldx, ld3, ldq
    b.ids, b.V = (_p(ids), V) if ids_level else (None, 0)
    b.wqkvT_bf16, b.wa_bf16, b.waT_bf16 = _p(ops["wqkvT"].all), _p(ops["wa"].all), _p(ops["waT"].all)
    b.ba, b.qv = _p(ops["ba"].all), _p(ops["qv"].all)
    b.p_drop, b.seed = float(p_drop), kseed
    b.X_bf16, b.C_bf16, b.w, b.dout = _p(fb["X"].all), _p(fb["C"].all), _p(fb["w"].all), _p(dout)
    b.QKV_bf16 = _p(fb["QKV"].all) if "QKV" in fb else None  # precise: recomputed from X inside the backward
    b.wqkv_bf16, b.bqkv = _p(ops["wqkv"].all), _p(ops["bqkv"].all)
    b.dWqkv_ext, b.dWa_ext, b.dqv = _p(bb["dW3"].all), _p(bb["dWa"].all), _p(bb["dqv"].all)
    if ids_level:
        b.demb = _p(bb["demb"].all)
    else:
        b.ddense = _p(bb["ddense"].all)
        b.dpos = _p(bb["dpos"].all) if pos else None
    b.workspace, b.workspace_bytes = _p(ws.all), ws_bytes
    n0 = int(lib.nr_launch_count())
    check(lib.nr_mhsa_encoder_bwd(C.byref(b), _stream()), "nr_mhsa_encoder_bwd")
    bwd_launches = int(lib.nr_launch_count()) - n0
    torch.cuda.synchronize()
    res = {"fwd_launches": fwd_launches, "bwd_launches": bwd_launches,
           "guards_intact": all(g.guard_ok() for g in list(fb.values()) + list(bb.values()) + list(ops.values()) + [ws])}
    # the backward's first two stages as the kernels stored them in the workspace (abi.cu MhsaBwdWorkspace: fp32 dscore
    # [rows], then bf16 dPre [rows][ldq], each region 256-byte aligned), so that each is judged on its own inputs
    ds_ws = ws.body[:n_tok * 4].view(torch.float32).clone()
    off = (n_tok * 4 + 255) // 256 * 256
    dpre_ws = ws.body[off:off + n_tok * ldq * 2].view(torch.bfloat16).view(n_tok, ldq)[:, :q].clone()
    del ws
    if n_seq == 0:
        return res
    if ids_level:
        res["bad_id_flag"] = int(fb["flag"].body.item())
        ids_flat = ids.reshape(-1)
        bad = (ids_flat < 0) | (ids_flat >= V)
        res["bad_ids_planted"] = int(bad.sum())
        ids_safe = torch.where(bad, torch.zeros_like(ids_flat), ids_flat)
        scat = (ids_flat >= 1) & (ids_flat < V)
    res["fwd_outputs_finite"] = all(bool(torch.isfinite(fb[k].body.float()).all()) for k in ("X", "C", "w", "out") + (("Clo",) if accurate else ()))

    # ---- fp64 references, a chunk of sequences at a time (a few hundred MB of fp64 temporaries at any n_seq)
    X2, C2, w1 = fb["X"].body.view(n_tok, ldx), fb["C"].body.view(n_tok, ldx), fb["w"].body
    Clo2 = fb["Clo"].body.view(n_tok, ldx) if accurate else None
    QKV2 = fb["QKV"].body.view(n_tok, ld3) if "QKV" in fb else None
    Vlo2 = fb["Vlo"].body.view(n_tok, sec) if "Vlo" in fb else None
    Xk2, Q32 = (fb["Xk"].body.view(n_tok, 2 * ldx), fb["Q32"].body.view(n_tok, 3 * sec)) if precise else (None, None)
    out2 = fb["out"].body.view(n_seq, d)
    W3 = torch.stack(Wqkv).double()
    b3 = torch.stack(bqkv_l).double()
    Wa64, ba64, qv64 = Wa.double(), ba.double(), qv.double()
    metrics = ("qkv_ratio", "vlo_ratio", "qkv32_ratio", "ctx_ratio", "ctx_hi_only_ratio", "ctx_no_vlo_ratio", "w_err", "w_sum_err",
               "out_ratio", "dscore_ratio", "dpre_ratio")
    acc = {k: 0.0 for k in metrics}
    worst = lambda k, t: acc.__setitem__(k, max(acc[k], _worst(t)))
    cnt = dict(x_mismatch_rows=0, xk_mismatch_rows=0, ctx_dropped_nonzero=0)
    exact_flags = dict(qkv_pad_zero=True, ctx_ones_col=True, ctx_pitch_zero=True)
    variants = ("exact", "contract") + (("exact_no_ctx_mask", "contract_no_ctx_mask") if discriminate else ())
    grads = {v: dict(dW3=torch.zeros(3, d, d + 1, dtype=torch.float64, device=DEV),
                     dWa=torch.zeros(q, d + 1, dtype=torch.float64, device=DEV),
                     dqv=torch.zeros(q, dtype=torch.float64, device=DEV)) for v in variants}
    for v in variants:
        if ids_level:
            grads[v]["demb"] = torch.zeros(V, d, dtype=torch.float64, device=DEV)
        else:
            grads[v]["ddense"] = torch.zeros(n_tok, d, dtype=torch.float64, device=DEV)
    if discriminate and ids_level:
        grads["exact_no_gather_mask"] = dict(demb=torch.zeros(V, d, dtype=torch.float64, device=DEV))
        grads["contract_no_gather_mask"] = dict(demb=torch.zeros(V, d, dtype=torch.float64, device=DEV))
    cs = max(1, min(40960 // T, (1 << 24) // (heads * T * T)))
    for s0 in range(0, n_seq, cs):
        s1 = min(n_seq, s0 + cs)
        ns, r0, r1 = s1 - s0, s0 * T, s1 * T
        rows = torch.arange(r0, r1, device=DEV)
        # X: bit exact (masked gather or fp32 dense [+ pos] rounded once), ones column at d, zeros up to ldx
        if ids_level:
            mx = dropout_mask_dev(kseed, p_drop, rows, d, ldx)
            src = table_f[ids_safe[r0:r1]] * mx
        else:
            src = (dense[s0:s1] + posv if pos else dense[s0:s1]).reshape(-1, d)
        exp_x = torch.zeros(r1 - r0, ldx, dtype=torch.float32, device=DEV)
        exp_x[:, :d] = src
        exp_x[:, d] = 1.0
        exp_hi = exp_x.to(torch.bfloat16)
        cnt["x_mismatch_rows"] += int((X2[r0:r1].view(torch.int16) != exp_hi.view(torch.int16)).any(dim=1).sum())
        X64 = X2[r0:r1, :d].double()
        if precise:  # X_kcat = [hi | lo] of the same fp32 rows, as nr_rows_to_bf16_hilo writes them
            exp_lo = torch.zeros_like(exp_hi)
            exp_lo[:, :d] = (src - src.to(torch.bfloat16).float()).to(torch.bfloat16)
            exp_k = torch.cat([exp_hi, exp_lo], 1)
            cnt["xk_mismatch_rows"] += int((Xk2[r0:r1].view(torch.int16) != exp_k.view(torch.int16)).any(dim=1).sum())
            Xin = Xk2[r0:r1, :d].double() + Xk2[r0:r1, ldx:ldx + d].double()
        else:
            Xin = X64
        # Q|K|V against fp64 Xin . W^T + b, with the sum of |products| for the fp32 accumulation allowance
        ref = torch.stack([Xin @ W3[i].t() + b3[i] for i in range(3)])  # (3, rows, d)
        absum = torch.stack([Xin.abs() @ W3[i].abs().t() + b3[i].abs() for i in range(3)])
        if precise:
            got = torch.stack([Q32[r0:r1, i * sec:i * sec + d].double() for i in range(3)])
            worst("qkv32_ratio", _safe_div((got - ref).abs(), 1e-6 * absum))
            exact_flags["qkv_pad_zero"] &= all(bool((Q32[r0:r1, i * sec + d:(i + 1) * sec] == 0).all()) for i in range(3))
            Qa, Ka, Va = got[0], got[1], got[2]
        else:
            got = torch.stack([QKV2[r0:r1, i * sec:i * sec + d].double() for i in range(3)])
            worst("qkv_ratio", _safe_div((got - ref).abs(), _bf16_ulp(torch.maximum(got.abs(), ref.abs())) + 1e-6 * absum))
            exact_flags["qkv_pad_zero"] &= all(bool((QKV2[r0:r1, i * sec + d:(i + 1) * sec] == 0).all()) for i in range(3))
            Qa, Ka, Va = got[0], got[1], got[2]
            if Vlo2 is not None:
                Va = got[2] + Vlo2[r0:r1, :d].double()
                rb = 2.0 ** -16 * ref[2].norm(dim=1) + 1e-6 * absum[2].norm(dim=1)
                worst("vlo_ratio", _safe_div((Va - ref[2]).norm(dim=1), rb))
                exact_flags["qkv_pad_zero"] &= bool((Vlo2[r0:r1, d:] == 0).all())
        del ref, absum
        # context against fp64 mask * (A V), A from the stored Q, K
        sh = lambda t: t.reshape(ns, T, d)
        A = mhsa_attention_probs(sh(Qa), sh(Ka), heads)
        spv = lambda t: sh(t).reshape(ns, T, heads, d // heads).transpose(1, 2)
        mg = lambda t: t.transpose(1, 2).reshape(ns * T, d)
        AV, AabsV = mg(A @ spv(Va)), mg(A @ spv(Va.abs()))
        cm = dropout_mask_dev(kseed ^ 0x5BD1E995, p_ctx, rows, d, ldx).double()
        ref_c = AV * cm
        chi = C2[r0:r1, :d].double()
        if accurate:
            clo = Clo2[r0:r1, :d].double()
            bound = 2.0 ** -15 * AabsV * cm + 2.0 ** -16 * ref_c.abs()
            worst("ctx_ratio", _safe_div((chi + clo - ref_c).abs(), bound))
            worst("ctx_hi_only_ratio", _safe_div((chi - ref_c).abs(), bound))
            if Vlo2 is not None:  # a reference that leaves out V_lo: the kernel's pair must be far from it
                ref_nv = mg(A @ spv(got[2])) * cm
                worst("ctx_no_vlo_ratio", _safe_div((chi + clo - ref_nv).abs(), 2.0 ** -15 * AabsV * cm + 2.0 ** -16 * ref_nv.abs()))
            cnt["ctx_dropped_nonzero"] += int(((cm == 0) & ((chi != 0) | (clo != 0))).sum())
            exact_flags["ctx_ones_col"] &= bool((C2[r0:r1, d] == 1).all()) and bool((Clo2[r0:r1, d] == 0).all())
            exact_flags["ctx_pitch_zero"] &= bool((C2[r0:r1, d + 1:] == 0).all()) and bool((Clo2[r0:r1, d + 1:] == 0).all())
        else:
            ulps = _bf16_ulp(torch.maximum(chi.abs(), ref_c.abs())) * torch.where(cm > 1, 2.0, 1.0)
            bound = (2.0 ** -8 + 2.0 ** -15) * AabsV * cm + ulps
            rt = _safe_div((chi - ref_c).abs(), bound)
            if _worst(rt) > acc["ctx_ratio"]:
                i = int(torch.nan_to_num(rt, nan=float("inf")).argmax())
                res["ctx_worst"] = [float(t.reshape(-1)[i]) for t in (chi, ref_c, AabsV, cm, ulps)] + [r0 + i // d, i % d]
            worst("ctx_ratio", rt)
            cnt["ctx_dropped_nonzero"] += int(((cm == 0) & (chi != 0)).sum())
            exact_flags["ctx_ones_col"] &= bool((C2[r0:r1, d] == 1).all())
            exact_flags["ctx_pitch_zero"] &= bool((C2[r0:r1, d + 1:] == 0).all())
        del A, AV, AabsV, ref_c
        # pooling from the kernel's own C_hi (scores) and C_hi [+ C_lo] (pooled sum)
        score = torch.tanh(chi @ Wa64.t() + ba64) @ qv64
        w_ref = torch.softmax(score.view(ns, T), dim=1)
        wk = w1[r0:r1].double().view(ns, T)
        worst("w_err", (wk - w_ref).abs())
        worst("w_sum_err", (wk.sum(1) - 1).abs())
        cc = (chi + clo if accurate else chi).view(ns, T, d)
        o_ref, o_abs = (wk.unsqueeze(2) * cc).sum(1), (wk.unsqueeze(2) * cc.abs()).sum(1)
        worst("out_ratio", _safe_div((out2[s0:s1].double() - o_ref).norm(dim=1), o_abs.norm(dim=1)))
        # ---- backward, exact and under the bf16 contract, from the stored X, Q|K|V (the fp64 projection of the stored X where
        #      the backward recomputes it), C_hi and w; the contract takes the kernels' stored dPre (judged above), so the
        #      per-row rule measures the stages after it
        do = dout[s0:s1].double()
        # dscore = w (dw - sum w dw), dw = C_hi . dout: fp32 dot products of d terms (d 2^-24 sum |c||dout| each) and a few
        # fp32 operations on w (dw, sum w dw)
        cd = chi.view(ns, T, d) * do.unsqueeze(1)
        dw, aw = cd.sum(2), cd.abs().sum(2)
        ds_ref = wk * (dw - (wk * dw).sum(1, keepdim=True))
        ds_bound = wk * (d * 2.0 ** -24 * (aw + (wk * aw).sum(1, keepdim=True)) + 4 * 2.0 ** -24 * (dw.abs() + (wk * dw.abs()).sum(1, keepdim=True)))
        ds_k = ds_ws[r0:r1].double().view(ns, T)
        worst("dscore_ratio", _safe_div((ds_k - ds_ref).abs(), ds_bound))
        # dPre = dscore qv (1 - T^2) from the kernel's own dscore, T = tanh(C_hi Wa^T + ba): tanh.approx.f32 is within
        # 2^-10.987 of T relatively (PTX ISA), the fp32 pre-activation within 1e-6 sum |c||wa| (+|ba|), which moves T by
        # (1 - T^2) times that; 1 - T^2 then moves by up to 2|T| |dT| + dT^2; plus one bf16 ulp of the stored result
        pre = chi @ Wa64.t() + ba64
        th = torch.tanh(pre)
        dT = th.abs() * 2.0 ** -10.987 + (1 - th * th) * 1e-6 * (chi.abs() @ Wa64.abs().t() + ba64.abs())
        g1 = ds_k.reshape(-1, 1) * qv64
        dp_ref = g1 * (1 - th * th)
        dp_k = dpre_ws[r0:r1].double()
        dp_bound = g1.abs() * (2 * th.abs() * dT + dT * dT + 4 * 2.0 ** -24) + _bf16_ulp(torch.maximum(dp_ref.abs(), dp_k.abs()))
        worst("dpre_ratio", _safe_div((dp_k - dp_ref).abs(), dp_bound))
        del cd, pre, th, dT, g1, dp_ref
        if precise:
            proj = torch.stack([X64 @ W3[i].t() + b3[i] for i in range(3)])
        for v in variants:
            contract = v.startswith("contract")
            if precise:  # the backward recomputes Q|K|V from X_bf16 into a bf16 workspace
                qkv_in = [_bf16_round(t) if contract else t for t in proj]
            else:
                qkv_in = [got[0], got[1], got[2]]
            ch = mhsa_pool_bwd_chain(sh(X64), *[sh(t) for t in qkv_in], sh(chi), wk, W3, Wa64, ba64, qv64, do, heads,
                                     ctx_mask=None if v.endswith("no_ctx_mask") else sh(cm), contract=contract,
                                     dpre=dp_k if contract else None)
            g = grads[v]
            g["dqv"] += ch["dqv"]
            g["dWa"] += ch["dWa"]
            g["dW3"] += ch["dW3"]
            dX = ch["dX"].reshape(-1, d)
            if ids_level:
                sc = scat[r0:r1]
                g["demb"].index_add_(0, ids_flat[r0:r1][sc], (dX * mx.double())[sc])
                if discriminate and not v.endswith("no_ctx_mask"):
                    grads[v.split("_")[0] + "_no_gather_mask"]["demb"].index_add_(0, ids_flat[r0:r1][sc], dX[sc])
            else:
                g["ddense"][r0:r1] = dX
            del ch, dX
    res.update(acc)
    res.update(cnt)
    res.update(exact_flags)
    # ---- gradients: per row, kernel error against exact next to the bf16 contract's error
    ex, co = grads["exact"], grads["contract"]
    body = lambda k: bb[k].body.double() - (bb[k].prefill.double() if bb[k].prefill is not None else 0.0)
    dW3_k = body("dW3").view(3, sec, ldx)[:, :d, :d + 1]
    dWa_k = body("dWa").view(q, ldx)[:, :d + 1]
    dqv_k = body("dqv")
    rr = lambda kern, e, c: _row_ratio(kern, e, c, floor=grad_floor)
    # T = 1: A = 1 / (1 + 1e-8), so dS = A (dA - A dA) / sqrt(d_k) is 1e-8 of dA -- below fp32 resolution, the kernels' dQ, dK
    # are 0 -- and the Q, K rows of dWqkv_ext are 1e-8 of the V rows: they are held to that scale, the V rows to the rule
    s3 = slice(2, 3) if T == 1 else slice(0, 3)
    n3 = (s3.stop - s3.start) * d
    res["dWqkv_row_ratio"], res["dWqkv_ek"], res["dWqkv_ec"] = rr(dW3_k[s3].reshape(n3, -1), ex["dW3"][s3].reshape(n3, -1),
                                                                  co["dW3"][s3].reshape(n3, -1))
    if T == 1:
        res["t1_dWqk_rel"] = _worst(dW3_k[:2].abs()) / max(_worst(ex["dW3"][2].abs()), 1e-300)
    res["dWa_row_ratio"], res["dWa_ek"], res["dWa_ec"] = rr(dWa_k, ex["dWa"], co["dWa"])
    res["dqv_ratio"], res["dqv_ek"], res["dqv_ec"] = rr(dqv_k.view(1, -1), ex["dqv"].view(1, -1), co["dqv"].view(1, -1))
    if discriminate:
        res["dWqkv_ratio_without_ctx_mask"] = rr(dW3_k.reshape(3 * d, -1), grads["exact_no_ctx_mask"]["dW3"].reshape(3 * d, -1),
                                                 grads["contract_no_ctx_mask"]["dW3"].reshape(3 * d, -1))[0]
    # the pre-fill outside what the kernels own: section-padding rows and pitch columns of dWqkv_ext, pitch columns of dWa_ext
    m3 = torch.ones(3, sec, ldx, dtype=torch.bool, device=DEV)
    m3[:, :d, :d + 1] = False
    res["dWqkv_padding_untouched"] = bb["dW3"].unchanged(m3)
    ma = torch.zeros(q, ldx, dtype=torch.bool, device=DEV)
    ma[:, d + 1:] = True
    res["dWa_pitch_cols_untouched"] = bb["dWa"].unchanged(ma)
    if ids_level:
        touched = torch.zeros(V, dtype=torch.bool, device=DEV)
        touched[ids_flat[scat]] = True
        res["demb_rows_touched"] = int(touched.sum())
        demb_k = body("demb").view(V, d)
        res["demb_row_ratio"], res["demb_ek"], res["demb_ec"] = rr(demb_k[touched], ex["demb"][touched], co["demb"][touched])
        res["demb_untouched_rows_exact"] = bb["demb"].unchanged((~touched).view(V, 1).expand(V, d))
        res["demb_row0_untouched"] = bb["demb"].unchanged(torch.arange(V, device=DEV).view(V, 1).expand(V, d) == 0)
        if discriminate:
            res["demb_ratio_without_gather_mask"] = rr(demb_k[touched], grads["exact_no_gather_mask"]["demb"][touched],
                                                       grads["contract_no_gather_mask"]["demb"][touched])[0]
    else:
        dd_k = bb["ddense"].body.double().view(n_tok, d)
        res["ddense_row_ratio"], res["ddense_ek"], res["ddense_ec"] = rr(dd_k, ex["ddense"], co["ddense"])
        if pos:  # dpos = sum over the sequences of ddense
            sum_seq = lambda t: t.view(n_seq, T, d).sum(0)
            res["dpos_row_ratio"], res["dpos_ek"], res["dpos_ec"] = rr(body("dpos").view(T, d), sum_seq(ex["ddense"]),
                                                                       sum_seq(co["ddense"]))
    del grads, ex, co, bb

    # ---- determinism: a second forward is bit-identical (run last, when the references are freed)
    fb2, _ = forward()
    torch.cuda.synchronize()
    res["fwd_deterministic"] = all(_bits_equal(fb[k].body, fb2[k].body) for k in fb if k != "flag")
    return res


# ------------------------------------------------------------------------------------------------
# The LSTUR GRU (nr_gru_fwd / _bwd) step by step.  The fp64 step functions below work in the (S, B, .) layout on any device;
# tests/test_gru_host.py checks them against torch.autograd through the oracle on the CPU, tests/test_gpu_gru.py holds the
# kernels to them (bounds derived there).
# ------------------------------------------------------------------------------------------------
def gru_gates(gi, gh, Hd):
    """r, z, n of torch's gate order r | z | n and the pre-activations a_r, a_z, v = gi_n + r gh_n."""
    a_r = gi[..., :Hd] + gh[..., :Hd]
    a_z = gi[..., Hd:2 * Hd] + gh[..., Hd:2 * Hd]
    r, z = torch.sigmoid(a_r), torch.sigmoid(a_z)
    v = gi[..., 2 * Hd:] + r * gh[..., 2 * Hd:]
    return dict(r=r, z=z, n=torch.tanh(v), a_r=a_r, a_z=a_z, v=v)


def gru_proj(rows, w, b):
    """rows . w^T + b and the sum of |products| (with |b|): gi from the stored bf16 x rows (hi, then lo), gh[t] from hb[t]."""
    return rows @ w.t() + b, rows.abs() @ w.abs().t() + b.abs()


def gru_step(gi_t, gh_t, h_t, active):
    """hs[t+1] from gi[t], gh[t] and hs[t]; rows with active False (t >= max(len, 1)) keep h_t."""
    g = gru_gates(gi_t, gh_t, h_t.shape[-1])
    return torch.where(active.view(-1, 1), (1 - g["z"]) * g["n"] + g["z"] * h_t, h_t)


def gru_bwd_chain(gi, gh, hs, L, w_ih, w_hh, x_ext, h_ext, dout, contract=False, dgh_stored=None):
    """The backward of the recurrence written out step by step, in the inputs' dtype, from the forward values the kernels store:
    gi, gh (S, B, 3Hd), hs (S+1, B, Hd), L (B,) = max(len, 1), w_ih (3Hd, D), w_hh (3Hd, Hd), x_ext (S, B, D+1) and h_ext
    (S, B, Hd+1) the operand rows of the two projections with their ones column, dout (B, Hd).  contract=True rounds dgi and dgh
    to bf16 where the kernels store them.  The dh entering step t - 1 is dh z (frozen rows: dh) + dgh[t] W_hh, with dgh[t] the
    chain's own or, when dgh_stored is given, the kernel's stored one.  Returns dgi, dgh (S, B, 3Hd), dh (S, B, Hd) the gradient
    entering each step, dh0, dx (S, B, D), dWih (3Hd, D+1), dWhh (3Hd, Hd+1) (last column: the bias)."""
    S, B, H3 = gi.shape
    Hd = H3 // 3
    rnd = _bf16_round if contract else (lambda t: t)
    dgi, dgh, dh_in = torch.empty_like(gi), torch.empty_like(gh), torch.empty_like(hs[1:])
    dh = dout
    for t in range(S - 1, -1, -1):
        act = (t < L).view(-1, 1)
        g = gru_gates(gi[t], gh[t], Hd)
        r, z, n = g["r"], g["z"], g["n"]
        dh_in[t] = dh
        dn = dh * (1 - z)
        dz = dh * (hs[t] - n)
        dpn = dn * (1 - n * n)
        dpz = dz * z * (1 - z)
        dpr = dpn * gh[t, :, 2 * Hd:] * r * (1 - r)
        dgi[t] = rnd(torch.where(act, torch.cat([dpr, dpz, dpn], 1), 0.0))
        dgh[t] = rnd(torch.where(act, torch.cat([dpr, dpz, dpn * r], 1), 0.0))
        rec = (dgh[t] if dgh_stored is None else dgh_stored[t]) @ w_hh
        dh = torch.where(act, dh * z, dh) + rec
    flat = lambda t: t.reshape(S * B, -1)
    return dict(dgi=dgi, dgh=dgh, dh=dh_in, dh0=dh, dx=dgi @ w_ih, dWih=flat(dgi).t() @ flat(x_ext), dWhh=flat(dgh).t() @ flat(h_ext))


def gru_bwd_workspace_layout(B, S, Hd):
    """gru.cu GruBwdWorkspace: byte offsets of dgi bf16 [B*S][ldb] (rows b*S + t), dgh bf16 [S][B][ldb], dh_direct and dh_rec fp32
    [B][round_up(Hd, 4)], each region rounded up to 256 bytes, and the total (one more 256-byte slot)."""
    a256 = lambda n: (n + 255) // 256 * 256
    ldb, P = ru8(3 * Hd + 1), (Hd + 3) // 4 * 4
    off, lay = 0, {}
    for k, n in (("dgi", B * S * ldb * 2), ("dgh", B * S * ldb * 2), ("dh_direct", B * P * 4), ("dh_rec", B * P * 4)):
        lay[k] = off
        off += a256(n)
    return lay, off + 256


def gru_lengths(B, S, seed):
    """Lengths 1..S with 0, -3, 1, S - 1 and S planted at scattered rows (unsorted)."""
    lens = O.det_randint((B,), seed, 1, S + 1)
    for pos, v in zip((B // 2, 0, B - 1, B // 3, (2 * B) // 3), (0, -3, 1, S - 1, S)):
        if B > 0:
            lens[pos] = v
    return lens


_U = 2.0 ** -24      # fp32 unit roundoff
_EX2 = 2.0 ** -22    # ex2.approx.f32: 2 ulp, at most 2^-22 relative
_DIV = 2.0 ** -22    # div.approx.f32 (__fdividef): 2 ulp for divisors in [2^-126, 2^126]
_TINY = 2.0 ** -100  # flush-to-zero of results below 2^-126 and the divisors above 2^126


def gru_gate_errors(g, gh_n):
    """Absolute error bounds of the kernels' fp32 gates on the stored gi, gh (tests/test_gpu_gru.py derives them): r, z, n."""
    def sig(a, s):
        return s * ((1 - s) * (3 * _U * a.abs() + _EX2) + _U + _DIV) + _TINY
    Er, Ez = sig(g["a_r"], g["r"]), sig(g["a_z"], g["z"])
    n, v = g["n"], g["v"]
    Ev = gh_n.abs() * Er + _U * (g["r"] * gh_n).abs() + _U * v.abs()
    En = (1 - n * n) * Ev + (1 - n * n) / 2 * (4 * _U * v.abs() + _EX2) + (1 - n) * (_U + _DIV) + _U * n.abs() + _TINY
    return Er, Ez, En


def _dev_error(lib):
    e = (C.c_int * 4)()
    lib.nr_device_error(C.byref(e))
    return list(e)


def check_gru_stages(B=37, S=50, D=900, Hd=900, accurate=True, h0_zero=False, x_layout="contig", wscale=1.0, seed=3,
                     paths=("default",), e2e=True):
    """nr_gru_fwd / _bwd stage by stage against fp64 references built from what the kernels stored (gi, gh, hs, hb, and the
    workspace's dgi, dgh, dh_direct, dh_rec), per element.  paths: "default" (the library's choice), "persistent" / "stepwise"
    (nr_debug_set_gru_stepwise 0 / 1); each path runs its own forward and backward on the same operands.  x_layout: "contig",
    "perm" ([S][B][D] storage), "col2" (column stride 2), "slice" (s_b > S D); storage elements x does not cover are NaN.
    Every "=" output starts as NaN, the "+=" outputs with a small pattern, the workspace with 0xFF; every buffer, the operands
    included, is followed by a guard.  Bounds: tests/test_gpu_gru.py."""
    import os
    from newsrec_b200 import GruBwdArgs, GruFwdArgs
    from newsrec_b200.ops_gru import ru4
    lib = load_library()
    ldd, ldh, ldg, ldb = ru8(D + 1), ru8(Hd + 1), ru4(3 * Hd), ru8(3 * Hd + 1)
    H3, R = 3 * Hd, B * S
    nan = float("nan")
    G_ = lambda t: _Guarded(t.numel(), t.dtype, t)
    a_w = wscale / math.sqrt(Hd)
    Wih, Whh = _rand_bf16((H3, D), seed, a_w).to(DEV), _rand_bf16((H3, Hd), seed + 1, a_w).to(DEV)
    bih = O.det_uniform((H3,), seed + 2, -a_w, a_w).to(DEV)
    bhh = O.det_uniform((H3,), seed + 3, -a_w, a_w).to(DEV)
    xv = O.det_uniform((B, S, D), seed + 4).to(DEV)
    h0v = torch.zeros(B, Hd, device=DEV) if h0_zero else O.det_uniform((B, Hd), seed + 5, -0.5, 0.5).to(DEV)
    lens = gru_lengths(B, S, seed + 6).to(DEV)
    dout = O.det_uniform((B, Hd), seed + 7).to(DEV)
    ops = dict(wih=G_(cast_pad(Wih, ldd)), whh=G_(cast_pad(Whh, ldh)), wihT=G_(cast_pad(Wih, ldb, transpose=True)),
               whhT=G_(cast_pad(Whh, ldb, transpose=True)), bih=G_(bih), bhh=G_(bhh), h0=G_(h0v), len=G_(lens), dout=G_(dout))
    # x: a strided view into guarded storage
    shape, off = {"contig": ((B, S, D), 0), "perm": ((S, B, D), 0), "col2": ((B, S, 2 * D), 0), "slice": ((B, S + 3, D), D)}[x_layout]
    xs = _Guarded(math.prod(shape), torch.float32, nan)
    st = xs.body.view(shape)
    x = {"contig": st, "perm": st.transpose(0, 1), "col2": st[..., ::2], "slice": st[:, 1:S + 1]}[x_layout]
    x.copy_(xv)
    ops["x"] = xs
    assert x_layout != "slice" or x.stride()[0] > S * D
    L = lens.clamp(min=1)
    act = torch.arange(S, device=DEV).view(S, 1) < L.view(1, B)  # (S, B)
    env_default = 1 if os.environ.get("NEWSREC_GRU_STEPWISE") is not None else 0

    def forward(path):
        fb = dict(xb=_Guarded(R * ldd, torch.bfloat16, nan), gi=_Guarded(R * ldg, torch.float32, nan),
                  gh=_Guarded(S * B * ldg, torch.float32, nan), hs=_Guarded((S + 1) * B * Hd, torch.float32, nan),
                  hb=_Guarded((S + 1) * B * ldh, torch.bfloat16, nan), out=_Guarded(B * Hd, torch.float32, nan))
        if accurate:
            fb["xlo"] = _Guarded(R * ldd, torch.bfloat16, nan)
        a = GruFwdArgs()
        a.B, a.S, a.D, a.Hd = B, S, D, Hd
        a.x = _p(x if x.numel() else xs.all)  # an empty view may report a null data pointer
        a.x_s_b, a.x_s_t, a.x_s_c = x.stride()
        a.len, a.h0 = _p(ops["len"].all), _p(ops["h0"].all)
        a.wih_bf16, a.whh_bf16, a.bih, a.bhh = _p(ops["wih"].all), _p(ops["whh"].all), _p(ops["bih"].all), _p(ops["bhh"].all)
        a.xb, a.gi, a.gh, a.hs, a.hb, a.out = (_p(fb[k].all) for k in ("xb", "gi", "gh", "hs", "hb", "out"))
        a.x_lo_bf16 = _p(fb["xlo"].all) if accurate else None
        lib.nr_debug_set_gru_stepwise({"default": env_default, "persistent": 0, "stepwise": 1}[path])
        try:
            n0 = int(lib.nr_launch_count())
            check(lib.nr_gru_fwd(C.byref(a), _stream()), "nr_gru_fwd")
            launches = int(lib.nr_launch_count()) - n0
        finally:
            lib.nr_debug_set_gru_stepwise(env_default)
        torch.cuda.synchronize()
        return fb, launches, _dev_error(lib)

    def backward(fb):
        pat = lambda n, s: O.det_uniform((n,), s, 0.5, 1.0).to(DEV) * 2.0 ** -16  # small non-zero "+=" pre-fill
        bb = dict(dWih=_Guarded(H3 * ldd, torch.float32, pat(H3 * ldd, seed + 20)),
                  dWhh=_Guarded(H3 * ldh, torch.float32, pat(H3 * ldh, seed + 21)),
                  dx=_Guarded(R * D, torch.float32, nan), dh0=_Guarded(B * Hd, torch.float32, nan))
        ws_bytes = int(lib.nr_gru_bwd_workspace(B, S, D, Hd))
        ws = _Guarded(ws_bytes, torch.uint8, 0xFF, sentinel=0xA5)  # 0xFFFF.. = NaN in bf16 and fp32
        b = GruBwdArgs()
        b.B, b.S, b.D, b.Hd = B, S, D, Hd
        b.len, b.wihT_bf16, b.whhT_bf16 = _p(ops["len"].all), _p(ops["wihT"].all), _p(ops["whhT"].all)
        b.xb, b.gi, b.gh, b.hs, b.hb = (_p(fb[k].all) for k in ("xb", "gi", "gh", "hs", "hb"))
        b.dout, b.dWih_ext, b.dWhh_ext, b.dx, b.dh0 = _p(ops["dout"].all), _p(bb["dWih"].all), _p(bb["dWhh"].all), _p(bb["dx"].all), \
            _p(bb["dh0"].all)
        b.workspace, b.workspace_bytes = _p(ws.all), ws_bytes
        n0 = int(lib.nr_launch_count())
        check(lib.nr_gru_bwd(C.byref(b), _stream()), "nr_gru_bwd")
        launches = int(lib.nr_launch_count()) - n0
        torch.cuda.synchronize()
        return bb, ws, launches, _dev_error(lib)

    res = {"persistent_supported": bool(lib.nr_gru_persistent_supported(B, Hd)), "sms": int(lib.nr_num_sms()), "paths": {}}
    saved = {}
    ref = None
    if B > 0 and e2e:
        ref = _gru_end_to_end_refs(xv, L, h0v, Wih, Whh, bih, bhh, dout, accurate)
    for path in paths:
        fb, fl, fe = forward(path)
        bb, ws, bl, be = backward(fb)
        m = {"fwd_launches": fl, "bwd_launches": bl, "fwd_device_error": fe, "bwd_device_error": be,
             "guards_intact": all(g.guard_ok() for g in list(fb.values()) + list(bb.values()) + list(ops.values()) + [ws])}
        if B == 0:
            res["paths"][path] = m
            continue
        m.update(_gru_judge(fb, bb, ws, xv, h0v, L, act, Wih, Whh, bih, bhh, dout, accurate, B, S, D, Hd, ref))
        del ws, bb
        fb2, _, _ = forward(path)
        m["fwd_deterministic"] = all(_bits_equal(fb[k].body, fb2[k].body) for k in fb)
        del fb2
        res["paths"][path] = m
        saved[path] = fb
    if len(saved) == 2:
        a_, b_ = saved.values()
        res["paths_bit_identical"] = {k: _bits_equal(a_[k].body, b_[k].body) for k in a_}
    return res


def gru_reference(x, h0, L, w_ih, w_hh, b_ih, b_hh, dout, contract=None):
    """The GRU in the inputs' dtype from x (B, S, D), forward and backward.  contract None: exact.  "bf16": x and every h rounded
    to bf16 as GEMM operands, dgi and dgh stored in bf16 (oracle.BF16).  "hilo": the same, but x enters the input projection as a
    hi/lo pair (taken as exact, oracle.BF16_FUSED) while the weight gradient reads the bf16 x rows, the only plane the kernels
    keep for the backward.  Returns out (B, Hd), dx (B, S, D), dh0, dWih (3Hd, D+1), dWhh (3Hd, Hd+1) (last column: the bias)."""
    B, S, D = x.shape
    rnd = (lambda t: t) if contract is None else _bf16_round
    xS = x.transpose(0, 1)
    gi = gru_proj((rnd(xS) if contract == "bf16" else xS).reshape(S * B, D), w_ih, b_ih)[0].view(S, B, -1)
    hs, gh, hop = [h0], [], []
    for t in range(S):
        hop.append(rnd(hs[t]))
        gh.append(gru_proj(hop[t], w_hh, b_hh)[0])
        hs.append(gru_step(gi[t], gh[t], hs[t], t < L))
    one = torch.ones(S, B, 1, dtype=x.dtype, device=x.device)
    ch = gru_bwd_chain(gi, torch.stack(gh), torch.stack(hs), L, w_ih, w_hh, torch.cat([rnd(xS), one], 2), torch.cat([torch.stack(hop), one], 2),
                       dout, contract=contract is not None)
    return dict(out=hs[S], dx=ch["dx"].transpose(0, 1), dh0=ch["dh0"], dWih=ch["dWih"], dWhh=ch["dWhh"])


def _gru_end_to_end_refs(xv, L, h0v, Wih, Whh, bih, bhh, dout, accurate):
    """The exact fp64 GRU and the bf16 storage contract of the mode, on the device (gru_reference)."""
    args = [t.double() for t in (xv, h0v)] + [L] + [t.double() for t in (Wih, Whh, bih, bhh, dout)]
    return {"exact": gru_reference(*args), "contract": gru_reference(*args, contract="hilo" if accurate else "bf16")}


def _gru_judge(fb, bb, ws, xv, h0v, L, act, Wih, Whh, bih, bhh, dout, accurate, B, S, D, Hd, ref):
    from newsrec_b200.ops_gru import ru4
    ldd, ldh, ldg, ldb = ru8(D + 1), ru8(Hd + 1), ru4(3 * Hd), ru8(3 * Hd + 1)
    H3, R = 3 * Hd, B * S
    m = {}
    i16 = lambda t: t.contiguous().view(torch.int16)
    # ---- the operand rows: bit exact
    exp_x = torch.zeros(B, S, ldd, device=DEV)
    exp_x[..., :D] = xv
    exp_x[..., D] = 1.0
    xb = fb["xb"].body.view(B, S, ldd)
    m["xb_mismatch_rows"] = int((i16(xb) != i16(exp_x.to(torch.bfloat16))).any(-1).sum())
    if accurate:
        exp_lo = torch.zeros(B, S, ldd, device=DEV)
        exp_lo[..., :D] = xv - bf16r(xv)
        m["xlo_mismatch_rows"] = int((i16(fb["xlo"].body.view(B, S, ldd)) != i16(exp_lo.to(torch.bfloat16))).any(-1).sum())
    hs = fb["hs"].body.view(S + 1, B, Hd)
    hb = fb["hb"].body.view(S + 1, B, ldh)
    exp_hb = torch.zeros(S + 1, B, ldh, device=DEV)
    exp_hb[..., :Hd] = hs
    exp_hb[..., Hd] = 1.0
    m["hs0_exact"] = _bits_equal(hs[0], h0v)
    m["hb_mismatch_rows"] = int((i16(hb) != i16(exp_hb.to(torch.bfloat16))).any(-1).sum())  # hb[0] and every hb[t+1]
    m["out_equals_hs_S"] = _bits_equal(fb["out"].body.view(B, Hd), hs[S])
    m["fwd_outputs_finite"] = all(bool(torch.isfinite(t.float()).all()) for t in (
        xb, fb["gi"].body.view(R, ldg)[:, :H3], fb["gh"].body.view(S, B, ldg)[..., :H3], hs, hb, fb["out"].body))
    # ---- gi and every gh[t]: fp64 product of the stored bf16 operands plus the bias, within 1e-6 sum |x||w|
    W1, W2 = Wih.double(), Whh.double()
    gi = fb["gi"].body.view(B, S, ldg).transpose(0, 1)[..., :H3].double()  # (S, B, 3Hd)
    gh = fb["gh"].body.view(S, B, ldg)[..., :H3].double()
    xbS = xb.transpose(0, 1)[..., :D].double()
    xloS = fb["xlo"].body.view(B, S, ldd).transpose(0, 1)[..., :D].double() if accurate else None
    acc = {k: 0.0 for k in ("gi_ratio", "gi_no_lo_ratio", "gh_ratio", "hs_ratio", "hs_bhn_outside_r_ratio", "dg_ratio",
                            "dgh_n_without_r_ratio", "dx_ratio", "dh0_ratio", "max_preact")}
    worst = lambda k, t: acc.__setitem__(k, max(acc[k], _worst(t)))
    frozen_ok = True
    for t in range(S):
        g_ref, g_abs = gru_proj(xbS[t], W1, bih.double())
        if accurate:
            lo_ref, lo_abs = gru_proj(xloS[t], W1, torch.zeros_like(bih, dtype=torch.float64))
            worst("gi_no_lo_ratio", _safe_div((gi[t] - g_ref).abs(), 1e-6 * (g_abs + lo_abs)))
            g_ref, g_abs = g_ref + lo_ref, g_abs + lo_abs
        worst("gi_ratio", _safe_div((gi[t] - g_ref).abs(), 1e-6 * g_abs))
        h_ref, h_abs = gru_proj(hb[t, :, :Hd].double(), W2, bhh.double())
        worst("gh_ratio", _safe_div((gh[t] - h_ref).abs(), 1e-6 * h_abs))
        # hs[t+1]: active rows within the gate bound, frozen rows bit-identical to hs[t]
        h_t = hs[t].double()
        g = gru_gates(gi[t], gh[t], Hd)
        Er, Ez, En = gru_gate_errors(g, gh[t, :, 2 * Hd:])
        r, z, n = g["r"], g["z"], g["n"]
        hn = (1 - z) * n + z * h_t
        bound = (h_t - n).abs() * Ez + (1 - z) * En + 3 * _U * ((1 - z) * n.abs() + z * h_t.abs())
        a_t = act[t]
        worst("max_preact", torch.cat([g["a_r"], g["a_z"], g["v"]], 1).abs()[a_t])
        worst("hs_ratio", _safe_div((hs[t + 1].double() - hn).abs(), bound)[a_t])
        bhn = bhh.double()[2 * Hd:]
        n_cudnn = torch.tanh(gi[t, :, 2 * Hd:] + r * (gh[t, :, 2 * Hd:] - bhn) + bhn)  # b_hn outside r
        worst("hs_bhn_outside_r_ratio", _safe_div((hs[t + 1].double() - ((1 - z) * n_cudnn + z * h_t)).abs(), bound)[a_t])
        frozen_ok &= _bits_equal(hs[t + 1][~a_t], hs[t][~a_t])
    m["hs_frozen_rows_exact"] = frozen_ok
    # ---- backward: the workspace as the kernels left it
    lay, total = gru_bwd_workspace_layout(B, S, Hd)
    m["workspace_bytes_match"] = total == ws.n
    wsb = ws.body
    dgi_k = wsb[lay["dgi"]:lay["dgi"] + R * ldb * 2].view(torch.bfloat16).view(B, S, ldb)
    dgh_k = wsb[lay["dgh"]:lay["dgh"] + R * ldb * 2].view(torch.bfloat16).view(S, B, ldb)
    P = (Hd + 3) // 4 * 4
    dh_dir = wsb[lay["dh_direct"]:lay["dh_direct"] + B * P * 4].view(torch.float32).view(B, P)[:, :Hd]
    dh_rec = wsb[lay["dh_rec"]:lay["dh_rec"] + B * P * 4].view(torch.float32).view(B, P)[:, :Hd]
    m["dg_pad_cols_zero"] = bool((i16(dgi_k[..., H3:]) == 0).all()) and bool((i16(dgh_k[..., H3:]) == 0).all())
    dgiS = dgi_k.transpose(0, 1)[..., :H3].double()
    dghS = dgh_k[..., :H3].double()
    ones = torch.ones(S, B, 1, dtype=torch.float64, device=DEV)
    x_ext = torch.cat([xbS, ones], 2)
    h_ext = torch.cat([hb[:S, :, :Hd].double(), ones], 2)
    ch = gru_bwd_chain(gi, gh, hs.double(), L, W1, W2, x_ext, h_ext, dout.double(), dgh_stored=dghS)
    A = torch.zeros(B, Hd, dtype=torch.float64, device=DEV)  # bound on |dh_kernel - dh_reference| entering step t
    dh_is_dout, dg_frozen_ok = True, True
    for t in range(S - 1, -1, -1):
        a_t = act[t].view(-1, 1)
        g = gru_gates(gi[t], gh[t], Hd)
        Er, Ez, En = gru_gate_errors(g, gh[t, :, 2 * Hd:])
        r, z, n = g["r"], g["z"], g["n"]
        ghn = gh[t, :, 2 * Hd:]
        dh = ch["dh"][t]
        last = (L - 1 == t) & (L < S)
        dh_is_dout &= bool((dh[last] == dout.double()[last]).all())
        hp = hs[t].double()
        dn, dz = dh * (1 - z), dh * (hp - n)
        dpn, dpz = dn * (1 - n * n), dz * z * (1 - z)
        dpr = dpn * ghn * r * (1 - r)
        E_dn = (1 - z) * A + dh.abs() * Ez + 2 * _U * dn.abs()
        E_dpn = (1 - n * n) * E_dn + dn.abs() * 2 * n.abs() * En + 3 * _U * dpn.abs() + _TINY
        E_dz = (hp - n).abs() * A + dh.abs() * En + 2 * _U * dz.abs()
        E_dpz = z * (1 - z) * E_dz + dz.abs() * (1 - 2 * z).abs() * Ez + 3 * _U * dpz.abs() + _TINY
        E_dpr = (ghn * r * (1 - r)).abs() * E_dpn + (dpn * ghn).abs() * (1 - 2 * r).abs() * Er + 4 * _U * dpr.abs() + _TINY
        E_dghn = r * E_dpn + dpn.abs() * Er + _U * (dpn * r).abs() + _TINY
        ref_gi = torch.cat([dpr, dpz, dpn], 1)
        ref_gh = torch.cat([dpr, dpz, dpn * r], 1)
        e_gi = torch.cat([E_dpr, E_dpz, E_dpn], 1)
        e_gh = torch.cat([E_dpr, E_dpz, E_dghn], 1)
        half_ulp = lambda k, rf: _bf16_ulp(torch.maximum(k.abs(), rf.abs())) / 2
        for k, rf, e in ((dgiS[t], ref_gi, e_gi), (dghS[t], ref_gh, e_gh)):
            worst("dg_ratio", _safe_div((k - rf).abs(), half_ulp(k, rf) + e)[a_t.view(-1)])
        kn = dghS[t, :, 2 * Hd:]
        worst("dgh_n_without_r_ratio", _safe_div((kn - dpn).abs(), half_ulp(kn, dpn) + E_dghn)[a_t.view(-1)])
        dg_frozen_ok &= bool((i16(dgi_k[:, t, :H3])[~act[t]] == 0).all()) and bool((i16(dgh_k[t, :, :H3])[~act[t]] == 0).all())
        # the dh entering step t - 1: dh z (fp32) + dgh[t] W_hh (fp32 GEMM, 1e-6 sum |dgh||w|), then one fp32 sum
        nxt = ch["dh"][t - 1] if t > 0 else ch["dh0"]
        G = 1e-6 * (dghS[t].abs() @ W2.abs())
        A = torch.where(a_t, z * A + dh.abs() * Ez + _U * (dh * z).abs() + G + _U * nxt.abs(), A)
    m["dg_frozen_zero"] = dg_frozen_ok
    m["dh_at_last_active_step_is_dout"] = dh_is_dout
    dh0_k = bb["dh0"].body.view(B, Hd)
    ftz = lambda t_: torch.where(t_.abs() < 2.0 ** -126, torch.zeros_like(t_), t_)  # the kernels flush fp32 subnormals
    m["dh0_equals_workspace_sum"] = _bits_equal(ftz(dh0_k), ftz(ftz(dh_dir) + ftz(dh_rec)))
    worst("dh0_ratio", _safe_div((dh0_k.double() - ch["dh0"]).abs(), A + _TINY))
    # ---- dx from the stored dgi: 1e-6 sum |dgi||w|, exactly 0 on frozen steps
    dx_k = bb["dx"].body.view(B, S, D).transpose(0, 1)
    for t in range(S):
        worst("dx_ratio", _safe_div((dx_k[t].double() - dgiS[t] @ W1).abs(), 1e-6 * (dgiS[t].abs() @ W1.abs()) + _TINY))
    m["dx_frozen_zero"] = bool((dx_k[~act] == 0).all())
    m["bwd_outputs_finite"] = bool(torch.isfinite(bb["dx"].body).all()) and bool(torch.isfinite(dh0_k).all())
    # ---- the weight gradients: pattern + dg^T [X | 1] from the stored operands, per element, against the split-K allowance
    steps = 5 * ((R + 63) // 64) + 1
    for key, dg, Xe, w in (("dWih", dgiS, x_ext, ldd), ("dWhh", dghS, h_ext, ldh)):
        K1 = Xe.shape[-1]
        pre = bb[key].prefill.double().view(H3, w)
        got = bb[key].body.view(H3, w)
        flat = lambda t_: t_.reshape(R, -1)
        rf = pre[:, :K1] + flat(dg).t() @ flat(Xe)
        ab = pre[:, :K1].abs() + flat(dg).abs().t() @ flat(Xe).abs()
        m[key + "_elem_ratio"] = _worst(_safe_div((got[:, :K1].double() - rf).abs(), 2.0 ** -22 * steps * ab + _TINY))
        cols = torch.zeros(H3, w, dtype=torch.bool, device=DEV)
        cols[:, K1:] = True
        m[key + "_pitch_cols_untouched"] = bb[key].unchanged(cols)
    m.update(acc)
    # ---- end to end: each row against the exact fp64 GRU, next to the bf16 contract's error (the project's gradient rule)
    if ref is not None:
        ex, co = ref["exact"], ref["contract"]
        kern = dict(out=fb["out"].body.view(B, Hd).double(), dx=bb["dx"].body.view(R, D).double(), dh0=dh0_k.double(),
                    dWih=(bb["dWih"].body.double() - bb["dWih"].prefill.double()).view(H3, ldd)[:, :D + 1],
                    dWhh=(bb["dWhh"].body.double() - bb["dWhh"].prefill.double()).view(H3, ldh)[:, :Hd + 1])
        for k, v in kern.items():
            e_, c_ = ex[k].reshape(v.shape), co[k].reshape(v.shape)
            m[k + "_tensor_rel_vs_contract"] = relerr(v, c_)
            # rows whose exact norm is below fp32's normal range (a gradient that decays over hundreds of steps) cannot be
            # held to a relative rule: the kernels flush subnormals to zero
            keep = e_.norm(dim=1) > 2.0 ** -100
            m[k + "_rows_below_fp32_range"] = int((~keep).sum())
            m[k + "_row_ratio"], m[k + "_ek"], m[k + "_ec"] = _row_ratio(v[keep], e_[keep], c_[keep])
    return m


def check_gru_autograd(B=37, S=50, D=900, Hd=900, accurate=True, seed=3):
    """GruLastHiddenFn (the model's entry: operand cache, dW_ext split into weight and bias gradients) end to end: each row of
    the output and of every gradient against the exact fp64 GRU next to the bf16 contract's error."""
    from newsrec_b200.ops import OperandCache
    from newsrec_b200.ops_gru import GruLastHiddenFn
    a_w = 1.0 / math.sqrt(Hd)
    Wih, Whh = _rand_bf16((3 * Hd, D), seed, a_w).to(DEV), _rand_bf16((3 * Hd, Hd), seed + 1, a_w).to(DEV)
    bih = O.det_uniform((3 * Hd,), seed + 2, -a_w, a_w).to(DEV)
    bhh = O.det_uniform((3 * Hd,), seed + 3, -a_w, a_w).to(DEV)
    xv = O.det_uniform((B, S, D), seed + 4).to(DEV)
    h0v = O.det_uniform((B, Hd), seed + 5, -0.5, 0.5).to(DEV)
    lens = gru_lengths(B, S, seed + 6).to(DEV)
    dout = O.det_uniform((B, Hd), seed + 7).to(DEV)
    ref = _gru_end_to_end_refs(xv, lens.clamp(min=1), h0v, Wih, Whh, bih, bhh, dout, accurate)
    leaves = [t.clone().requires_grad_(True) for t in (xv, h0v, Wih, Whh, bih, bhh)]
    x, h0, wi, wh, bi, bh = leaves
    out = GruLastHiddenFn.apply(x, lens, h0, wi, wh, bi, bh, OperandCache(), "gru", accurate)
    out.backward(dout)
    torch.cuda.synchronize()
    res = {}
    ex, co = ref["exact"], ref["contract"]
    kern = dict(out=out.detach().double(), dx=x.grad.double().reshape(B * S, D), dh0=h0.grad.double(),
                dWih=torch.cat([wi.grad, bi.grad.view(-1, 1)], 1).double(), dWhh=torch.cat([wh.grad, bh.grad.view(-1, 1)], 1).double())
    for k, v in kern.items():
        res[k + "_row_ratio"], res[k + "_ek"], res[k + "_ec"] = _row_ratio(v, ex[k].reshape(v.shape), co[k].reshape(v.shape))
    return res
