"""The additive-attention backward (nr_additive_attention_bwd) judged stage by stage, element by element, against fp64 at every
plan its kernels take (tests/gemm_cases.py POOL_BWD_CASES, regimes checked on the CPU by tests/test_gemm_plan_host.py).

The softmax weights w come from the real producer, nr_additive_attention_fwd (or _hilo) on the same operands.  The backward
then runs with a NaN-filled workspace and dX, a known non-zero pre-fill in the "+=" outputs dWa_ext and dqv, and guard bands
behind every output.  Each stage is judged from the kernel's own output of the previous stage, read back from the workspace,
so that one stage's rounding does not widen the next stage's bound:
  dscore  w_r (dw_r - sum_t w_t dw_t), dw_r = X_r . dout_seg (bf16 X, fp32 dout): fp32 dot products of D terms, a weighted sum
          over the segment and one product
  dPre    dscore_r qv_c (1 - t_rc^2), t = tanh(X Wa^T + ba) in fp64: the GEMM bound on pre, tanh.approx.f32's relative error
          (TANH_REL), the products, then half a bf16 ulp; the columns [q, round_up(q, 16)) are exact zeros
  dqv     pre-fill + sum_r dscore_r t_rc: the tanh error of each term plus the fp32 sums (warp butterfly, shared and global
          atomics)
  dX      dPre . Wa + w_r dout_seg: the GEMM bound 4u (ceil(q/16) + 2) sum |products| (as gpu_checks.gemm_elem_ratio), plus
          half a bf16 ulp
  dWa_ext pre-fill + dPre^T . [X | 1] over D + 1 columns (the ones column gives d(bias)): the same bound over the rows, with
          gemm_tn's k-ranges
Every bound also allows for flush-to-zero (the library is built with fast math): results and inputs below 2^-126 may be 0.
The ratios reported are the share of the relative allowance used beyond that, <= 1 exactly when every element is inside.
Around the values: NaN in X's columns (D + 1, ldx), Wa's [D, ldw), WaT's [q, ldwT) and dout's [D, ldo) never reaches a result
(the dX GEMM reads WaT through a tensor map of q columns, so its pitch columns are never loaded); dX's pitch columns, dWa_ext's
columns past D and every guard band keep their pre-fill.  dscore, dPre and dX are written once per element with no atomics:
a second run gives the same bits.  dqv (EpiDPre's per-CTA atomicAdd) and dWa_ext (gemm_tn's k-ranges added with red.add) are
sums in run-dependent order: they are judged by the bound only.

Also here: AdditiveAttentionFn's gradients against the ABI on the same operands in both precision modes, the refusal of bad
shapes before any launch, and the two small ABI entries of the same gradient chain, nr_dot_score_bwd and nr_accumulate_ext_grad."""
import pytest
import torch

import gemm_cases as C
import gemm_plan_ref as P
import gpu_checks as G

pytestmark = pytest.mark.gpu

DEV = "cuda"
NAN = float("nan")
# PTX ISA, "tanh": tanh.approx.f32 implements an approximation with a maximum relative error of 2^-10.987 (subnormal results
# flush to zero)
TANH_REL = 2.0 ** -10.987
TINY = 2.0 ** -126


def _cdiv(a, b):
    return -(-a // b)


def _inputs(c, seed=5):
    """fp32 rows x [rows][D], Wa [q][D] (bf16 values), ba, qv [q] in the case's score regime, dout [n_seg][D]."""
    n_seg, seg, D, q = c["n_seg"], c["seg"], c["D"], c["q"]
    rows = n_seg * seg
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((rows, D), generator=g) * 2 - 1
    wa = (torch.rand((q, D), generator=g) * 2 - 1) * (3.0 / D) ** 0.5
    ba = (torch.rand((q,), generator=g) - 0.5) * 0.2
    qv = (torch.rand((q,), generator=g) * 2 - 1) * (3.0 / q) ** 0.5
    dout = torch.rand((n_seg, D), generator=g) * 2 - 1
    scores = c.get("scores", "unit")
    if scores == "peaked":  # column 0 drives every pre-activation into tanh saturation: score_r ~ 100 tanh(8 x_r0)
        wa[:, 1:] *= 0.1
        wa[:, 0] = 8.0
        qv = torch.full((q,), 100.0 / q)
    elif scores == "tied":  # every row of a segment equals its first: uniform weights
        x = x.view(n_seg, seg, D)[:, :1].expand(n_seg, seg, D).reshape(rows, D).clone()
    if not c.get("hilo"):
        x = x.to(torch.bfloat16).float()
    return x, wa.to(torch.bfloat16).float(), ba, qv, dout


def _pack(c, x, wa, ba, qv, dout):
    """The operands as the kernels read them, NaN in every pitch column: X (+ X_lo) bf16 [rows][ldx] with the ones column at
    D, Wa bf16 [q][ldx], WaT bf16 [D][ldwT], dout fp32 [n_seg][ldo]; w from the forward."""
    D, q, n_seg, seg = c["D"], c["q"], c["n_seg"], c["seg"]
    ldx, ldwT = G.ru8(D + 1), G.ru8(q) + 8
    ldo = c.get("ldo", (D + 3) // 4 * 4 + 4)
    X = torch.full((x.shape[0], ldx), NAN, dtype=torch.bfloat16, device=DEV)
    xd = x.to(DEV)
    X[:, :D] = xd.to(torch.bfloat16)
    X[:, D] = 1.0
    X_lo = None
    if c.get("hilo"):
        X_lo = torch.full_like(X, NAN)
        X_lo[:, :D] = (xd - X[:, :D].float()).to(torch.bfloat16)
    Wa = torch.full((q, ldx), NAN, dtype=torch.bfloat16, device=DEV)
    Wa[:, :D] = wa.to(DEV).to(torch.bfloat16)
    WaT = torch.full((D, ldwT), NAN, dtype=torch.bfloat16, device=DEV)
    WaT[:, :q] = Wa[:, :D].t()
    dO = torch.full((n_seg, ldo), NAN, dtype=torch.float32, device=DEV)
    dO[:, :D] = dout.to(DEV)
    r = dict(X=X, X_lo=X_lo, Wa=Wa, WaT=WaT, ba=ba.to(DEV), qv=qv.to(DEV), dout=dO, ldx=ldx, ldw=ldx, ldwT=ldwT, ldo=ldo)
    lib = G.load_library()
    out = torch.empty((n_seg, G.ru8(D)), device=DEV)
    w = torch.full((n_seg * seg,), NAN, device=DEV)
    if X_lo is not None:
        rc = lib.nr_additive_attention_fwd_hilo(G._p(X), G._p(X_lo), n_seg, seg, D, ldx, G._p(Wa), q, ldx, G._p(r["ba"]),
                                                G._p(r["qv"]), G._p(out), out.shape[1], G._p(w), G._stream())
    else:
        rc = lib.nr_additive_attention_fwd(G._p(X), n_seg, seg, D, ldx, G._p(Wa), q, ldx, G._p(r["ba"]), G._p(r["qv"]), G._p(out),
                                           out.shape[1], G._p(w), G._stream())
    G.check(rc, "additive_attention_fwd")
    r["w"] = w
    return r


def _prefill(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((n,), generator=g) * 2 - 1).to(DEV)


def _run_bwd(c, k, ld_dx):
    """One backward on the kernel operands k with fresh NaN / pre-filled outputs: (dX, dWa_ext, dqv, workspace)."""
    lib = G.load_library()
    n_seg, seg, D, q = c["n_seg"], c["seg"], c["D"], c["q"]
    rows = n_seg * seg
    ws_bytes = int(lib.nr_additive_attention_bwd_workspace(n_seg, seg, q))
    ws = torch.full((ws_bytes // 4,), NAN, device=DEV)
    dX = G._Guarded(rows * ld_dx, torch.bfloat16, NAN)
    dX.prefill = dX.body.clone()
    dWa = G._Guarded(q * k["ldx"], torch.float32, _prefill(q * k["ldx"], 1))
    dqv = G._Guarded(q, torch.float32, _prefill(q, 2))
    G.check(lib.nr_additive_attention_bwd(G._p(k["X"]), n_seg, seg, D, k["ldx"], G._p(k["Wa"]), G._p(k["WaT"]), q, k["ldw"], k["ldwT"],
                                          G._p(k["ba"]), G._p(k["qv"]), G._p(k["w"]), G._p(k["dout"]), k["ldo"], G._p(dX.all), ld_dx,
                                          G._p(dWa.all), G._p(dqv.all), G._p(ws), ws_bytes, G._stream()),
            "additive_attention_bwd")
    torch.cuda.synchronize()
    return dX, dWa, dqv, ws


def _workspace_views(ws, rows, q):
    """dscore fp32 [rows] at 0 and dPre bf16 [rows][round_up(q, 16)] at the next 256-byte boundary."""
    off = (4 * rows + 255) // 256 * 256
    ldq = G.ru16(q)
    return ws[:rows], ws.view(torch.bfloat16)[off // 2:off // 2 + rows * ldq].view(rows, ldq)


def _bounds(c, r, ds_k, dpre_k, sms):
    """fp64 references of every stage, from the reference operands r and the kernel's own dscore / dPre, with the relative part
    of each bound (e) and its flush-to-zero allowance (f: the library runs with flush-to-zero, so a product or a sum below 2^-126,
    and a subnormal input, may come out 0)."""
    n_seg, seg, D, q = c["n_seg"], c["seg"], c["D"], c["q"]
    rows = n_seg * seg
    X, Wa = r["X"][:, :D].double(), r["Wa"][:, :D].double()
    ba, qv, w = r["ba"].double(), r["qv"].double(), r["w"].double().view(n_seg, seg)
    dout = r["dout"][:, :D].double()
    U = G.U32
    b = {}
    # dscore: dw_r = X_r . dout_seg in fp32 (each lane's fma chain, then a warp reduction), dot = sum_t w_t dw_t, ds = w (dw - dot)
    Xv = X.view(n_seg, seg, D)
    dw = torch.einsum("nsd,nd->ns", Xv, dout)
    e_dw = 4 * U * (_cdiv(D, 8) + 16) * torch.einsum("nsd,nd->ns", Xv.abs(), dout.abs())
    b["dscore"] = ((w * (dw - (w * dw).sum(dim=1, keepdim=True))).reshape(-1),
                   (w * (e_dw + (w * e_dw).sum(dim=1, keepdim=True) + 4 * U * (seg + 4) * (dw.abs() + (w * dw.abs()).sum(dim=1, keepdim=True)))).reshape(-1),
                   (seg + 2) * TINY)
    # dPre from the kernel's dscore: t = tanh(pre) with pre off by the GEMM bound, then tanh.approx's relative error
    pre = X @ Wa.t() + ba
    e_pre = 4 * U * (_cdiv(D, 16) + 2) * (X.abs() @ Wa.abs().t() + ba.abs())
    t = torch.tanh(pre)
    e_t = e_pre + TANH_REL * (t.abs() + e_pre) + TINY
    omt = 1 - t * t
    dsq = ds_k.view(rows, 1) * qv
    b["dPre"] = (dsq * omt, dsq.abs() * (e_t * (2 * t.abs() + e_t) + 3 * U * omt), 2 * TINY)
    # dqv: two rows per lane, a 3-level butterfly, shared atomics over the CTA's tiles (4 warps each), one global atomic per CTA
    pd = P.plan_nt(rows, q, D, 1, P.kTileM, sms, P.EPI_DPRE_SMEM, max_slices=1)
    n_dqv = 8 + 4 * max(len(a) + len(b_) for a, b_ in pd["wg_tiles"]) + pd["grid"] + 2
    b["n_dqv"] = n_dqv
    b["dqv"] = ((ds_k.view(rows, 1) * t).sum(dim=0),
                (ds_k.abs().view(rows, 1) * e_t).sum(dim=0) + 4 * U * (n_dqv + 2) * (ds_k.abs().view(rows, 1) * t.abs()).sum(dim=0),
                (rows + 2) * TINY)
    # dX from the kernel's dPre: the GEMM over q (ceil(q / 16) k-steps), then the fma with w_r dout
    dout_r = dout.repeat_interleave(seg, dim=0)
    wr = w.reshape(rows, 1)
    b["dX"] = (dpre_k @ Wa + wr * dout_r, 4 * U * (_cdiv(q, 16) + 2) * (dpre_k.abs() @ Wa.abs() + (wr * dout_r).abs()),
               TINY * (Wa.abs().sum(dim=0) + dout_r.abs() + q + 2))
    # [dWa | dba] from the kernel's dPre over X's D + 1 columns: gemm_tn over the rows, k-ranges added with red.add
    Xe = r["X"][:, :D + 1].double()
    n_dwa = _cdiv(rows, 16) + max(p["k_slices_max"] for p in P.plan_pool_bwd(n_seg, seg, D, q, sms)["wgrad"])
    b["dWa"] = (dpre_k.t() @ Xe, 4 * U * (n_dwa + 2) * (dpre_k.abs().t() @ Xe.abs()), TINY * (Xe.abs().sum(dim=0) + rows + 2))
    b["n_dwa"] = n_dwa
    return b


def _ratio(got, ref, e, bf16=False, flush=0.0):
    """The worst (|got - ref| - flush allowance - half a bf16 ulp of a bf16 output) / e, clamped at 0: the share of the
    relative allowance e used, <= 1 exactly when every element is inside its bound (+inf for a NaN)."""
    err = ((got.double() - ref).abs() - flush).clamp_min(0)
    if bf16:
        err = (err - 0.5 * G._bf16_ulp(ref.abs() + e)).clamp_min(0)
    return G._worst(G._safe_div(err, e))


def judge_bwd(c, r, k=None):
    """Run the backward on the kernel operands k (default: r) and judge it against the reference operands r."""
    k = r if k is None else k
    lib = G.load_library()
    n_seg, seg, D, q = c["n_seg"], c["seg"], c["D"], c["q"]
    rows, ldx = n_seg * seg, r["ldx"]
    ld_dx = c.get("ld_dx", ldx)
    runs = [_run_bwd(c, k, ld_dx) for _ in range(2)]
    dX, dWa, dqv, ws = runs[0]
    ds_k, dpre = _workspace_views(ws, rows, q)
    dpre_k = dpre[:, :q].double()
    b = _bounds(c, r, ds_k.double(), dpre_k, lib.nr_num_sms())
    U = G.U32
    pf_q = dqv.prefill.double()
    pf_w = dWa.prefill.double().view(q, ldx)[:, :D + 1]
    got = {"dscore": ds_k, "dPre": dpre_k, "dqv": dqv.body, "dX": dX.body.view(rows, ld_dx)[:, :D], "dWa": dWa.body.view(q, ldx)[:, :D + 1]}
    ref = {s: b[s][0] for s in STAGES}
    e = {s: b[s][1] for s in STAGES}
    ref["dqv"], e["dqv"] = pf_q + ref["dqv"], e["dqv"] + 4 * U * (b["n_dqv"] + 2) * pf_q.abs()
    ref["dWa"], e["dWa"] = pf_w + ref["dWa"], e["dWa"] + 4 * U * (b["n_dwa"] + 2) * pf_w.abs()
    res = {s: _ratio(got[s], ref[s], e[s], s in ("dPre", "dX"), b[s][2]) for s in STAGES}
    res["dpre_pad_zero"] = bool((dpre[:, q:] == 0).all())
    dx_pitch = torch.zeros(rows, ld_dx, dtype=torch.bool, device=DEV)
    dx_pitch[:, D:] = True
    dwa_pitch = torch.zeros(q, ldx, dtype=torch.bool, device=DEV)
    dwa_pitch[:, D + 1:] = True
    res["pitch_untouched"] = dX.unchanged(dx_pitch) and dWa.unchanged(dwa_pitch)
    res["guards"] = all(o.guard_ok() for run in runs for o in run[:3])
    ds2, dpre2 = _workspace_views(runs[1][3], rows, q)
    res["rerun_bit_identical"] = G._bits_equal(ds_k, ds2) and G._bits_equal(dpre, dpre2) and G._bits_equal(dX.body, runs[1][0].body)
    return res


STAGES = ("dscore", "dPre", "dqv", "dX", "dWa")


@pytest.mark.parametrize("c", C.POOL_BWD_CASES, ids=lambda c: c["id"])
def test_additive_bwd_elements(c):
    r = _pack(c, *_inputs(c))
    res = judge_bwd(c, r)
    print(c["id"], res)
    assert all(res[s] <= 1 for s in STAGES), res
    assert res["dpre_pad_zero"] and res["pitch_untouched"] and res["guards"] and res["rerun_bit_identical"], res


@pytest.mark.parametrize("precision", ["fast", "accurate"])
@pytest.mark.parametrize("N,S,D,q", [(37, 20, 300, 200), (200, 4, 400, 200)])
def test_autograd_matches_the_abi(precision, N, S, D, q):
    """AdditiveAttentionFn's gradients against nr_additive_attention_bwd on the operands it builds: dX bit for bit, the atomic
    sums [dWa | dba] and dqv within twice their accumulation bound (both runs lie within one bound of the exact sum)."""
    from newsrec_b200.ops import AdditiveAttentionFn, OperandCache, cast_pad
    lib = G.load_library()
    g = torch.Generator().manual_seed(11)
    x = (torch.rand((N, S, D), generator=g) * 2 - 1).to(DEV)
    wa = ((torch.rand((q, D), generator=g) * 2 - 1) * (3.0 / D) ** 0.5).to(DEV)
    ba = ((torch.rand((q,), generator=g) - 0.5) * 0.2).to(DEV)
    qv = ((torch.rand((q,), generator=g) * 2 - 1) * (3.0 / q) ** 0.5).to(DEV)
    dout = (torch.rand((N, D), generator=g) * 2 - 1).to(DEV)
    xg = x.clone().requires_grad_(True)
    prm = [t.clone().requires_grad_(True) for t in (wa, ba, qv)]
    out = AdditiveAttentionFn.apply(xg, *prm, OperandCache(), "t", precision)
    out.backward(dout)
    rows, ldx, ldq = N * S, G.ru8(D + 1), G.ru16(q)
    Wa, WaT = cast_pad(wa, ldx), cast_pad(wa, ldq, transpose=True)
    xs = x.reshape(rows, D)
    X = torch.empty((rows, ldx), dtype=torch.bfloat16, device=DEV)
    out2 = torch.empty((N, D), device=DEV)
    w = torch.empty((rows,), device=DEV)
    if precision == "accurate":
        X_lo = torch.empty_like(X)
        G.check(lib.nr_rows_to_bf16_hilo(G._p(xs), rows, D, D, 1, G._p(X), G._p(X_lo), ldx, G._stream()), "rows_to_bf16_hilo")
        G.check(lib.nr_additive_attention_fwd_hilo(G._p(X), G._p(X_lo), N, S, D, ldx, G._p(Wa), q, ldx, G._p(ba), G._p(qv), G._p(out2), D,
                                                   G._p(w), G._stream()), "fwd_hilo")
    else:
        G.check(lib.nr_rows_to_bf16(G._p(xs), rows, D, D, 1, G._p(X), ldx, G._stream()), "rows_to_bf16")
        G.check(lib.nr_additive_attention_fwd(G._p(X), N, S, D, ldx, G._p(Wa), q, ldx, G._p(ba), G._p(qv), G._p(out2), D, G._p(w),
                                              G._stream()), "fwd")
    dX = torch.empty((rows, ldx), dtype=torch.bfloat16, device=DEV)
    dWa = torch.zeros((q, ldx), device=DEV)
    dqv = torch.zeros((q,), device=DEV)
    ws_bytes = int(lib.nr_additive_attention_bwd_workspace(N, S, q))
    ws = torch.empty((ws_bytes // 4,), device=DEV)
    G.check(lib.nr_additive_attention_bwd(G._p(X), N, S, D, ldx, G._p(Wa), G._p(WaT), q, ldx, ldq, G._p(ba), G._p(qv), G._p(w),
                                          G._p(dout), D, G._p(dX), ldx, G._p(dWa), G._p(dqv), G._p(ws), ws_bytes, G._stream()), "bwd")
    torch.cuda.synchronize()
    assert G._bits_equal(out.detach(), out2)  # the same forward, so the same saved w
    assert torch.equal(xg.grad.reshape(rows, D), dX[:, :D].float())
    ds, dpre = _workspace_views(ws, rows, q)
    dpre = dpre[:, :q].double()
    Xe = X[:, :D + 1].double()
    n_dwa = _cdiv(rows, 16) + max(p["k_slices_max"] for p in P.plan_pool_bwd(N, S, D, q, lib.nr_num_sms())["wgrad"])
    e_dwa = 4 * G.U32 * (n_dwa + 2) * (dpre.abs().t() @ Xe.abs())
    t = torch.tanh(X[:, :D].double() @ Wa[:, :D].double().t() + ba.double())
    e_dqv = 4 * G.U32 * (rows + 2) * (ds.double().abs().view(rows, 1) * t.abs()).sum(dim=0) * 2
    assert bool(((prm[0].grad.double() - dWa[:, :D].double()).abs() <= 2 * e_dwa[:, :D]).all())
    assert bool(((prm[1].grad.double() - dWa[:, D].double()).abs() <= 2 * e_dwa[:, D]).all())
    assert bool(((prm[2].grad.double() - dqv.double()).abs() <= 2 * e_dqv).all())


def test_additive_bwd_refuses_bad_shapes_before_any_launch():
    """Each bad shape returns non-zero with no launch and dX, dWa_ext and dqv bit-unchanged: seg_len 0 (no rows at all) and 65
    (w only comes from the forward, seg_len <= 64), n_seg < 0, q 0 and 257, D % 4 != 0, every pitch below its minimum or off
    its alignment, a dX GEMM that cannot be planned (seg_len 1 caps its slices at 16 columns: D = 1028 needs 65) and a small
    workspace.  n_seg = 0 is an empty problem: 0, nothing launched.  The buffers are large flat allocations, so that a library
    that launched a bad shape anyway would still stay inside them."""
    lib = G.load_library()
    cap = 1 << 16
    g = torch.Generator().manual_seed(9)
    X = (torch.rand((cap,), generator=g) - 0.5).to(torch.bfloat16).to(DEV)
    Wa = (torch.rand((cap,), generator=g) - 0.5).to(torch.bfloat16).to(DEV)
    vec = torch.rand((cap,), generator=g).to(DEV)  # ba, qv, w, dout
    dX = G._Guarded(cap, torch.bfloat16, _prefill(cap, 3))
    dWa = G._Guarded(cap, torch.float32, _prefill(cap, 4))
    dqv = G._Guarded(cap, torch.float32, _prefill(cap, 5))
    ws = torch.zeros((4 * cap,), device=DEV)
    base = dict(n_seg=4, seg=8, D=64, q=32, ldx=72, ldw=72, ldwT=32, ldo=64, ld_dx=72, ws=ws.numel() * 4)

    def call(**kw):
        a = dict(base, **kw)
        return lib.nr_additive_attention_bwd(G._p(X), a["n_seg"], a["seg"], a["D"], a["ldx"], G._p(Wa), G._p(Wa), a["q"], a["ldw"],
                                             a["ldwT"], G._p(vec), G._p(vec), G._p(vec), G._p(vec), a["ldo"], G._p(dX.all), a["ld_dx"],
                                             G._p(dWa.all), G._p(dqv.all), G._p(ws), a["ws"], G._stream())

    bad = [dict(seg=0), dict(seg=65, n_seg=1), dict(n_seg=-1), dict(q=0), dict(q=257), dict(D=62), dict(ldx=64), dict(ldx=76),
           dict(ldw=56), dict(ldw=68), dict(ldwT=24), dict(ldwT=36), dict(ldo=60), dict(ldo=66), dict(ld_dx=56), dict(ld_dx=68),
           dict(n_seg=4, seg=1, D=1028, ldx=1032, ldw=1032, ldo=1028, ld_dx=1032), dict(ws=1024)]
    failed = []
    for b in bad:
        before = [o.all.clone() for o in (dX, dWa, dqv)]
        n0 = lib.nr_launch_count()
        rc = call(**b)
        torch.cuda.synchronize()
        launched = lib.nr_launch_count() - n0
        same = all(G._bits_equal(o.all, x) for o, x in zip((dX, dWa, dqv), before))
        if rc == 0 or launched or not same:
            failed.append((b, rc, launched, same))
    assert not failed, failed
    n0 = lib.nr_launch_count()
    assert call(n_seg=0) == 0
    torch.cuda.synchronize()
    assert lib.nr_launch_count() == n0
    assert all(o.unchanged(torch.ones(cap, dtype=torch.bool, device=DEV)) and o.guard_ok() for o in (dX, dWa, dqv))


# ---- the rest of the chain: the click predictor's backward and the carry of dWa_ext into .grad --------------------------------
@pytest.mark.parametrize("B,Cn,D", [(9, 5, 300), (1, 1, 1), (64, 1, 400), (3, 50, 129)])
def test_dot_score_bwd_elements(B, Cn, D):
    """dcand[b][j] = g[b][j] user[b] (one product: exact up to one rounding) and duser[b] = sum_j g[b][j] cand[b][j] (an fp32 fma
    chain of Cn terms), both overwriting NaN-filled outputs with guard bands."""
    lib = G.load_library()
    g = torch.Generator().manual_seed(B * 1000 + Cn)
    cand = (torch.rand((B, Cn, D), generator=g) * 2 - 1).to(DEV)
    user = (torch.rand((B, D), generator=g) * 2 - 1).to(DEV)
    dl = (torch.rand((B, Cn), generator=g) * 2 - 1).to(DEV)
    dcand = G._Guarded(B * Cn * D, torch.float32, NAN)
    duser = G._Guarded(B * D, torch.float32, NAN)
    G.check(lib.nr_dot_score_bwd(G._p(cand), G._p(user), G._p(dl), B, Cn, D, G._p(dcand.all), G._p(duser.all), G._stream()), "dot_bwd")
    torch.cuda.synchronize()
    c64, u64, g64 = cand.double(), user.double(), dl.double()
    ref_c = g64[:, :, None] * u64[:, None, :]
    ref_u = torch.einsum("bj,bjd->bd", g64, c64)
    e_u = 4 * G.U32 * (Cn + 2) * torch.einsum("bj,bjd->bd", g64.abs(), c64.abs()) + TINY
    r_c = _ratio(dcand.body.view(B, Cn, D), ref_c, G.U32 * ref_c.abs() + TINY)
    r_u = _ratio(duser.body.view(B, D), ref_u, e_u)
    assert r_c <= 1 and r_u <= 1 and dcand.guard_ok() and duser.guard_ok(), (r_c, r_u)


@pytest.mark.parametrize("rows,D,ld,with_db", [(200, 300, 304, True), (200, 300, 301, True), (7, 1, 8, False), (300, 400, 416, False)])
def test_accumulate_ext_grad(rows, D, ld, with_db):
    """dW += ext[:, :D] and db += ext[:, D] (one fp32 add each: exact up to one rounding); db may be null, and then column D is
    cleared but added nowhere; ext is cleared over [rows][D + 1] and its pitch columns (D, ld) keep their bits."""
    lib = G.load_library()
    ext = G._Guarded(rows * ld, torch.float32, _prefill(rows * ld, 6))
    if ld > D + 1:  # pitch columns hold NaN: the kernel must neither read them into a result nor clear them
        ext.all[:rows * ld].view(rows, ld)[:, D + 1:] = NAN
        ext.prefill = ext.body.clone()
    dW = G._Guarded(rows * D, torch.float32, _prefill(rows * D, 7))
    db = G._Guarded(rows, torch.float32, _prefill(rows, 8)) if with_db else None
    G.check(lib.nr_accumulate_ext_grad(G._p(ext.all), rows, ld, D, G._p(dW.all), G._p(db.all) if db is not None else None, G._stream()),
            "accumulate_ext_grad")
    torch.cuda.synchronize()
    e = ext.prefill.double().view(rows, ld)
    ref_w = dW.prefill.double().view(rows, D) + e[:, :D]
    assert _ratio(dW.body.view(rows, D), ref_w, G.U32 * ref_w.abs() + TINY) <= 1 and dW.guard_ok()
    if db is not None:
        ref_b = db.prefill.double() + e[:, D]
        assert _ratio(db.body, ref_b, G.U32 * ref_b.abs() + TINY) <= 1 and db.guard_ok()
    body = ext.body.view(rows, ld)
    assert bool((body[:, :D + 1] == 0).all())
    pitch = torch.zeros(rows, ld, dtype=torch.bool, device=DEV)
    pitch[:, D + 1:] = True
    assert ext.unchanged(pitch) and ext.guard_ok()
