"""Helpers of the CNN text encoder tests at window_size 1 to 4: the window golden cases (oracle/make_golden_cnn_window.py)
and nr_cnn_encoder_fwd / _bwd stage by stage against fp64 at any window.

A window golden case is a family's case at another conv window: the oracle, the drop-in and the state_dict are the family's,
with the conv weights (F, 1, w, d).  With p = (w - 1) // 2 a title of T tokens has L = T + 2p - w + 1 conv outputs."""
import ctypes as C
import math

import torch

import golden_util as GU
import hifiark_oracle as HO
import newsrec_oracle as O

# case -> (family case, window_size); the fixtures record their window (window_size)
WINDOW_CASES = {"naml_w4": ("naml", 4), "tanr_w1": ("tanr", 1), "lstur_ini_w2": ("lstur_ini", 2), "hifiark_w2": ("hifiark", 2)}
FAMILY_MODEL = {"naml": "NAML", "tanr": "TANR", "lstur_ini": "LSTUR", "hifiark": "HiFiArk"}


def out_len(T, w):
    """Conv outputs of a T-token title at window w (the reference's padding (w - 1) // 2)."""
    return T + 2 * ((w - 1) // 2) - w + 1


def case_shapes(case):
    family, w = WINDOW_CASES[case]
    if family == "naml":
        return O.naml_shapes(GU.V, GU.NCAT, window=w)
    if family == "tanr":
        return O.tanr_shapes(GU.V, GU.NCAT, window=w)
    if family == "hifiark":
        return HO.hifiark_shapes(GU.V, window=w)
    return O.lstur_shapes(GU.V, GU.NCAT, GU.NUSERS, window=w, method=family.split("_")[1])


def state_dict(case, g):
    """The recipe's deterministic state_dict of a window case."""
    if WINDOW_CASES[case][0] == "hifiark":
        return O.det_state_dict(case_shapes(case), int(g["seed"]), {"omap.W": 0.1})
    return O.tie_shared(O.det_state_dict(case_shapes(case), int(g["seed"])))


def case_params(case, g, dtype=torch.float32, requires_grad=True):
    """golden_util.case_params of a window case: tied storage stays one leaf tensor."""
    out, seen = {}, {}
    for k, v in state_dict(case, g).items():
        if id(v) in seen:
            out[k] = out[seen[id(v)]]
            continue
        seen[id(v)] = k
        out[k] = v.to(dtype).clone().requires_grad_(requires_grad)
    return out


def oracle_forward(case, g, p, contract=O.EXACT, fused=False):
    """golden_util.oracle_forward of the family (NAML, TANR, LSTUR): the window comes with the conv weights."""
    return GU.oracle_forward(WINDOW_CASES[case][0], g, p, contract, fused)


def build_model(case, dev, dropout=0.2, fused=False):
    """The drop-in of a window case at the golden shapes (gpu_checks.build_model with the case's window_size)."""
    import importlib

    import config as cfgmod
    family, w = WINDOW_CASES[case]
    name = FAMILY_MODEL[family]
    over = dict(num_words=GU.V, num_categories=GU.NCAT, num_users=GU.NUSERS, num_clicked_news_a_user=6, dropout_probability=dropout,
                window_size=w)
    if name == "LSTUR":
        over.update(precision="accurate" if fused else "fast", long_short_term_method=family.split("_")[1])
    cfg = type("Cfg", (getattr(cfgmod, name + "Config"),), over)
    return getattr(importlib.import_module("model." + name), name)(cfg).to(dev)


# ---- nr_cnn_encoder_fwd / _bwd at window w, stage by stage against fp64 ---------------------------------------------------
def cnn_operands(n_seq, T, d, F, q, V, window, seed, bad_ids=True):
    """Device operands of the encoder at `window`, built the way CnnPoolEncoderFn.build does (tap-major conv rows, the
    transposed taps in reverse order for the embedding gradient)."""
    import gpu_checks as G
    from newsrec_b200.ops import cast_pad, ru8, ru16
    dev = G.DEV
    ldx, ldf, ldq = ru8(d + 1), ru8(F + 1), ru16(q)
    a_w = 0.5 * math.sqrt(3.0 / (d * window / 3.0))  # pre-activation std ~0.5 at every window: both signs reach the ReLU
    Wc = G._rand_bf16((F, window, d), seed + 1, a_w).to(dev)
    bc = O.det_uniform((F,), seed + 2, -0.05, 0.05).to(dev)
    Wa = G._rand_bf16((q, F), seed + 3, math.sqrt(3.0 / F)).to(dev)
    ba = O.det_uniform((q,), seed + 4, -0.1, 0.1).to(dev)
    qv = O.det_uniform((q,), seed + 5, -1.0, 1.0).to(dev)
    table_f = G._rand_bf16((V, d), seed + 6).to(dev)
    return dict(n_seq=n_seq, T=T, d=d, F=F, q=q, V=V, window=window, ldx=ldx, ldf=ldf, ldq=ldq, Wc=Wc, bc=bc, Wa=Wa, ba=ba, qv=qv,
                table_f=table_f, wconv=cast_pad(Wc.permute(1, 0, 2).reshape(window * F, d), ldx),
                wconvT=cast_pad(torch.cat([Wc[:, window - 1 - s, :].t() for s in range(window)], 0), ldf),
                wa=cast_pad(Wa, ldf), waT=cast_pad(Wa, ldq, transpose=True), table=cast_pad(table_f, ldx),
                ids=G._cnn_ids(n_seq, T, V, seed + 7, bad_ids), dout=O.det_uniform((max(n_seq, 1), F), seed + 8).to(dev),
                kseed=(0x9E3779B97F4A7C15 * (seed + 11)) & 0xFFFFFFFFFFFFFFFF, seed=seed)


def run_cnn(o, p_drop, accurate, window_field):
    """One forward and one backward through the C ABI with args.window = window_field (0: the default, 3).  Every "=" output,
    Y, w and the workspace start as NaN, every "+=" output at a small non-zero pre-fill, each followed by a guard band.
    Returns (forward buffers, backward buffers, launches of each)."""
    import gpu_checks as G
    from newsrec_b200 import CnnEncoderBwdArgs, CnnEncoderFwdArgs, check, load_library
    from newsrec_b200.ops import _p, _stream
    lib = load_library()
    n_seq, T, d, F, q, V, w = o["n_seq"], o["T"], o["d"], o["F"], o["q"], o["V"], o["window"]
    ldx, ldf, ldq, seed = o["ldx"], o["ldf"], o["ldq"], o["seed"]
    n_out, Mp = n_seq * out_len(T, w), n_seq * (T + 2)
    nan = float("nan")
    fb = dict(Xp=G._Guarded(Mp * ldx, torch.bfloat16, nan), Y=G._Guarded(n_out * ldf, torch.bfloat16, nan),
              w=G._Guarded(n_out, torch.float32, nan), out=G._Guarded(n_seq * F, torch.float32, nan),
              flag=G._Guarded(1, torch.int32, 0, sentinel=-7))
    if accurate:
        fb["Ylo"] = G._Guarded(n_out * ldf, torch.bfloat16, nan)
    a = CnnEncoderFwdArgs()
    a.n_seq, a.T, a.d, a.F, a.q, a.ldx, a.ldf, a.window = n_seq, T, d, F, q, ldx, ldf, window_field
    a.ids, a.table_bf16, a.V = _p(o["ids"]), _p(o["table"]), V
    a.wconv_bf16, a.bconv, a.wa_bf16, a.ba, a.qv = _p(o["wconv"]), _p(o["bc"]), _p(o["wa"]), _p(o["ba"]), _p(o["qv"])
    a.p_drop, a.seed = float(p_drop), o["kseed"]
    a.Xp_bf16, a.Y_bf16, a.w, a.out, a.bad_id_flag = _p(fb["Xp"].all), _p(fb["Y"].all), _p(fb["w"].all), _p(fb["out"].all), _p(fb["flag"].all)
    if accurate:
        a.Y_lo_bf16 = _p(fb["Ylo"].all)
    n0 = int(lib.nr_launch_count())
    check(lib.nr_cnn_encoder_fwd(C.byref(a), _stream()), "nr_cnn_encoder_fwd")
    fwd_launches = int(lib.nr_launch_count()) - n0
    pat = lambda n, s: O.det_uniform((n,), s, 0.5, 1.0).to(G.DEV) * 2.0 ** -16
    bb = dict(dWc=G._Guarded(w * F * ldx, torch.float32, pat(w * F * ldx, seed + 20)),
              dWa=G._Guarded(q * ldf, torch.float32, pat(q * ldf, seed + 21)),
              dqv=G._Guarded(q, torch.float32, pat(q, seed + 22)), demb=G._Guarded(V * d, torch.float32, pat(V * d, seed + 23)))
    ws_bytes = int(lib.nr_cnn_encoder_bwd_workspace(n_seq, T, F, q))
    bb["ws"] = G._Guarded(ws_bytes, torch.uint8, 0xFF, sentinel=0xA5)  # 0xFFFF.. is NaN in bf16 and fp32
    b = CnnEncoderBwdArgs()
    b.n_seq, b.T, b.d, b.F, b.q, b.ldx, b.ldf, b.ldq, b.window = n_seq, T, d, F, q, ldx, ldf, ldq, window_field
    b.ids, b.V = _p(o["ids"]), V
    b.wconvT_bf16, b.wa_bf16, b.waT_bf16, b.ba, b.qv = _p(o["wconvT"]), _p(o["wa"]), _p(o["waT"]), _p(o["ba"]), _p(o["qv"])
    b.p_drop, b.seed = float(p_drop), o["kseed"]
    b.Xp_bf16, b.Y_bf16, b.w, b.dout = _p(fb["Xp"].all), _p(fb["Y"].all), _p(fb["w"].all), _p(o["dout"])
    b.dWconv_ext, b.dWa_ext, b.dqv, b.demb = _p(bb["dWc"].all), _p(bb["dWa"].all), _p(bb["dqv"].all), _p(bb["demb"].all)
    b.workspace, b.workspace_bytes = _p(bb["ws"].all), ws_bytes
    n0 = int(lib.nr_launch_count())
    check(lib.nr_cnn_encoder_bwd(C.byref(b), _stream()), "nr_cnn_encoder_bwd")
    bwd_launches = int(lib.nr_launch_count()) - n0
    torch.cuda.synchronize()
    return fb, bb, fwd_launches, bwd_launches


def check_cnn_window(n_seq, T, window, d=300, F=400, q=200, V=3000, p_drop=0.2, accurate=False, seed=1, bad_ids=True,
                     grad_floor=2e-3):
    """gpu_checks.check_cnn_encoder at window w: the fp64 references are built from the kernels' own stored Xp, Y, w; the conv
    output j of a title reads padded rows j + 1 - p + s (s < w), dW_s = dY^T . X[rows + s - p] with the bias gradient in column
    d of tap p, and the embedding gradient is the transposed conv over the same padded dY."""
    import gpu_checks as G
    dev = G.DEV
    o = cnn_operands(n_seq, T, d, F, q, V, window, seed, bad_ids)
    fb, bb, fwd_launches, bwd_launches = run_cnn(o, p_drop, accurate, window)
    res = {"fwd_launches": fwd_launches, "bwd_launches": bwd_launches, "guards_intact": all(g.guard_ok() for g in list(fb.values()) + list(bb.values()))}
    del bb["ws"]
    if n_seq == 0:
        return res
    w, pad, L, T_p = window, (window - 1) // 2, out_len(T, window), T + 2
    ldx, ldf, ids, dout = o["ldx"], o["ldf"], o["ids"], o["dout"]
    n_tok, n_out = n_seq * T, n_seq * L
    res["bad_id_flag"] = int(fb["flag"].body.item())
    ids_flat = ids.reshape(-1)
    bad = (ids_flat < 0) | (ids_flat >= V)
    res["bad_ids_planted"] = int(bad.sum())
    res["fwd_outputs_finite"] = all(bool(torch.isfinite(fb[k].body.float()).all()) for k in ("Xp", "Y", "w", "out")) and \
        (not accurate or bool(torch.isfinite(fb["Ylo"].body.view(n_out, ldf)[:, :F].float()).all()))
    Xp3 = fb["Xp"].body.view(n_seq, T_p, ldx)
    Y2 = fb["Y"].body.view(n_out, ldf)
    Ylo2 = fb["Ylo"].body.view(n_out, ldf) if accurate else None
    w1, out2 = fb["w"].body, fb["out"].body.view(n_seq, F)
    W64 = o["Wc"].double().permute(1, 0, 2).contiguous()  # (w, F, d)
    Wa64, ba64, qv64, bc64 = o["Wa"].double(), o["ba"].double(), o["qv"].double(), o["bc"].double()
    table_f, kseed = o["table_f"], o["kseed"]
    scale = float(1.0 / (1.0 - torch.tensor(p_drop, dtype=torch.float32))) if p_drop > 0 else 1.0
    ids_safe = torch.where(bad, torch.zeros_like(ids_flat), ids_flat)
    scat = (ids_flat >= 1) & (ids_flat < V)
    acc = {k: 0.0 for k in ("y_ratio", "ylo_ratio", "w_err", "w_sum_err", "out_ratio")}
    worst = lambda k, t: acc.__setitem__(k, max(acc[k], G._worst(t)))
    cnt = dict(xp_mismatch_rows=0, y_dropped_nonzero=0, y_pos=0, y_n=0)
    ones_ok = True
    grads = {v: dict(dWc=torch.zeros(w, F, d + 1, dtype=torch.float64, device=dev),
                     dWa=torch.zeros(q, F + 1, dtype=torch.float64, device=dev),
                     dqv=torch.zeros(q, dtype=torch.float64, device=dev),
                     demb=torch.zeros(V, d, dtype=torch.float64, device=dev)) for v in ("exact", "contract")}
    cs = max(1, 8192 // T_p)
    for s0 in range(0, n_seq, cs):
        s1 = min(n_seq, s0 + cs)
        ns = s1 - s0
        r0, r1, o0, o1 = s0 * T, s1 * T, s0 * L, s1 * L
        seg = torch.arange(s0, s1, device=dev)
        tok_rows = (seg.view(-1, 1) * T_p + 1 + torch.arange(T, device=dev).view(1, -1)).reshape(-1)
        # Xp: masked gather, ones column at d, zero pad rows -- bit exact
        mx = G.dropout_mask_dev(kseed, p_drop, tok_rows, d, ldx)
        exp_x = torch.zeros(ns, T_p, ldx, dtype=torch.float32, device=dev)
        exp_x[:, 1:T + 1, :d] = ((table_f[ids_safe[r0:r1]] * mx).to(torch.bfloat16).float()).view(ns, T, d)
        exp_x[:, 1:T + 1, d] = 1.0
        got_x = Xp3[s0:s1]
        cnt["xp_mismatch_rows"] += int((got_x.view(torch.int16) != exp_x.to(torch.bfloat16).view(torch.int16)).any(dim=2).sum())
        X64 = got_x.double()
        # conv: pre[s, j] = sum_k Xp[s, j + 1 - p + k] . W_k + b, j < L
        pre = torch.zeros(ns * L, F, dtype=torch.float64, device=dev) + bc64
        absum = torch.zeros(ns * L, F, dtype=torch.float64, device=dev) + bc64.abs()
        for k in range(w):
            xk = X64[:, 1 - pad + k:1 - pad + k + L, :d].reshape(-1, d)
            pre += xk @ W64[k].t()
            absum += xk.abs() @ W64[k].abs().t()
        my = G.dropout_mask_dev(kseed ^ 0x5BD1E995, p_drop, torch.arange(o0, o1, device=dev), F, ldf).double()
        ref_y = pre.clamp_min(0) * my
        y = Y2[o0:o1]
        y64 = y[:, :F].double()
        bound = G._bf16_ulp(torch.maximum(ref_y.abs(), y64.abs())) + 1e-6 * absum * my.clamp_min(1.0)
        worst("y_ratio", G._safe_div((y64 - ref_y).abs(), bound))
        cnt["y_dropped_nonzero"] += int(((my == 0) & (y64 != 0)).sum())
        cnt["y_pos"] += int((pre > 0).sum())
        cnt["y_n"] += pre.numel()
        ones_ok &= bool((y[:, F] == 1).all()) and bool((y[:, F + 1:] == 0).all())
        yy = y64
        if accurate:
            yy = y64 + Ylo2[o0:o1, :F].double()
            rb = 2.0 ** -16 * ref_y.norm(dim=1) + 1e-6 * (absum * my).norm(dim=1)
            worst("ylo_ratio", G._safe_div((yy - ref_y).norm(dim=1), rb))
        # pooling over the L outputs of a title, from the kernel's own Y
        score = torch.tanh(y64 @ Wa64.t() + ba64) @ qv64
        w_ref = torch.softmax(score.view(ns, L), dim=1)
        wk = w1[o0:o1].double().view(ns, L)
        worst("w_err", (wk - w_ref).abs())
        worst("w_sum_err", (wk.sum(1) - 1).abs())
        yy3 = yy.view(ns, L, F)
        o_ref = (wk.unsqueeze(2) * yy3).sum(1)
        o_abs = (wk.unsqueeze(2) * yy3.abs()).sum(1)
        worst("out_ratio", G._safe_div((out2[s0:s1].double() - o_ref).norm(dim=1), o_abs.norm(dim=1)))
        # backward, exact and under the bf16 contract (dPre and dY stored in bf16)
        do = dout[s0:s1].double()
        dw = (y64.view(ns, L, F) * do.unsqueeze(1)).sum(2)
        dscore = wk * (dw - (wk * dw).sum(1, keepdim=True))
        th = torch.tanh(y64 @ Wa64.t() + ba64)
        dpre = dscore.reshape(-1, 1) * qv64 * (1 - th * th)
        dqv_c = (dscore.reshape(-1, 1) * th).sum(0)
        relu_keep = (y64 > 0).double() * scale
        xs = X64[:, :, :d + 1].reshape(-1, d + 1)
        y1 = torch.cat([y64, torch.ones(ns * L, 1, dtype=torch.float64, device=dev)], 1)
        sc_ids = ids_flat[r0:r1][scat[r0:r1]]
        for v in ("exact", "contract"):
            dp = dpre if v == "exact" else G.bf16r(dpre.float()).double()
            dyc = (dp @ Wa64 + wk.reshape(-1, 1) * do.repeat_interleave(L, 0)) * relu_keep
            if v == "contract":
                dyc = G.bf16r(dyc.float()).double()
            g = grads[v]
            g["dqv"] += dqv_c
            g["dWa"] += dp.t() @ y1
            dyp = torch.zeros(ns, T_p, F, dtype=torch.float64, device=dev)
            dyp[:, 1:L + 1] = dyc.view(ns, L, F)
            dyp = dyp.view(-1, F)
            n_p = dyp.shape[0]
            dX = torch.zeros(n_p, d, dtype=torch.float64, device=dev)
            for k in range(w):  # dW_k += dY^T . X[rows + k - p]; dX[r] += dY[r - k + p] . W_k
                sh = k - pad
                xsh = torch.zeros_like(xs)
                dys = torch.zeros_like(dyp)
                if sh >= 0:
                    xsh[:n_p - sh] = xs[sh:]
                    dys[sh:] = dyp[:n_p - sh]
                else:
                    xsh[-sh:] = xs[:n_p + sh]
                    dys[:n_p + sh] = dyp[-sh:]
                g["dWc"][k] += dyp.t() @ xsh
                dX += dys @ W64[k]
            dXt = dX.view(ns, T_p, d)[:, 1:T + 1].reshape(-1, d) * mx.double()
            g["demb"].index_add_(0, sc_ids, dXt[scat[r0:r1]])
    res.update(acc)
    res.update(cnt)
    res["y_pos_fraction"] = cnt["y_pos"] / max(1, cnt["y_n"])
    res["y_ones_col_and_pad_exact"] = ones_ok
    ex, co = grads["exact"], grads["contract"]
    dWc_k = (bb["dWc"].body.double() - bb["dWc"].prefill.double()).view(w, F, ldx)[:, :, :d + 1]
    dWa_k = (bb["dWa"].body.double() - bb["dWa"].prefill.double()).view(q, ldf)[:, :F + 1]
    dqv_k = bb["dqv"].body.double() - bb["dqv"].prefill.double()
    demb_k = (bb["demb"].body.double() - bb["demb"].prefill.double()).view(V, d)
    res["dWconv_tap_row_ratio"] = [G._row_ratio(dWc_k[k, :, :d], ex["dWc"][k, :, :d], co["dWc"][k, :, :d], floor=grad_floor)[0]
                                   for k in range(w)]
    res["dbias_ratio"] = G._row_ratio(*[t[pad, :, d].reshape(1, -1) for t in (dWc_k, ex["dWc"], co["dWc"])], floor=grad_floor)[0]
    res["dWa_row_ratio"] = G._row_ratio(dWa_k, ex["dWa"], co["dWa"], floor=grad_floor)[0]
    res["dqv_ratio"] = G._row_ratio(*[t.view(1, -1) for t in (dqv_k, ex["dqv"], co["dqv"])], floor=grad_floor)[0]
    touched = torch.zeros(V, dtype=torch.bool, device=dev)
    touched[ids_flat[scat]] = True
    res["demb_rows_touched"] = int(touched.sum())
    res["demb_row_ratio"] = G._row_ratio(demb_k[touched], ex["demb"][touched], co["demb"][touched], floor=grad_floor)[0]
    # the "+=" pre-fill outside what the kernels own: pitch columns, embedding rows no valid token reads
    colmask = torch.zeros(w, F, ldx, dtype=torch.bool, device=dev)
    colmask[:, :, d + 1:] = True
    res["dWconv_pitch_cols_untouched"] = bb["dWc"].unchanged(colmask)
    colmask = torch.zeros(q, ldf, dtype=torch.bool, device=dev)
    colmask[:, F + 1:] = True
    res["dWa_pitch_cols_untouched"] = bb["dWa"].unchanged(colmask)
    res["demb_untouched_rows_exact"] = bb["demb"].unchanged((~touched).view(V, 1).expand(V, d))
    return res


def assert_cnn_window(r, L):
    """The bounds of tests/test_gpu_cnn_encoder.py::assert_cnn, per conv tap and for the bias."""
    assert r["guards_intact"] and r["fwd_outputs_finite"], r
    assert r["xp_mismatch_rows"] == 0, r
    assert r["y_ratio"] <= 1.0 and r["y_dropped_nonzero"] == 0 and r["y_ones_col_and_pad_exact"], r
    assert 0.3 < r["y_pos_fraction"] < 0.7, r
    assert r["ylo_ratio"] <= 1.0, r
    assert r["w_err"] <= 2e-5 and r["w_sum_err"] <= 1e-5 and r["out_ratio"] <= 2e-6, r
    assert r["bad_id_flag"] == int(r["bad_ids_planted"] > 0), r
    assert max(r["dWconv_tap_row_ratio"]) <= 1.5 and r["dbias_ratio"] <= 1.5 and r["demb_row_ratio"] <= 1.5, r
    if L > 1:  # one output per title: w = 1, dscore = 0, dqv and dWa keep their pre-fill (not compared here)
        assert r["dWa_row_ratio"] <= 1.5 and r["dqv_ratio"] <= 1.5, r
    assert r["dWconv_pitch_cols_untouched"] and r["dWa_pitch_cols_untouched"] and r["demb_untouched_rows_exact"], r
