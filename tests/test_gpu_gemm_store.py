"""gemm_store (gemm_nt + EpiStore) with every option of its epilogue, through nr_debug_gemm_store, judged element by element
against fp64 evaluations on the device of the exact bf16 operands the kernel read, at the cases of tests/gemm_cases.py
STORE_CASES (whose option, regime and store-path labels tests/test_gemm_plan_host.py checks against gemm_plan_ref).

Bounds per output element, with e = 4u (n_acc + 2) S as in gpu_checks.gemm_elem_ratio (u = 2^-24, S = sum of |products| +
|bias| (+ |pre-fill| for "+="), n_acc = taps * ceil(K / 16)), and half a bf16 ulp of |y| + allowance on top for a bf16 output:
  plain / ReLU   y = pre (ReLU: max(pre, 0), 1-Lipschitz): allowance e.
  tanh           y = tanh(pre): |tanh'| <= 1 passes e through with a factor of at most 1; fast_tanh adds TANH_ERR absolute, and
                 its fp32 evaluation 4u absolute (|tanh| <= 1): allowance e + TANH_ERR + 4u.
  dtanh          y = pre (1 - t^2), t the bf16 source value: t^2 has 16 significant bits and is exact in fp32, so 1 - t^2 and the
                 product cost at most two roundings: allowance (1 - t^2) e + 2u |y|.
  dropout        the mask (gpu_checks.dropout_mask_dev, keyed on the OUTPUT row after the map and the output pitch) multiplies
                 y and the allowance by 0 or the scale, plus one rounding u |y|: a dropped element must be exactly 0, in the
                 output and in the low plane.
  low plane      hi + lo (lo = bf16(y - bf16(y)) of the fp32 result) stays within the allowance + 2^-17 |y| (hi + lo misses
                 the fp32 value by at most half a bf16 ulp of |y - hi| <= 2^-18 |y|); the hi plane alone must miss that bound by
                 >= 8x on its worst element (half a bf16 ulp is 2^-9 |y|), or the plane would carry nothing.
  "+="           y = pre-fill + act(pre) (the epilogue's result is added to the output), the pre-fill counted in S (as in the
                 gemm_tn test).
  ones column    exactly 1.0 at column N and exactly 0 up to the limit, in mapped rows only.
The ratio (|got - y| - rounding) / allowance must stay <= 1 everywhere (+inf for a NaN).  A dropped k-chunk, a tap read from
the wrong row, a mask keyed on the wrong row or a lost pre-fill misses it by orders of magnitude; the reference-side checks
below show the last two.

Around the values: pitch columns, unmapped rows (pad rows, rows past a window's L, the row past the result), the low plane's
pitch and a guard band behind every buffer keep their pre-fill bit for bit; a second run is bit-identical (one CTA owns each
element, the dropout mask is a hash); each call is one launch; every configuration gemm_store refuses returns -1 before any
launch; and the low plane is accepted exactly where gemm_plan_ref.lo_supported says it is chunk aligned."""
import ctypes

import pytest
import torch

import gemm_cases as C
import gemm_plan_ref as P
import gpu_checks as G
import newsrec_b200 as nb

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = G.U32
SEED = 0x9E3779B97F4A7C15


def _bf16_rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return ((torch.rand(shape, generator=g) * 2 - 1) * scale).to(torch.bfloat16).to(DEV)


def _ptr(t, off_bytes=0):
    return None if t is None else t.data_ptr() + off_bytes


def _operands(c, s, seed=1):
    """bf16 A [M][lda] and W [taps * N][lda] with NaN in their pitch columns, fp32 bias or None, the bf16 tanh-backward source
    (values in (-1, 1), NaN outside the output's rows and columns) and its pitch and offset."""
    N, K, taps, M = c["N"], c["K"], c.get("taps", 1), s["M"]
    lda = c.get("lda", G.ru8(K + 1))
    A = torch.full((M, lda), float("nan"), dtype=torch.bfloat16, device=DEV)
    A[:, :K] = _bf16_rand((M, K), seed)
    W = torch.full((taps * N, lda), float("nan"), dtype=torch.bfloat16, device=DEV)
    W[:, :K] = _bf16_rand((taps * N, K), seed + 1, 0.1)
    bias = (torch.rand(N, generator=torch.Generator().manual_seed(seed + 2)) - 0.5).to(DEV) if c.get("bias", True) else None
    dsrc, d_ld, d_off = None, 0, 0
    if c.get("dtanh"):
        d_ld, d_off = c.get("dtanh_ld", s["ld_out"] + 8), c.get("dtanh_off", 0)
        dsrc = torch.full((d_off + s["out_rows"] * d_ld + 8,), float("nan"), dtype=torch.bfloat16, device=DEV)
        dsrc[d_off:d_off + s["out_rows"] * d_ld].view(s["out_rows"], d_ld)[:, :N] = _bf16_rand((s["out_rows"], N), seed + 3, 0.999)
    return A, W, lda, bias, dsrc, d_ld, d_off


def _args(c, s, ops, out_buf, lo_buf, **over):
    """The entry's arguments for a case with the _operands ops; over sets fields directly."""
    A, W, lda, bias, dsrc, d_ld, d_off = ops
    a = nb.GemmStoreArgs(A=_ptr(A), M=s["M"], lda=lda, W=_ptr(W), N=c["N"], ldw=lda, K=c["K"], taps=c.get("taps", 1),
                         w_tap_rows=s["w_tap_rows"], tap_origin=c.get("tap_origin", -1),
                         out=_ptr(out_buf, out_buf.element_size() * c.get("out_off", 0)), ld_out=s["ld_out"], out_bf16=c.get("out_bf16", 1),
                         relu=c.get("relu", 0), tanh=c.get("tanh", 0), dtanh_src=_ptr(dsrc, 2 * d_off), dtanh_ld=d_ld, bias=_ptr(bias),
                         p_drop=c.get("p", 0.0), seed=SEED, ones_col=s["ones_col"], ones_zero_upto=s["ones_upto"],
                         lo_out=_ptr(lo_buf), ld_lo=s["ld_lo"], lo_col0=s["lo_col0"] if s["lo_col0"] is not None else 0,
                         accumulate=c.get("acc", 0), rows_per_tile=s["rpt"])
    for i, f in enumerate(("rm_seg_in", "rm_in_off", "rm_seg_len", "rm_seg_out", "rm_out_off")):
        setattr(a, f, s["rm"][i])
    for k, v in over.items():
        setattr(a, k, v)
    return a


def _row_map(s):
    """RowMap::map over the A rows: (A rows that reach the output, their output rows)."""
    g = torch.arange(s["M"], device=DEV)
    seg_in, in_off, seg_len, seg_out, out_off = s["rm"]
    if seg_in == 0:
        return g, g
    sg = g // seg_in
    t = g - sg * seg_in - in_off
    ok = (t >= 0) & (t < seg_len)
    return g[ok], (sg * seg_out + t + out_off)[ok]


def _expect(c, s, A, W, bias, dsrc, d_ld, d_off, prefill, mask_rows="output", with_prefill=True):
    """fp64 value y and allowance of every mapped output element (the rows of _row_map, columns [0, N)).  mask_rows / with_prefill
    perturb the reference for the discrimination checks: "input" keys the dropout mask on the A row."""
    N, K, taps = c["N"], c["K"], c.get("taps", 1)
    grow, orow = _row_map(s)
    origin = c.get("tap_origin", -1)
    pre, absum = G.linear_ref(A[:, :K].double(), W[:, :K].double(), None if bias is None else bias.double(), N, taps,
                              s["w_tap_rows"], origin if origin >= 0 else None)
    pre, absum = pre[grow], absum[grow]
    pf = 0
    if c.get("acc") and with_prefill:
        pf = prefill[c.get("out_off", 0):c.get("out_off", 0) + s["out_rows"] * s["ld_out"]].view(s["out_rows"], s["ld_out"])
        pf = pf[orow, :N].double()
        absum = absum + pf.abs()
    e = 4 * U * (taps * -(-K // 16) + 2) * absum
    if c.get("relu"):
        y, allow = pre.clamp_min(0), e
    elif c.get("tanh"):
        y, allow = torch.tanh(pre), e + G.TANH_ERR + 4 * U
    elif c.get("dtanh"):
        t = dsrc[d_off:d_off + s["out_rows"] * d_ld].view(s["out_rows"], d_ld)[orow, :N].double()
        y = pre * (1 - t * t)
        allow = (1 - t * t) * e + 2 * U * y.abs()
    else:
        y, allow = pre, e
    if c.get("p", 0) > 0:
        m = G.dropout_mask_dev(SEED, c["p"], orow if mask_rows == "output" else grow, N, s["ld_out"]).double()
        y = y * m
        allow = allow * m + U * y.abs()
    return y + pf, allow, orow


def _ratio(got, y, allow, bf16):
    err = (got.double() - y).abs()
    if bf16:
        err = (err - 0.5 * G._bf16_ulp(y.abs() + allow)).clamp_min(0)
    return G._worst(G._safe_div(err, allow))


def _buffers(c, s):
    """The output (NaN, or a random pre-fill for "+="; out_off elements before it, one row past it) and the low plane (NaN, one
    row past the result), each followed by a guard band."""
    n = c.get("out_off", 0) + (s["out_rows"] + 1) * s["ld_out"]
    if c.get("out_bf16", 1):
        out = G._Guarded(n, torch.bfloat16, float("nan"))
    elif c.get("acc"):
        out = G._Guarded(n, torch.float32, torch.rand(n, generator=torch.Generator().manual_seed(5)).to(DEV) * 2 - 1)
    else:
        out = G._Guarded(n, torch.float32, float("nan"))
    if out.prefill is None:
        out.prefill = out.body.clone()
    lo = None
    if s["lo_col0"] is not None:
        lo = G._Guarded((s["out_rows"] + 1) * s["ld_lo"], torch.bfloat16, float("nan"))
        lo.prefill = lo.body.clone()
    return out, lo


@pytest.mark.parametrize("c", C.STORE_CASES, ids=lambda c: c["id"])
def test_gemm_store_elements(c):
    lib = G.load_library()
    s = C.store_setup(c)
    N, ld, bf16, off = c["N"], s["ld_out"], c.get("out_bf16", 1), c.get("out_off", 0)
    ops = _operands(c, s)
    A, W, lda, bias, dsrc, d_ld, d_off = ops
    runs = []
    for _ in range(2):
        out, lo = _buffers(c, s)
        n0 = lib.nr_launch_count()
        args = _args(c, s, ops, out.all, None if lo is None else lo.all)
        G.check(lib.nr_debug_gemm_store(ctypes.byref(args), G._stream()), "nr_debug_gemm_store")
        torch.cuda.synchronize()
        assert lib.nr_launch_count() == n0 + 1
        runs.append((out, lo))
    out, lo = runs[0]
    y, allow, orow = _expect(c, s, A, W, bias, dsrc, d_ld, d_off, out.prefill)
    view = out.body[off:off + s["out_rows"] * ld].view(s["out_rows"], ld)
    got = view[orow, :N]
    res = {"elem_ratio": _ratio(got, y, allow, bf16)}
    written = torch.zeros(out.n, dtype=torch.bool, device=DEV)
    wview = written[off:off + s["out_rows"] * ld].view(s["out_rows"], ld)
    wview[orow.view(-1, 1), torch.arange(N, device=DEV).view(1, -1)] = True
    if s["ones_col"] >= 0:
        oc, upto = s["ones_col"], s["ones_upto"]
        res["ones_exact"] = bool((view[orow, oc] == 1.0).all()) and bool((view[orow, oc + 1:upto].view(torch.int16) == 0).all())
        wview[orow.view(-1, 1), torch.arange(oc, max(upto, oc + 1), device=DEV).view(1, -1)] = True
    res["untouched"] = out.unchanged(~written)
    res["guard"] = all(o.guard_ok() and (l is None or l.guard_ok()) for o, l in runs)
    res["rerun_bit_identical"] = G._bits_equal(runs[0][0].body, runs[1][0].body) and (
        lo is None or G._bits_equal(runs[0][1].body, runs[1][1].body))
    if lo is not None:
        l0 = s["lo_col0"]
        lview = lo.body.view(s["out_rows"] + 1, s["ld_lo"])
        lgot, hi, yl = lview[orow, :N - l0].double(), got[:, l0:].double(), y[:, l0:]
        bound = allow[:, l0:] + 2.0 ** -17 * yl.abs()
        res["hilo_ratio"] = G._worst(G._safe_div((hi + lgot - yl).abs(), bound))
        res["hi_only_ratio"] = G._worst(G._safe_div((hi - yl).abs(), bound))
        lw = torch.zeros(s["out_rows"] + 1, s["ld_lo"], dtype=torch.bool, device=DEV)
        lw[orow.view(-1, 1), torch.arange(N - l0, device=DEV).view(1, -1)] = True
        res["lo_untouched"] = lo.unchanged(~lw)
        assert res["hilo_ratio"] <= 1 and res["hi_only_ratio"] >= 8 and res["lo_untouched"], res
    # reference-side discrimination: the judge fails a mask keyed on the A row, and a "+=" reference without the pre-fill
    if c.get("p", 0) > 0 and c.get("rm"):
        yw, aw, _ = _expect(c, s, A, W, bias, dsrc, d_ld, d_off, out.prefill, mask_rows="input")
        res["input_row_mask_ratio"] = _ratio(got, yw, aw, bf16)
        assert res["input_row_mask_ratio"] > 10, res
    if c.get("acc"):
        yw, aw, _ = _expect(c, s, A, W, bias, dsrc, d_ld, d_off, out.prefill, with_prefill=False)
        res["no_prefill_ratio"] = _ratio(got, yw, aw, bf16)
        assert res["no_prefill_ratio"] > 10, res
    assert res["elem_ratio"] <= 1 and res.get("ones_exact", True), res
    assert res["untouched"] and res["guard"] and res["rerun_bit_identical"], res
    print(c["id"], res)


# a configuration gemm_store takes (64 x 64 x 64, bf16, TMA), and the changes to it that it must refuse before any launch, with
# a word of the message that names the reason
_BASE = dict(id="base", M=64, N=64, K=64, dtanh=1)
_REFUSED = {
    "ones column on an fp32 output": (dict(out_bf16=0, ld_out=68, ones_col=64, ones_zero_upto=68), "ones column"),
    "ones column inside the result (N - 1)": (dict(ones_col=63), "ones column"),
    "ones column inside the result (0)": (dict(ones_col=0), "ones column"),
    "ones column past the pitch": (dict(ones_col=72, ones_zero_upto=72), "ones column"),
    "zeroed columns past the pitch": (dict(ones_col=64, ones_zero_upto=80), "zeroed columns"),
    "output base off 16 bytes": (dict(out_shift=8), "aligned bases"),
    "low plane base off 16 bytes": (dict(lo=True, lo_shift=8), "aligned bases"),
    "tanh-backward source off 4 bytes": (dict(dtanh_shift=2), "aligned bases"),
    "relu and tanh": (dict(relu=1, tanh=1), "one activation"),
    "+= on a bf16 output": (dict(accumulate=1), "accumulation needs an fp32 output"),
    "low plane on an fp32 output": (dict(out_bf16=0, ld_out=68, lo=True), "low plane needs"),
    "low plane from column N": (dict(lo=True, lo_col0=64), "low plane needs"),
    "low plane from a negative column": (dict(lo=True, lo_col0=-8), "low plane needs"),
    "low plane pitch not a multiple of 8": (dict(lo=True, ld_lo=68), "low plane needs"),
    "low plane pitch below its columns": (dict(lo=True, ld_lo=56), "low plane needs"),
    "low plane off a chunk boundary": (dict(lo=True, lo_col0=16), "not chunk aligned"),
    "low plane off 8 columns without TMA": (dict(lo=True, lo_col0=4, rows_per_tile=50), "low plane needs"),
    "odd tanh-backward pitch": (dict(dtanh_ld=73), "tanh-backward source"),
    "tap origin past the taps": (dict(taps=2, w_tap_rows=64, tap_origin=2), "tap origin"),
    "five taps": (dict(taps=5, w_tap_rows=64), "bad shape"),
    "bf16 output pitch not a multiple of 8": (dict(ld_out=68), "output pitch"),
    "fp32 output pitch not a multiple of 4": (dict(out_bf16=0, ld_out=66), "output pitch"),
    "null A": (dict(A=None), "null operand"),
    "null W": (dict(W=None), "null operand"),
    "null output": (dict(out=None), "null operand"),
}


def test_gemm_store_refuses_before_any_launch():
    """Every refused configuration returns -1 with a message, launches nothing and writes nothing; the base configuration runs."""
    lib = G.load_library()
    s = C.store_setup(_BASE)
    ops = _operands(_BASE, s)
    out = G._Guarded(64 * 80 * 2 + 64, torch.float32, float("nan"))  # 64 rows at every pitch below, as fp32
    out.prefill = out.body.clone()
    lo = G._Guarded(64 * 80, torch.bfloat16, float("nan"))
    A5 = torch.zeros(64, 72, dtype=torch.bfloat16, device=DEV)
    W5 = torch.zeros(5 * 64, 72, dtype=torch.bfloat16, device=DEV)
    for name, (over, reason) in _REFUSED.items():
        over = dict(over)
        shifts = {k: over.pop(k, 0) for k in ("out_shift", "lo_shift", "dtanh_shift")}
        use_lo = over.pop("lo", False)
        a = _args(_BASE, s, ops, out.all, lo.all if use_lo else None, **over)
        if "taps" in over:
            a.A, a.W = A5.data_ptr(), W5.data_ptr()
        a.out = None if "out" in over else out.all.data_ptr() + shifts["out_shift"]
        if use_lo:
            a.lo_out = lo.all.data_ptr() + shifts["lo_shift"]
            a.ld_lo = over.get("ld_lo", 64)
            a.lo_col0 = over.get("lo_col0", 0)
        a.dtanh_src = ops[4].data_ptr() + shifts["dtanh_shift"]
        n0 = lib.nr_launch_count()
        rc = lib.nr_debug_gemm_store(ctypes.byref(a), G._stream())
        msg = lib.nr_last_error()
        assert rc == -1 and reason.encode() in msg and lib.nr_launch_count() == n0, (name, rc, msg)
    torch.cuda.synchronize()
    assert out.unchanged(torch.ones(out.n, dtype=torch.bool, device=DEV)) and out.guard_ok() and lo.guard_ok()
    assert bool(torch.isnan(lo.body.float()).all())
    n0 = lib.nr_launch_count()
    a = _args(_BASE, s, ops, out.all, None)
    G.check(lib.nr_debug_gemm_store(ctypes.byref(a), G._stream()), "nr_debug_gemm_store")
    torch.cuda.synchronize()
    assert lib.nr_launch_count() == n0 + 1 and out.guard_ok()


@pytest.mark.parametrize("N,K", [(72, 20), (120, 40), (192, 60), (400, 300), (432, 140), (912, 300), (840, 280), (257, 65)])
def test_gemm_store_low_plane_accepted_where_chunk_aligned(N, K):
    """For every lo_col0 = 0, 8, ... < N the entry accepts the low plane (and launches once) exactly where gemm_plan_ref.lo_supported
    says no 32-column chunk of a weight slice straddles it; the configuration is otherwise on the TMA path, where only the chunk
    alignment decides."""
    lib = G.load_library()
    c = dict(id="sweep", M=64, N=N, K=K)
    s = C.store_setup(c)
    ops = _operands(c, s)
    out = torch.empty(64 * s["ld_out"], dtype=torch.bfloat16, device=DEV)
    ld_lo = G.ru8(N) + 8
    lo = torch.empty(64 * ld_lo, dtype=torch.bfloat16, device=DEV)
    got, want = [], []
    for l0 in range(0, N, 8):
        a = _args(c, s, ops, out, lo, ld_lo=ld_lo, lo_col0=l0)
        n0 = lib.nr_launch_count()
        rc = lib.nr_debug_gemm_store(ctypes.byref(a), G._stream())
        assert rc in (0, -1) and lib.nr_launch_count() == n0 + (rc == 0), (l0, rc)
        got.append(rc == 0)
        want.append(P.lo_supported(N, K, l0))
    torch.cuda.synchronize()
    assert got == want, [(8 * i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert any(want)
