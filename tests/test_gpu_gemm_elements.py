"""nr_linear (gemm_nt + the store epilogue) and nr_gemm_tn (the split-K weight-gradient GEMM) judged element by element
against fp64 evaluations on the device of the exact bf16 operands the kernels read, at one case per planner regime
(tests/gemm_cases.py, whose labels tests/test_gemm_plan_host.py checks against the planner restatement).

Bound per element (gpu_checks.gemm_elem_ratio): 4u (n_acc + 2) S with S = sum of |products| + |bias| (+ |pre-fill| for the
"+=" output), n_acc = taps * ceil(K/16) for gemm_nt and ceil(Kr/16) + k-ranges for gemm_tn, plus half a bf16 ulp for a bf16
output.  A dropped or doubled k-chunk, a tap shifted by a row or a misplaced slice misses it by orders of magnitude.

Around the values: outputs nobody should write (pitch columns, rows past the result, the guard band behind the buffer) keep
their pre-fill bit for bit; gemm_nt gives bit-identical results on a second run (one CTA owns each element, in a fixed
order); the per-CTA counters of nr_debug_set_gemm_timing show the slice and the tile counts gemm_plan_ref predicts."""
import pytest
import torch

import gemm_cases as C
import gemm_plan_ref as P
import gpu_checks as G

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture(autouse=True)
def _library_defaults():
    """nr_debug_set_gemm_timing and nr_reserve_sms_for_comm are process-wide: back to their defaults after every test."""
    yield
    lib = G.load_library()
    lib.nr_debug_set_gemm_timing(None, 0)
    lib.nr_reserve_sms_for_comm(0)


def _bf16_rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return ((torch.rand(shape, generator=g) * 2 - 1) * scale).to(torch.bfloat16).to(DEV)


def _pack_linear(c, seed=1):
    """bf16 A [M][lda] and W [taps * N][ldw] with NaN in their pitch columns (the kernels' maps end at K), fp32 bias or None.
    taps 3: n_seg segments of T token rows between zero pad rows, tap s of W at rows [s N, s N + N)."""
    M, _, _ = C.linear_shape(c)
    N, K, taps = c["N"], c["K"], c.get("taps", 1)
    lda = G.ru8(K + 1)
    A = torch.full((M, lda), float("nan"), dtype=torch.bfloat16, device=DEV)
    if taps > 1:
        T = c["T"]
        Xp = torch.zeros(c["n_seg"], T + 2, K, dtype=torch.bfloat16, device=DEV)
        Xp[:, 1:T + 1] = _bf16_rand((c["n_seg"], T, K), seed)
        A[:, :K] = Xp.view(M, K)
    else:
        A[:, :K] = _bf16_rand((M, K), seed)
    W = torch.full((taps * N, lda), float("nan"), dtype=torch.bfloat16, device=DEV)
    Wt = _bf16_rand((N, taps, K), seed + 1, 0.1)
    for s in range(taps):
        W[s * N:(s + 1) * N, :K] = Wt[:, s]
    bias = (torch.rand(N, generator=torch.Generator().manual_seed(seed + 2)) - 0.5).to(DEV) if c.get("bias", True) else None
    return A, W, bias, lda


def _run_linear(lib, c, A, W, bias, lda, out):
    M, rpt, w_tap_rows = C.linear_shape(c)
    N, ld_out = c["N"], out.n // (M + 1)
    G.check(lib.nr_linear(G._p(A), M, lda, G._p(W), N, lda, c["K"], c.get("taps", 1), w_tap_rows, rpt, G._p(bias), c.get("relu", 0),
                          G._p(out.all), ld_out, c.get("out_bf16", 1), G._stream()), "nr_linear")


@pytest.mark.parametrize("c", C.LINEAR_CASES, ids=lambda c: c["id"])
def test_linear_elements(c):
    lib = G.load_library()
    M, rpt, w_tap_rows = C.linear_shape(c)
    N, K, taps, out_bf16 = c["N"], c["K"], c.get("taps", 1), c.get("out_bf16", 1)
    A, W, bias, lda = _pack_linear(c)
    ld_out = G.ru8(N + 1) if out_bf16 else (N + 3) // 4 * 4 + 4  # pitch columns on both
    dt = torch.bfloat16 if out_bf16 else torch.float32
    outs = []
    for run in range(2):
        out = G._Guarded((M + 1) * ld_out, dt, float("nan"))  # one row past M, then the guard band
        out.prefill = out.body.clone()
        timing = None
        if run == 1 and c.get("sched"):
            timing = torch.full((148 * 16,), -1, dtype=torch.int64, device=DEV)
            lib.nr_debug_set_gemm_timing(G._p(timing), 1)
        try:
            _run_linear(lib, c, A, W, bias, lda, out)
            torch.cuda.synchronize()
        finally:
            lib.nr_debug_set_gemm_timing(None, 0)
        outs.append(out)
    out = outs[0]
    pre, absum = G.linear_ref(A[:, :K].double(), W[:, :K].double(), None if bias is None else bias.double(), N, taps, w_tap_rows)
    got = out.body.view(M + 1, ld_out)[:M, :N]
    ratio, zero_exact = G.gemm_elem_ratio(got, pre, absum, taps * -(-K // 16), out_bf16, c.get("relu", 0))
    untouched = torch.ones(M + 1, ld_out, dtype=torch.bool, device=DEV)
    untouched[:M, :N] = False
    res = {"elem_ratio": ratio, "relu_zero_exact": zero_exact, "untouched": out.unchanged(untouched),
           "guard": outs[0].guard_ok() and outs[1].guard_ok(), "rerun_bit_identical": G._bits_equal(outs[0].body, outs[1].body)}
    assert res["elem_ratio"] <= 1 and res["relu_zero_exact"], res
    assert res["untouched"] and res["guard"] and res["rerun_bit_identical"], res
    if c.get("sched"):
        _check_schedule(timing, P.plan_nt(M, N, K, taps, rpt, sms=int(lib.nr_num_sms())))
    print(c["id"], res)


def _check_schedule(timing, plan):
    """Per CTA of the launch: [1] the weight slice, [8 + 4w + 3] the tiles warpgroup w processed; CTAs past the grid wrote nothing."""
    t = timing.view(148, 16).cpu()
    grid = plan["grid"]
    assert int((t[:, 5] >= 0).sum()) == grid and bool((t[grid:] == -1).all()), ("CTAs", grid, int((t[:, 5] >= 0).sum()))
    for b in range(grid):
        w0, w1 = plan["wg_tiles"][b]
        assert int(t[b, 1]) == plan["slice_of"][b], ("slice", b, int(t[b, 1]), plan["slice_of"][b])
        assert (int(t[b, 8 + 3]), int(t[b, 12 + 3])) == (len(w0), len(w1)), ("tiles", b, t[b].tolist(), len(w0), len(w1))


def test_linear_empty_launches_nothing():
    lib = G.load_library()
    A = torch.zeros(8, 8, dtype=torch.bfloat16, device=DEV)
    out = G._Guarded(64, torch.bfloat16, float("nan"))
    n0 = lib.nr_launch_count()
    G.check(lib.nr_linear(G._p(A), 0, 8, G._p(A), 4, 8, 4, 1, 0, 64, None, 0, G._p(out.all), 8, 1, G._stream()), "nr_linear")
    torch.cuda.synchronize()
    assert lib.nr_launch_count() == n0 and out.guard_ok()


# ------------------------------------------------------------------------------------------------
# nr_gemm_tn
# ------------------------------------------------------------------------------------------------
def _pack_tn(c, seed=11):
    """A [Kr][lda] bf16 (columns < Ma), B [Kr][ldb] bf16 (columns < b_cols), NaN in both pitches (the maps end at Ma / b_cols)."""
    Kr, Ma = c["Kr"], c["Ma"]
    b_cols = c.get("b_cols", c.get("b_col0", 0) + c["Nb"])
    lda, ldb = G.ru8(Ma + 1), G.ru8(b_cols + 1)
    A = torch.full((max(Kr, 1), lda), float("nan"), dtype=torch.bfloat16, device=DEV)
    B = torch.full((max(Kr, 1), ldb), float("nan"), dtype=torch.bfloat16, device=DEV)
    A[:Kr, :Ma] = _bf16_rand((Kr, Ma), seed, 0.5)
    B[:Kr, :b_cols] = _bf16_rand((Kr, b_cols), seed + 1, 0.5)
    return A, B, lda, ldb, b_cols


@pytest.mark.parametrize("c", C.GEMM_TN_CASES, ids=lambda c: c["id"])
def test_gemm_tn_elements(c):
    lib = G.load_library()
    Kr, Ma, Nb, shift, b_col0 = c["Kr"], c["Ma"], c["Nb"], c.get("shift", 0), c.get("b_col0", 0)
    A, B, lda, ldb, b_cols = _pack_tn(c)
    ldd = Nb + 2 if not c.get("odd_d") else Nb + (2 if Nb % 2 == 0 else 1) + 1  # pitch columns; odd_d: an odd pitch
    off = 1 if c.get("odd_d") else 0                                            # odd_d: D one float past an aligned base
    rows = Ma + 2                                                               # two rows past Ma
    n = off + rows * ldd
    D = G._Guarded(n, torch.float32, torch.rand(n, generator=torch.Generator().manual_seed(5)).to(DEV) * 2 - 1)
    reserve = c.get("reserve", 0)
    sms = int(lib.nr_num_sms())
    lib.nr_reserve_sms_for_comm(sms if reserve == "all" else reserve)
    try:
        G.check(lib.nr_gemm_tn(G._p(A), Kr, Ma, lda, G._p(B), Kr, b_cols, ldb, b_col0, Nb, shift,
                               G.C.c_void_p(D.all.data_ptr() + 4 * off), ldd, G._stream()), "nr_gemm_tn")
        torch.cuda.synchronize()
    finally:
        lib.nr_reserve_sms_for_comm(0)
    prod, absum = G.gemm_tn_ref(A[:Kr, :Ma].double(), B[:Kr, b_col0:b_col0 + Nb].double(), shift)
    pre = D.prefill[off:].view(rows, ldd)[:Ma, :Nb].double()
    got = D.body[off:].view(rows, ldd)[:Ma, :Nb]
    plan = P.plan_tn(Kr, Ma, Nb, sms=sms, reserved=sms if reserve == "all" else reserve)
    ratio, _ = G.gemm_elem_ratio(got, prod + pre, absum + pre.abs(), -(-Kr // 16) + plan["k_slices_max"], 0)
    untouched = torch.ones(n, dtype=torch.bool, device=DEV)
    untouched[off:].view(rows, ldd)[:Ma, :Nb] = False
    res = {"elem_ratio": ratio, "untouched": D.unchanged(untouched), "guard": D.guard_ok(), "plan": plan}
    assert res["elem_ratio"] <= 1 and res["untouched"] and res["guard"], res
    print(c["id"], res)


def test_gemm_tn_empty_and_refused_shapes_launch_nothing():
    """Kr = 0 adds nothing and launches nothing; Nb = 0, Nb = 513 and Ma = 0 are refused before any launch."""
    lib = G.load_library()
    A, B = (torch.zeros(64, 1024, dtype=torch.bfloat16, device=DEV) for _ in range(2))
    D = G._Guarded(64 * 520, torch.float32, torch.rand(64 * 520).to(DEV))
    n0 = lib.nr_launch_count()
    G.check(lib.nr_gemm_tn(G._p(A), 0, 64, 1024, G._p(B), 64, 513, 1024, 0, 64, 0, G._p(D.all), 520, G._stream()), "nr_gemm_tn")
    for Ma, Nb in [(64, 0), (64, 513), (0, 64)]:
        assert lib.nr_gemm_tn(G._p(A), 64, Ma, 1024, G._p(B), 64, 513, 1024, 0, Nb, 0, G._p(D.all), 520, G._stream()) != 0, (Ma, Nb)
    torch.cuda.synchronize()
    assert lib.nr_launch_count() == n0
    assert D.unchanged(torch.ones(D.n, dtype=torch.bool, device=DEV)) and D.guard_ok()
