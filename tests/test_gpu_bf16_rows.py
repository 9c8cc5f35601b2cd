"""fp32 -> bf16 row conversions on the H100, bit for bit: every job configuration of the one conversion kernel (Bf16Rows in
csrc/nr_ops.h), reached through the unchanged C ABI or the composites that run it, against torch's round-to-nearest bf16.

  hi plane:  bf16(x), 1.0 at column D where the caller asks for the ones column, zeros up to the pitch
  low plane: bf16(x - bf16(x)), zeros from column D on

Sources are strided, transposed or misaligned views.  Outputs are pre-filled with a sentinel, so an element left unwritten fails,
and carry a guard row that must stay untouched.  Values stay out of the fp32 denormal range: the library builds with
--use_fast_math, which flushes denormals."""
import ctypes as C

import pytest
import torch

import newsrec_b200
from newsrec_b200 import GruFwdArgs, check, load_library
from newsrec_b200.ops import _p, _stream, cast_pad, ru8
from test_gpu_exp1 import _dense_forward_planes

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SENTINEL = 7.0
BF = torch.bfloat16


def _bits(t):
    return t.view(torch.int16)


def _values(shape, seed, special=True):
    """fp32 values over six decades; special: -0 and a value near the fp32 maximum in the first row"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g) * torch.logspace(-3, 3, shape[-1])
    if special:
        x.view(-1)[:2] = torch.tensor([-0.0, 3.0e38])
    return x.to(DEV)


def _buf(rows, ld):
    """rows of pitch ld plus one guard row, all sentinel"""
    return torch.full((rows + 1, ld), SENTINEL, dtype=BF, device=DEV)


def _want(x, ld, ones_col):
    """(hi, lo) planes of fp32 rows x (n, D) at pitch ld, with the untouched guard row after them"""
    n, D = x.shape
    hi = torch.zeros((n + 1, ld), dtype=BF, device=DEV)
    lo = torch.zeros((n + 1, ld), dtype=BF, device=DEV)
    hi[:n, :D] = x.to(BF)
    if ones_col:
        hi[:n, D] = 1.0
    lo[:n, :D] = (x - x.to(BF).float()).to(BF)
    hi[n], lo[n] = SENTINEL, SENTINEL
    return hi, lo


def _launches():
    return newsrec_b200.launch_count()


@pytest.mark.parametrize("R,Cc,ld,transpose,offset", [
    (97, 300, 304, False, 0),     # 16-byte aligned rows: float4 loads
    (97, 300, 320, False, 1),     # misaligned rows: scalar loads; padding beyond the next multiple of 8
    (97, 300, 104, True, 0),
    (2700, 300, 2704, True, 0),   # LSTUR's W_ih^T (Hd = 900): 338 chunks per row, more than one block of threads
    (33, 2750, 2760, False, 0),
])
def test_cast_pad(R, Cc, ld, transpose, offset):
    lib = load_library()
    lds = Cc + 5
    src = _values((R, lds), R + Cc)[:, offset:offset + Cc]
    dst = _buf(Cc if transpose else R, ld)
    n0 = _launches()
    check(lib.nr_cast_pad_bf16(_p(src), R, Cc, lds, _p(dst), ld, int(transpose), _stream()), "nr_cast_pad_bf16")
    torch.cuda.synchronize()
    assert _launches() - n0 == 1
    assert torch.equal(_bits(dst), _bits(_want(src.t() if transpose else src, ld, False)[0]))


def test_cast_pad_many_runs_eight_mixed_jobs_in_one_launch():
    lib = load_library()
    specs = [(300, 300, 304, False), (300, 912, 304, True), (200, 300, 304, False), (200, 300, 208, True),
             (2700, 300, 2704, True), (50, 7, 8, False), (3, 2750, 2752, False), (900, 301, 904, True)]
    srcs, dsts = [], []
    for i, (R, Cc, ld, tr) in enumerate(specs):
        srcs.append(_values((R, Cc + 3), 40 + i)[:, :Cc])
        dsts.append(_buf(Cc if tr else R, ld))
    n = len(specs)
    ints = lambda vals: (C.c_int * n)(*vals)
    n0 = _launches()
    check(lib.nr_cast_pad_bf16_many(n, (C.c_void_p * n)(*[s.data_ptr() for s in srcs]), ints([s[0] for s in specs]),
                                    ints([s[1] for s in specs]), ints([s[1] + 3 for s in specs]),
                                    (C.c_void_p * n)(*[d.data_ptr() for d in dsts]), ints([s[2] for s in specs]),
                                    ints([int(s[3]) for s in specs]), _stream()), "nr_cast_pad_bf16_many")
    torch.cuda.synchronize()
    assert _launches() - n0 == 1
    for (R, Cc, ld, tr), src, dst in zip(specs, srcs, dsts):
        assert torch.equal(_bits(dst), _bits(_want(src.t() if tr else src, ld, False)[0])), (R, Cc, ld, tr)


def _rows(layout, n, D, seed):
    """(n, D) fp32 rows: strided and misaligned rows, or a column-major view (element stride n + 2 along a row)"""
    if layout == "rows":
        return _values((n, D + 3), seed)[:, 1:1 + D]
    return _values((D, n + 2), seed).t()[:n]


@pytest.mark.parametrize("layout", ["rows", "columns"])
@pytest.mark.parametrize("D", [300, 2700])
def test_rows_to_bf16(layout, D):
    lib = load_library()
    n, ld = 1029, ru8(D + 1)
    x = _rows(layout, n, D, D)
    dst = _buf(n, ld)
    check(lib.nr_rows_to_bf16(_p(x), n, D, x.stride(0), x.stride(1), _p(dst), ld, _stream()), "nr_rows_to_bf16")
    torch.cuda.synchronize()
    assert torch.equal(_bits(dst), _bits(_want(x, ld, True)[0]))


@pytest.mark.parametrize("layout", ["rows", "columns"])
@pytest.mark.parametrize("D", [300, 2700])
def test_rows_to_bf16_hilo_planes(layout, D):
    lib = load_library()
    n, ld = 1029, ru8(D + 1)
    x = _rows(layout, n, D, D + 1)
    hi, lo = _buf(n, ld), _buf(n, ld)
    n0 = _launches()
    check(lib.nr_rows_to_bf16_hilo(_p(x), n, D, x.stride(0), x.stride(1), _p(hi), _p(lo), ld, _stream()), "nr_rows_to_bf16_hilo")
    torch.cuda.synchronize()
    assert _launches() - n0 == 1
    want_hi, want_lo = _want(x, ld, True)
    assert torch.equal(_bits(hi), _bits(want_hi))
    assert torch.equal(_bits(lo), _bits(want_lo))


@pytest.mark.parametrize("accurate", [True, False])
@pytest.mark.parametrize("layout", ["seq_major", "columns"])
def test_dense_encoder_input_rows(layout, accurate):
    """nr_mhsa_encoder_fwd's dense input: X (+ pos) and, in accurate mode, the K-concatenated [hi | lo] rows"""
    n_seq, T, d = 37, 50, 300
    if layout == "seq_major":  # (n_seq, T, d) viewed from [T][n_seq][d + 7] storage, rows starting 3 elements in
        x = _values((T, n_seq, d + 7), 5).transpose(0, 1)[:, :, 3:3 + d]
    else:                      # element stride n_seq * T along a row
        x = _values((d, n_seq, T), 6).permute(1, 2, 0)
    ldx = ru8(d + 1)
    pos = (torch.rand(T, d, device=DEV) * 0.2 - 0.1).contiguous()
    for p in (None, pos):
        X, kcat = _dense_forward_planes(x, p, accurate)
        xs = (x if p is None else x + p).reshape(n_seq * T, d)  # fp32 sum, then the one rounding
        want_hi, want_lo = _want(xs, ldx, True)
        assert torch.equal(_bits(X), _bits(want_hi[:-1])), p is None
        if accurate:
            assert torch.equal(_bits(kcat), _bits(torch.cat((want_hi[:-1], want_lo[:-1]), dim=1))), p is None


def test_gru_input_planes():
    """nr_gru_fwd in accurate mode: x as hi rows with the ones column plus the low plane alone (no ones column), h0 as hi rows"""
    from newsrec_b200.ops_gru import ru4
    lib = load_library()
    B, S, D, Hd = 64, 50, 300, 128
    ldd, ldh, ldg = ru8(D + 1), ru8(Hd + 1), ru4(3 * Hd)
    x = _values((S, B, D + 4), 9, special=False).transpose(0, 1)[:, :, 2:2 + D]  # (B, S, D), not contiguous
    h0 = _values((B, Hd), 10, special=False) * 1e-3
    g = torch.Generator().manual_seed(11)
    wih = cast_pad((torch.randn(3 * Hd, D, generator=g) * 0.05).to(DEV), ldd)
    whh = cast_pad((torch.randn(3 * Hd, Hd, generator=g) * 0.05).to(DEV), ldh)
    bih, bhh = torch.zeros(3 * Hd, device=DEV), torch.zeros(3 * Hd, device=DEV)
    lengths = torch.randint(1, S + 1, (B,), generator=g).to(DEV)
    xb, x_lo = _buf(B * S, ldd), _buf(B * S, ldd)
    gi = torch.empty((B * S, ldg), device=DEV)
    gh = torch.empty((S, B, ldg), device=DEV)
    hs = torch.empty((S + 1, B, Hd), device=DEV)
    hb = torch.full(((S + 1) * B, ldh), SENTINEL, dtype=BF, device=DEV)
    out = torch.empty((B, Hd), device=DEV)
    a = GruFwdArgs()
    a.B, a.S, a.D, a.Hd = B, S, D, Hd
    a.x = _p(x)
    a.x_s_b, a.x_s_t, a.x_s_c = x.stride()
    a.len, a.h0, a.wih_bf16, a.whh_bf16, a.bih, a.bhh = _p(lengths), _p(h0), _p(wih), _p(whh), _p(bih), _p(bhh)
    a.xb, a.gi, a.gh, a.hs, a.hb, a.out, a.x_lo_bf16 = _p(xb), _p(gi), _p(gh), _p(hs), _p(hb), _p(out), _p(x_lo)
    check(lib.nr_gru_fwd(C.byref(a), _stream()), "nr_gru_fwd")
    torch.cuda.synchronize()
    want_hi, want_lo = _want(x.reshape(B * S, D), ldd, True)
    assert torch.equal(_bits(xb), _bits(want_hi))
    assert torch.equal(_bits(x_lo), _bits(want_lo))
    assert torch.equal(_bits(hb[:B]), _bits(_want(h0, ldh, True)[0][:B]))


def test_empty_problems_launch_nothing():
    lib = load_library()
    D, ld = 300, 304
    x = _values((4, D), 12)
    hi, lo = _buf(4, ld), _buf(4, ld)
    one_i, one_p = (C.c_int * 1)(1), (C.c_void_p * 1)(x.data_ptr())
    n0 = _launches()
    check(lib.nr_rows_to_bf16(_p(x), 0, D, D, 1, _p(hi), ld, _stream()), "nr_rows_to_bf16")
    check(lib.nr_rows_to_bf16_hilo(_p(x), 0, D, D, 1, _p(hi), _p(lo), ld, _stream()), "nr_rows_to_bf16_hilo")
    check(lib.nr_cast_pad_bf16(_p(x), 0, D, D, _p(hi), ld, 0, _stream()), "nr_cast_pad_bf16")
    check(lib.nr_cast_pad_bf16_many(0, one_p, one_i, one_i, one_i, one_p, one_i, one_i, _stream()), "nr_cast_pad_bf16_many")
    torch.cuda.synchronize()
    assert _launches() == n0
    assert bool((hi.float() == SENTINEL).all()) and bool((lo.float() == SENTINEL).all())
