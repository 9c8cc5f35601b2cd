"""Case tables of the element-by-element GEMM and pooling tests (tests/test_gpu_gemm_elements.py,
tests/test_gpu_additive_fwd.py, tests/test_gpu_additive_bwd_elements.py).  Each case names the planner regimes it is there to reach; tests/test_gemm_plan_host.py
checks those names against the planner restatement (tests/gemm_plan_ref.py) on an H100 SXM's 132 SMs, and that every
regime has a case.  Plain Python: importable without CUDA."""
from __future__ import annotations

# nr_linear: M rows (taps 3: n_seg segments of T tokens in the padded layout, M = n_seg * (T + 2)), N x K weights.
# sched: the GPU test also reads the kernel's per-CTA counters and compares the schedule with gemm_plan_ref.
LINEAR_CASES = [
    dict(id="M1_N900", M=1, N=900, K=300, regimes=("slices > 1", "warpgroup 1 idle")),
    dict(id="M63_N20", M=63, N=20, K=300, regimes=("N < 32", "1 slice")),
    dict(id="M64_N33_K64", M=64, N=33, K=64, regimes=("slice width % 32 != 0",)),
    dict(id="M65_N240_K16", M=65, N=240, K=16, relu=1, regimes=("1 slice", "slice width % 32 != 0")),
    dict(id="pp_M64x27", M=64 * 27, N=900, K=300, sched=True, regimes=("slices > 1", "warpgroup 1 idle", "even tiles per CTA")),
    dict(id="pp_M64x53p5", M=64 * 53 + 5, N=900, K=300, sched=True, regimes=("odd tiles per CTA",)),
    dict(id="pp_M64x26x40p33", M=64 * 26 * 40 + 33, N=900, K=300, sched=True, regimes=("even tiles per CTA", "resident >= 6 stages")),
    dict(id="N400_K300_slice144", M=4000, N=400, K=300, sched=True, regimes=("slices > 1", "slice width % 32 != 0")),
    dict(id="N256_K1000_5stages", M=4000, N=256, K=1000, regimes=("resident < 6 stages",)),
    dict(id="N64_K4000_streamed", M=64 * 70 + 3, N=64, K=4000, regimes=("streamed weights", "1 slice")),
    dict(id="N300_K2000_streamed", M=4000, N=300, K=2000, sched=True, regimes=("streamed weights", "slices > 1")),
    dict(id="N257_K65", M=4000, N=257, K=65, regimes=("slices > 1", "slice width % 32 != 0")),
    dict(id="N256_K63_relu", M=3000, N=256, K=63, relu=1, regimes=("1 slice",)),
    dict(id="K1_nobias", M=1000, N=128, K=1, bias=False, regimes=("1 slice",)),
    dict(id="f32_N301_K1000", M=777, N=301, K=1000, out_bf16=0, regimes=("slices > 1", "resident < 6 stages")),
    dict(id="f32_N33_nobias", M=64 * 41, N=33, K=300, out_bf16=0, bias=False, regimes=("slice width % 32 != 0",)),
    dict(id="rpt1", M=300, N=96, K=64, rpt=1, regimes=("rows_per_tile < 64",)),
    dict(id="rpt50_relu", M=1000, N=200, K=300, rpt=50, relu=1, regimes=("rows_per_tile < 64",)),
    dict(id="rpt60_N900", M=999, N=900, K=300, rpt=60, regimes=("rows_per_tile < 64", "slices > 1")),
    dict(id="conv_T20", n_seg=37, T=20, N=300, K=300, taps=3, relu=1, regimes=("taps 3", "slices > 1")),
    dict(id="conv_T30_streamed", n_seg=20, T=30, N=400, K=900, taps=3, relu=1, regimes=("taps 3", "streamed weights")),
    dict(id="conv_T50", n_seg=11, T=50, N=400, K=300, taps=3, regimes=("taps 3",)),
]

# nr_gemm_tn: D[Ma][Nb] += A[Kr][Ma]^T . B[rows + shift][b_col0 + n].  reserve: nr_reserve_sms_for_comm ("all" = every SM,
# which the GEMM clamps to half of them).  b_cols: columns of B that exist (default b_col0 + Nb).  odd_d: odd ldd and D one
# float past an aligned base (the scalar red path).
GEMM_TN_CASES = [
    dict(id="Kr1_Ma900_Nb512", Kr=1, Ma=900, Nb=512, regimes=("single k-range", "cluster 2x2", "NT 256", "n_tiles 2")),
    dict(id="Kr63_Ma1_Nb50", Kr=63, Ma=1, Nb=50, regimes=("cluster 1x1", "NT 64", "single k-range")),
    dict(id="Kr64_Ma64_Nb100_s1", Kr=64, Ma=64, Nb=100, shift=1, regimes=("NT 128", "single k-range")),
    dict(id="Kr65_Ma65_Nb150", Kr=65, Ma=65, Nb=150, regimes=("NT 192", "cluster 1x1")),
    dict(id="Kr1000_Ma129_Nb256_sm3", Kr=1000, Ma=129, Nb=256, shift=-3, regimes=("cluster 2x1", "NT 256")),
    dict(id="Kr1000_Ma300_Nb257_s3", Kr=1000, Ma=300, Nb=257, shift=3, regimes=("cluster 1x2", "n_tiles 2", "NT 192")),
    dict(id="Kr44813_Ma900_Nb301_sm1", Kr=64 * 700 + 13, Ma=900, Nb=301, shift=-1, regimes=("cluster 2x2", "NT 192")),
    dict(id="second_launch_col512", Kr=1000, Ma=300, Nb=389, b_col0=512, b_cols=901, regimes=("cluster 1x2", "n_tiles 2")),
    dict(id="odd_ldd", Kr=1000, Ma=300, Nb=301, odd_d=True, regimes=("cluster 1x2",)),
    dict(id="reserve0", Kr=64 * 700 + 13, Ma=300, Nb=100, reserve=0, regimes=("cluster 1x1", "NT 128")),
    dict(id="reserve32", Kr=64 * 700 + 13, Ma=300, Nb=100, reserve=32, regimes=("cluster 1x1",)),
    dict(id="reserve_all", Kr=64 * 700 + 13, Ma=300, Nb=100, reserve="all", regimes=("cluster 1x1",)),
]

# nr_additive_attention_fwd[_hilo]: n_seg segments of seg rows, X [rows][D], Wa [q][D].  scores: "unit" (random), "peaked"
# (scores spread over +-100: exp overflows fp32 without the max subtraction), "tied" (the rows of a segment are equal, so
# its weights are uniform).  ldo: output pitch (default: D rounded up to 4, plus 4).
POOL_CASES = [
    dict(id="S20_D300_partial", n_seg=37, seg=20, D=300, q=200, regimes=("rows_per_tile < 64", "slice width % 32 != 0")),
    dict(id="S20_D300_news", n_seg=3000, seg=20, D=300, q=200, scores="peaked", regimes=("rows_per_tile < 64",)),
    dict(id="S50_D400_streamed", n_seg=100, seg=50, D=400, q=200, regimes=("streamed weights", "rows_per_tile < 64")),
    dict(id="S50_D400_hilo", n_seg=64, seg=50, D=400, q=200, hilo=True, regimes=("streamed weights",)),
    dict(id="S1_D2_q1", n_seg=1000, seg=1, D=2, q=1, regimes=("N < 32", "resident >= 6 stages")),
    dict(id="S2_D8_q16", n_seg=777, seg=2, D=8, q=16, regimes=("N < 32",)),
    dict(id="S3_D296_q24_many", n_seg=5000, seg=3, D=296, q=24, regimes=("N < 32", "rows_per_tile < 64", "even tiles per CTA")),
    dict(id="S4_D298_q100_ldo2", n_seg=3000, seg=4, D=298, q=100, ldo=298, regimes=("slice width % 32 != 0",)),
    dict(id="S30_D64_q256", n_seg=50, seg=30, D=64, q=256, regimes=("rows_per_tile < 64", "warpgroup 1 idle")),
    dict(id="S32_D300_hilo", n_seg=300, seg=32, D=300, q=200, hilo=True, regimes=("1 slice",)),
    dict(id="S33_D300_one_seg_peaked", n_seg=1, seg=33, D=300, q=200, scores="peaked", regimes=("rows_per_tile < 64",)),
    dict(id="S63_D300_tied", n_seg=200, seg=63, D=300, q=200, scores="tied", regimes=("rows_per_tile < 64",)),
    dict(id="S64_D300_peaked_nowout", n_seg=150, seg=64, D=300, q=200, scores="peaked", w_out=False, regimes=("1 slice",)),
    dict(id="S20_D300_tied_hilo_ldo2", n_seg=500, seg=20, D=300, q=200, scores="tied", hilo=True, ldo=302,
         regimes=("rows_per_tile < 64",)),
]


def linear_shape(c):
    """(M, rows_per_tile, w_tap_rows) nr_linear runs a LINEAR_CASES entry with."""
    taps = c.get("taps", 1)
    M = c["n_seg"] * (c["T"] + 2) if taps > 1 else c["M"]
    return M, c.get("rpt", 64), (c["N"] if taps > 1 else 0)

# nr_additive_attention_bwd (tests/test_gpu_additive_bwd_elements.py): n_seg segments of seg rows, X [rows][D], Wa [q][D]; w
# comes from the forward on the same operands (hilo: from nr_additive_attention_fwd_hilo).  scores as in POOL_CASES.  ldo: dout
# pitch (default: D rounded up to 4, plus 4); ld_dx: dX pitch (default ldx = round_up(D + 1, 8)).  The regimes are those of
# gemm_plan_ref.regimes_bwd: BWD_REGIMES plus the NT_REGIMES of the dPre and dX plans, prefixed "dPre " and "dX ".
POOL_BWD_CASES = [
    dict(id="bwd_S1_D300", n_seg=1000, seg=1, D=300, q=200,
         regimes=("dscore warp", "dPre TMA", "dX fragment view", "dX slice capped by dOut staging", "dX slices > 1")),
    dict(id="bwd_S2_D300", n_seg=777, seg=2, D=300, q=200, regimes=("dX slice capped by dOut staging", "dX slices > 1")),
    dict(id="bwd_S3_D300", n_seg=2000, seg=3, D=300, q=200, regimes=("dX slice capped by dOut staging",)),
    dict(id="bwd_S4_D400_view_fusion", n_seg=1000, seg=4, D=400, q=200,
         regimes=("dX slice capped by dOut staging", "dPre streamed weights", "dX slice width % 32 != 0")),
    dict(id="bwd_S20_D300_news_peaked", n_seg=3000, seg=20, D=300, q=200, scores="peaked", regimes=("dscore warp", "dX slices > 1")),
    dict(id="bwd_S50_D300_user", n_seg=512, seg=50, D=300, q=200, regimes=("dscore block",)),
    dict(id="bwd_S32_D300", n_seg=300, seg=32, D=300, q=200, regimes=("dscore warp",)),
    dict(id="bwd_S33_D300", n_seg=300, seg=33, D=300, q=200, regimes=("dscore block",)),
    dict(id="bwd_S64_D300_tied", n_seg=100, seg=64, D=300, q=200, scores="tied", regimes=("dscore block",)),
    dict(id="bwd_S20_D604", n_seg=100, seg=20, D=604, q=200,
         regimes=("dscore block D>512", "weight grad 2 launches", "dPre streamed weights")),
    dict(id="bwd_S20_D24_q16", n_seg=500, seg=20, D=24, q=16, regimes=("dX row view", "dPre plain stores", "dX N < 32", "dPre N < 32")),
    dict(id="bwd_S30_D64_q256", n_seg=50, seg=30, D=64, q=256, regimes=("dPre TMA", "dX 1 slice")),
    dict(id="bwd_S3_D296_q24_many", n_seg=5000, seg=3, D=296, q=24, regimes=("dPre plain stores", "dX slices > 1")),
    dict(id="bwd_S20_D300_one_tile", n_seg=1, seg=20, D=300, q=200, regimes=("dPre warpgroup 1 idle", "dX warpgroup 1 idle")),
    dict(id="bwd_S20_D300_pitches", n_seg=37, seg=20, D=300, q=200, ldo=312, ld_dx=320, regimes=("dX fragment view",)),
    dict(id="bwd_S50_D400_hilo", n_seg=64, seg=50, D=400, q=200, hilo=True, regimes=("dscore block", "dPre streamed weights")),
]

# gemm_store through nr_debug_gemm_store (tests/test_gpu_gemm_store.py): every option of the store epilogue on the paths a
# 32-column chunk can leave by.  M rows of A (rm: n_seg segments of the map's seg_in rows, M = n_seg * seg_in), N x K weights,
# taps at tap_origin (-1: centred), rows_per_tile rpt.  Options: relu / tanh / dtanh (1 - t^2 from a bf16 source of pitch
# ld_out + 8, or dtanh_ld, starting dtanh_off elements into its buffer), p (dropout), rm = (seg_in, in_off, seg_len, seg_out, out_off), ones (column N = 1, zeros up to ones_upto, default
# ld_out), lo_col0 (low plane, pitch ld_lo, default N - lo_col0 rounded up to 8, plus 8), acc (fp32 +=), out_off (the output
# starts out_off elements into its buffer, as the KCNN entity section at X2 + sec), bias (default on), out_bf16 (default 1),
# ld_out (default: bf16 round_up(N + 1, 8), fp32 round_up(N, 4) + 4).  Labels: the options it sets (gemm_plan_ref.STORE_OPTIONS,
# checked against the configuration), the NT regimes of its plan and its store paths: gemm_plan_ref.store_paths' output paths,
# and its low-plane paths prefixed "lo ".
_T20_TO_PADDED = (20, 0, 20, 22, 1)   # compact title rows -> the zero-padded CNN layout (pad rows 0 and 21 are not written)
_T22_TO_COMPACT = (22, 1, 20, 20, 0)  # the CNN conv's map: padded rows 1..20 of a title -> compact rows 0..19
STORE_CASES = [
    # slice edges
    dict(id="N400_slice144_relu", M=4000, N=400, K=300, relu=1, options=("relu",),
         regimes=("slices > 1", "slice width % 32 != 0"), paths=("TMA", "cut chunk")),
    dict(id="M1_N900_tanh", M=1, N=900, K=300, tanh=1, options=("tanh",), regimes=("slices > 1", "warpgroup 1 idle"),
         paths=("TMA", "cut chunk")),
    dict(id="M63_N20_relu", M=63, N=20, K=300, relu=1, options=("relu",), regimes=("N < 32", "1 slice"), paths=("cut chunk",)),
    dict(id="rpt1_N96_relu_drop2", M=300, N=96, K=64, rpt=1, relu=1, p=0.2, options=("relu", "dropout"),
         regimes=("rows_per_tile < 64",), paths=("row pieces",)),
    dict(id="rpt50_N201_dtanh", M=1000, N=201, K=300, rpt=50, dtanh=1, options=("dtanh",), regimes=("rows_per_tile < 64", "slices > 1"),
         paths=("row pieces", "cut chunk")),
    dict(id="f32_N301_relu_drop5", M=777, N=301, K=300, out_bf16=0, relu=1, p=0.5, options=("relu", "dropout"),
         regimes=("slices > 1",), paths=("fp32 pairs", "fp32 scalar")),
    dict(id="f32_N33_tanh", M=64 * 41, N=33, K=300, out_bf16=0, tanh=1, options=("tanh",), regimes=("slice width % 32 != 0",),
         paths=("fp32 pairs", "fp32 scalar")),
    dict(id="f32_N99_dtanh", M=1000, N=99, K=300, out_bf16=0, dtanh=1, options=("dtanh",), regimes=("1 slice",),
         paths=("fp32 pairs", "fp32 scalar")),
    dict(id="N300_dtanh_drop5", M=4000, N=300, K=300, dtanh=1, p=0.5, options=("dtanh", "dropout"), regimes=("slices > 1",),
         paths=("TMA", "cut chunk")),
    dict(id="N257_tanh_rpt60", M=999, N=257, K=65, rpt=60, tanh=1, options=("tanh",), regimes=("rows_per_tile < 64", "slices > 1"),
         paths=("row pieces", "cut chunk")),
    # += (the second pass of a split operand): the odd fp32 tail of every slice leaves as one scalar
    dict(id="f32_acc_N301", M=777, N=301, K=1000, out_bf16=0, acc=1, options=("+=",), regimes=("resident < 6 stages",),
         paths=("fp32 pairs", "fp32 scalar")),
    # row maps
    dict(id="map_to_padded_drop2", n_seg=150, rm=_T20_TO_PADDED, N=400, K=300, p=0.2, options=("row map", "dropout"),
         regimes=("slices > 1",), paths=("row pieces", "cut chunk")),
    dict(id="map_f32_N151_drop5", n_seg=97, rm=_T20_TO_PADDED, N=151, K=300, out_bf16=0, p=0.5, relu=1,
         options=("row map", "dropout", "relu"), regimes=("1 slice",), paths=("fp32 pairs", "fp32 scalar")),
    dict(id="map_window_L17_tanh_f32", n_seg=100, rm=(20, 0, 17, 17, 0), N=64, K=100, out_bf16=0, tanh=1,
         options=("row map", "tanh"), regimes=("1 slice",), paths=("fp32 pairs",)),
    dict(id="map_window_L17_dtanh", n_seg=100, rm=(20, 0, 17, 17, 0), N=100, K=100, dtanh=1, options=("row map", "dtanh"),
         regimes=("1 slice",), paths=("row pieces", "cut chunk")),
    # conv taps at both ends of the window: tap rows before row 0 and past row M - 1 read zeros
    dict(id="taps2_origin0_N300", M=1000, N=300, K=300, taps=2, tap_origin=0, options=("taps",), regimes=("slices > 1",),
         paths=("TMA", "cut chunk")),
    dict(id="taps2_origin1_f32_N151_drop2", M=1000, N=151, K=300, taps=2, tap_origin=1, out_bf16=0, p=0.2,
         options=("taps", "dropout"), regimes=("slices > 1",), paths=("fp32 pairs", "fp32 scalar")),
    dict(id="taps4_origin0_rpt50_relu", M=1000, N=100, K=200, taps=4, tap_origin=0, rpt=50, relu=1, options=("taps", "relu"),
         regimes=("rows_per_tile < 64",), paths=("row pieces", "cut chunk")),
    dict(id="taps4_origin3_f32_tanh", M=333, N=77, K=100, taps=4, tap_origin=3, out_bf16=0, tanh=1, options=("taps", "tanh"),
         regimes=("1 slice",), paths=("fp32 pairs", "fp32 scalar")),
    dict(id="taps2_origin1_f32_dtanh", M=500, N=65, K=100, taps=2, tap_origin=1, out_bf16=0, dtanh=1, options=("taps", "dtanh"),
         regimes=("1 slice",), paths=("fp32 pairs", "fp32 scalar")),
    dict(id="taps3_f32_relu_acc", M=700, N=45, K=300, taps=3, out_bf16=0, relu=1, acc=1, options=("taps", "relu", "+="),
         regimes=("taps 3",), paths=("fp32 pairs", "fp32 scalar")),
    # ones column
    dict(id="ones_N300_tma", M=1000, N=300, K=100, ones=1, options=("ones column",), regimes=("slices > 1",),
         paths=("TMA", "cut chunk")),
    dict(id="ones_N20_upto_pitch", M=200, N=20, K=100, ones=1, relu=1, options=("ones column", "relu"), regimes=("N < 32",),
         paths=("cut chunk",)),
    dict(id="ones_rpt60_N64", M=999, N=64, K=100, rpt=60, ones=1, ones_upto=68, options=("ones column",),
         regimes=("rows_per_tile < 64",), paths=("row pieces",)),
    # low plane
    dict(id="lo_col0_0_N400", M=4000, N=400, K=300, lo_col0=0, options=("low plane",), regimes=("slices > 1",),
         paths=("TMA", "cut chunk", "lo TMA", "lo cut chunk")),
    dict(id="lo_slice1_chunk_N400_drop2", M=4000, N=400, K=300, lo_col0=176, p=0.2, options=("low plane", "dropout"),
         regimes=("slice width % 32 != 0",), paths=("TMA", "cut chunk", "lo TMA", "lo cut chunk")),
    dict(id="lo_rpt50_N200_relu", M=1000, N=200, K=300, rpt=50, lo_col0=64, relu=1, options=("low plane", "relu"),
         regimes=("rows_per_tile < 64",), paths=("row pieces", "cut chunk", "lo row pieces", "lo cut chunk")),
    dict(id="lo_N20_tanh", M=500, N=20, K=100, lo_col0=0, tanh=1, options=("low plane", "tanh"), regimes=("N < 32",),
         paths=("cut chunk", "lo cut chunk")),
    # the production configurations, as their callers pass them
    dict(id="cnn_conv_T20_F400", n_seg=613, rm=_T22_TO_COMPACT, N=400, K=300, taps=3, tap_origin=1, relu=1, p=0.2, ones=1,
         lo_col0=0, ld_lo=408, options=("taps", "row map", "relu", "dropout", "ones column", "low plane"),
         regimes=("taps 3", "slices > 1"),
         paths=("row pieces", "cut chunk", "lo row pieces", "lo cut chunk")),
    dict(id="kcnn_entity_tanh_X2_sec", M=500 * 20, N=300, K=100, tanh=1, ld_out=608, out_off=304, ones=1, ones_upto=304,
         options=("tanh", "ones column"), regimes=("slices > 1",), paths=("TMA", "cut chunk")),
    dict(id="kcnn_tconv_dtanh_taps4", M=500 * 20, N=300, K=416, lda=416, taps=4, tap_origin=3, bias=False, dtanh=1, ld_out=304,
         dtanh_ld=608, dtanh_off=304, options=("taps", "dtanh"), regimes=("slices > 1", "streamed weights"), paths=("TMA", "cut chunk")),
    dict(id="gru_x_lo_acc_N2700", M=37 * 50, N=2700, K=900, out_bf16=0, acc=1, bias=False, ld_out=2700, options=("+=",),
         regimes=("slices > 1",), paths=("fp32 pairs",)),
    dict(id="qkv_v_lo_h15", M=613 * 20, N=912, K=300, ld_out=912, lo_col0=608, ld_lo=304, options=("low plane",),
         regimes=("slices > 1",), paths=("TMA", "cut chunk", "lo TMA", "lo cut chunk")),
]


def store_setup(c):
    """The nr_debug_gemm_store configuration of a STORE_CASES entry: M, rows_per_tile, w_tap_rows, the output rows (the map's
    n_seg * seg_out, else M), ld_out, the ones column (-1 off) and its limit, the low plane's lo_col0 (None off) and ld_lo."""
    N, out_bf16, taps = c["N"], c.get("out_bf16", 1), c.get("taps", 1)
    rm = c.get("rm")
    M = c["n_seg"] * rm[0] if rm else c["M"]
    out_rows = c["n_seg"] * rm[3] if rm else M
    ld_out = c.get("ld_out", (N + 8) // 8 * 8 if out_bf16 else (N + 3) // 4 * 4 + 4)
    lo_col0 = c.get("lo_col0")
    ld_lo = c.get("ld_lo", (N - lo_col0 + 7) // 8 * 8 + 8) if lo_col0 is not None else 0
    return dict(M=M, rpt=c.get("rpt", 64), w_tap_rows=N if taps > 1 else 0, out_rows=out_rows, ld_out=ld_out,
                ones_col=N if c.get("ones") else -1, ones_upto=c.get("ones_upto", ld_out) if c.get("ones") else 0,
                lo_col0=lo_col0, ld_lo=ld_lo, rm=rm or (0, 0, 0, 0, 0))


def store_options(c):
    """The STORE_OPTIONS a STORE_CASES entry's configuration sets."""
    on = {"relu": c.get("relu"), "tanh": c.get("tanh"), "dtanh": c.get("dtanh"), "dropout": c.get("p", 0) > 0, "row map": c.get("rm"),
          "ones column": c.get("ones"), "low plane": c.get("lo_col0") is not None, "+=": c.get("acc"), "taps": c.get("taps", 1) > 1}
    return {k for k, v in on.items() if v}
