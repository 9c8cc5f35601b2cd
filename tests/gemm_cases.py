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
