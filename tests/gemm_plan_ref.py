"""Plain-Python restatement of the wgmma GEMM planners (importable without CUDA).

plan_nt restates plan_gemm_nt (csrc/gemm.cu) line for line and adds the tiles each (CTA, consumer warpgroup) processes under
gemm_nt_kernel's schedule; plan_tn restates gemm_tn_accumulate and launch_gemm_tn_kernel; plan_pool_bwd restates the kernel
choices of the additive-attention backward's four launches.  The GPU tests label every case
with the regime it is there to reach (regimes_nt / regimes_tn), tests/test_gemm_plan_host.py checks those labels here, and
tests/test_gpu_gemm_elements.py ties this restatement to the real planner through the kernel's per-CTA counters."""
from __future__ import annotations

# csrc/nr_gemm.cuh
kSmemLimit = 232448            # kSmemLimit: 227 KB of dynamic shared memory per CTA
kTileM = 64                    # kTileM: rows per gemm_nt tile (one m64 wgmma)
kChunkK = 64                   # kChunkK: bf16 elements per 128-byte swizzle row
kAStageBytes = kTileM * 128    # kAStageBytes: one 64 x 64 bf16 A box, 8 KB
kMaxStages = 12                # kMaxStages
# kEpiSmemBytes<Epi> = Epi::kScratchBytes (+ kXposeBytes for a row-view epilogue), csrc/nr_epilogues.cuh
kXposeBytes = 2 * 2 * kTileM * 16 * 4                  # kXposeBytes (row view: 2 warpgroups x 2 column halves)
EPI_STORE_SMEM = 1024 + (8 * 6 * 16 * 64 + 1024)       # EpiStore (fragment view): 1 KB bias + FragStore<6> = 51,200 B
EPI_POOL_SMEM = 4096 + kXposeBytes                     # EpiPool (row view): 4 KB scratch + transpose = 20,480 B
assert EPI_STORE_SMEM == 51200 and EPI_POOL_SMEM == 20480
# the pooling backward's epilogues
kStageFloats = 1536                                    # DOutStage::kStageFloats: staged dOut floats per buffer
DOUT_STAGE_SMEM = 4 * kStageFloats * 4                 # DOutStage: 2 buffers per warpgroup = 24,576 B
kTileStoreBytes = 8 * 2 * 2048 + 1024                  # kTileStoreBytes (nr_gemm.cuh): 2 staging tiles per epilogue warp
EPI_DPRE_SMEM = 3072 + (8 * 4 * 16 * 64 + 1024)        # EpiDPre (fragment view): 3 KB + FragStore<4> = 36,864 B
EPI_DPOOLIN_FRAG_SMEM = DOUT_STAGE_SMEM + (8 * 6 * 16 * 64 + 1024)   # EpiDPoolInFrag: dOut stage + FragStore<6> = 74,752 B
EPI_DPOOLIN_SMEM = DOUT_STAGE_SMEM + kTileStoreBytes + kXposeBytes   # EpiDPoolIn (row view) + transpose = 74,752 B
assert EPI_DPRE_SMEM == 36864 and EPI_DPOOLIN_FRAG_SMEM == 74752 and EPI_DPOOLIN_SMEM == 74752

H100_SMS = 132                 # H100 SXM5; the GPU tests plan with the device's own count (nr_num_sms)


def _cdiv(a, b):
    return -(-a // b)


def _round_up(a, b):
    return _cdiv(a, b) * b


def plan_nt(M, N, K, taps=1, rows_per_tile=kTileM, sms=H100_SMS, epi_smem_bytes=EPI_STORE_SMEM, max_slices=0, max_stride=0):
    """plan_gemm_nt: the weight slicing, ring and grid, plus wg_tiles[b][w] = the tiles warpgroup w of CTA b processes
    (CTA b takes slice b % n_slices and tiles b // n_slices + k * step, step = grid // n_slices; its warpgroup w takes every
    second one of those, starting at the w-th)."""
    assert M >= 0 and N >= 1 and K >= 1 and 1 <= taps <= 4 and 1 <= rows_per_tile <= kTileM and sms > 0
    num_m_tiles = _cdiv(M, rows_per_tile)
    k_chunks = _cdiv(K, kChunkK)
    fixed = 1024 + _round_up(epi_smem_bytes, 16) + 512
    slices, b_stream, bbytes = 1, 0, 0
    while True:
        assert slices <= 64, "cannot fit weight slice"
        n_stride = _round_up(_cdiv(N, slices), 16)
        n_box = _round_up(min(n_stride, N), 32)
        if n_box > 256 or (max_stride > 0 and n_stride > max_stride):
            slices += 1
            continue
        bbytes = taps * k_chunks * n_box * 128
        if bbytes + 6 * kAStageBytes + fixed <= kSmemLimit:
            break
        if slices == max_slices or n_box <= 64:
            if bbytes + 4 * kAStageBytes + fixed > kSmemLimit:
                b_stream, bbytes = 1, 0
            break
        slices += 1
    n_slices = _cdiv(N, n_stride)
    stage_bytes = kAStageBytes + (n_box * 128 if b_stream else 0)
    stages = min(kMaxStages, (kSmemLimit - fixed - bbytes) // stage_bytes)
    assert stages >= 2
    groups = max(1, min(sms // n_slices, num_m_tiles))
    grid = groups * n_slices
    step = grid // n_slices
    wg_tiles = []
    for b in range(grid):
        t0 = b // n_slices
        mine = list(range(t0, num_m_tiles, step))
        wg_tiles.append((mine[0::2], mine[1::2]))
    return {"n_stride": n_stride, "n_box": n_box, "n_slices": n_slices, "b_stream": b_stream, "stages": stages, "grid": grid,
            "num_m_tiles": num_m_tiles, "k_chunks": k_chunks, "slice_of": [b % n_slices for b in range(grid)], "wg_tiles": wg_tiles,
            "N": N, "taps": taps, "rows_per_tile": rows_per_tile}


def plan_pool(M, D, q, seg_len, sms=H100_SMS):
    """gemm_additive_pool's plan: pre = X . Wa^T with N = q, K = D, tiles of whole segments, one weight slice."""
    return plan_nt(M, q, D, 1, (kTileM // seg_len) * seg_len, sms, EPI_POOL_SMEM, max_slices=1)


def pool_dinput_max_stride(seg_len):
    """gemm_pool_dinput's cap on the slice width: the dOut rows of every segment a 64-row tile touches (<= 64 / seg_len + 2)
    must fit one DOutStage buffer."""
    return (kStageFloats // (kTileM // seg_len + 2)) & ~15


def plan_pool_bwd(n_seg, seg_len, D, q, sms=H100_SMS):
    """nr_additive_attention_bwd's four launches (csrc/abi.cu):
      dscore   pool_dscore: the warp kernel when seg_len <= 32 and D <= 512, else the block kernel
      dpre     gemm_additive_dpre: pre = X . Wa^T (N = q, K = D) in one weight slice; dPre leaves by TMA when q >= 32,
               by plain stores otherwise
      dx       gemm_pool_dinput: dPre . Wa (N = D, K = q), the slice width capped by the dOut staging; the fragment-view
               EpiDPoolInFrag when D >= 32, the row-view EpiDPoolIn otherwise
      wgrad    gemm_weight_grad: [dWa | dba] over the D + 1 columns of X (its ones column), one gemm_tn per 512 columns"""
    M = n_seg * seg_len
    frag = D >= 32
    smem = EPI_DPOOLIN_FRAG_SMEM if frag else EPI_DPOOLIN_SMEM
    dx = plan_nt(M, D, q, 1, kTileM, sms, smem, max_stride=pool_dinput_max_stride(seg_len))
    wgrad = [plan_tn(M, q, min(512, D + 1 - c0), sms) for c0 in range(0, D + 1, 512)]
    return {"dscore": "warp" if seg_len <= 32 and D <= 512 else "block",
            "dpre": plan_nt(M, q, D, 1, kTileM, sms, EPI_DPRE_SMEM, max_slices=1), "dpre_tma": q >= 32,
            "dx": dx, "dx_frag": frag, "dx_uncapped_stride": plan_nt(M, D, q, 1, kTileM, sms, smem)["n_stride"], "wgrad": wgrad,
            "D": D}


def plan_tn(Kr, Ma, Nb, sms=H100_SMS, reserved=0):
    """gemm_tn_accumulate: tiles, columns per CTA (NT), cluster shape and k_slices_max, an upper bound on the k-ranges.  With a
    cluster the launch further caps k_slices by cudaOccupancyMaxActiveClusters, which only the device can answer, so the
    exact count is known only there; without one k_slices_max is exact."""
    assert 1 <= Nb <= 512 and Ma >= 1 and Kr >= 1
    sms_eff = max(sms // 2, sms - max(0, reserved))
    m_tiles = _cdiv(Ma, 128)
    n_tiles = _cdiv(Nb, 256)
    nt = _round_up(_cdiv(Nb, n_tiles), 64)
    total_chunks = _cdiv(Kr, 64)
    cluster = (2 if m_tiles % 2 == 0 else 1, 2 if n_tiles % 2 == 0 else 1)
    k = max(1, min(sms_eff // (m_tiles * n_tiles), total_chunks))
    cps = _cdiv(total_chunks, k)
    return {"m_tiles": m_tiles, "n_tiles": n_tiles, "NT": nt, "cluster": cluster, "total_chunks": total_chunks,
            "k_slices_max": _cdiv(total_chunks, cps), "exact": cluster == (1, 1)}


# ------------------------------------------------------------------------------------------------
# regimes: the labels the GPU case tables carry
# ------------------------------------------------------------------------------------------------
NT_REGIMES = ("1 slice", "slices > 1", "slice width % 32 != 0", "N < 32", "resident >= 6 stages", "resident < 6 stages",
              "streamed weights", "taps 3", "rows_per_tile < 64", "warpgroup 1 idle", "odd tiles per CTA", "even tiles per CTA")
TN_REGIMES = ("cluster 1x1", "cluster 2x1", "cluster 1x2", "cluster 2x2", "NT 64", "NT 128", "NT 192", "NT 256", "n_tiles 2",
              "single k-range")
# how a 32-column chunk of gemm_store's output leaves EpiStore::frag (and the options of its configuration)
STORE_PATHS = ("TMA", "row pieces", "cut chunk", "fp32 pairs", "fp32 scalar")
STORE_OPTIONS = ("relu", "tanh", "dtanh", "dropout", "row map", "ones column", "low plane", "+=", "taps")
BWD_REGIMES = ("dscore warp", "dscore block", "dscore block D>512", "dPre TMA", "dPre plain stores", "dX fragment view",
               "dX row view", "dX slice capped by dOut staging", "dX slices > 1", "weight grad 2 launches")


def regimes_nt(p):
    """Every regime of NT_REGIMES a gemm_nt plan is in."""
    r = {"1 slice" if p["n_slices"] == 1 else "slices > 1"}
    if p["n_stride"] % 32 != 0:
        r.add("slice width % 32 != 0")
    if p["N"] < 32:
        r.add("N < 32")
    if p["b_stream"]:
        r.add("streamed weights")
    else:
        r.add("resident >= 6 stages" if p["stages"] >= 6 else "resident < 6 stages")
    if p["taps"] == 3:
        r.add("taps 3")
    if p["rows_per_tile"] < kTileM:
        r.add("rows_per_tile < 64")
    for w0, w1 in p["wg_tiles"]:
        if w0 and not w1:
            r.add("warpgroup 1 idle")
        if w0:
            r.add("odd tiles per CTA" if (len(w0) + len(w1)) % 2 else "even tiles per CTA")
    return r


def regimes_tn(p):
    """Every regime of TN_REGIMES a gemm_tn plan is in ("single k-range": the reduction has one 64-row chunk, so no launch
    can split it, whatever the cluster occupancy)."""
    r = {"cluster %dx%d" % p["cluster"], "NT %d" % p["NT"]}
    if p["n_tiles"] == 2:
        r.add("n_tiles 2")
    if p["total_chunks"] == 1:
        r.add("single k-range")
    return r


def regimes_bwd(p):
    """Every regime of BWD_REGIMES a backward plan (plan_pool_bwd) is in, plus the NT_REGIMES of its two gemm_nt plans
    prefixed "dPre " and "dX " ("dX slice capped by dOut staging": the staging cap, not the 256-column box limit, sets the
    slice width)."""
    r = {"dscore " + p["dscore"], "dPre TMA" if p["dpre_tma"] else "dPre plain stores",
         "dX fragment view" if p["dx_frag"] else "dX row view"}
    if p["dscore"] == "block" and p["D"] > 512:
        r.add("dscore block D>512")
    dx = p["dx"]
    if dx["n_slices"] > 1:
        r.add("dX slices > 1")
    if dx["n_stride"] < p["dx_uncapped_stride"]:
        r.add("dX slice capped by dOut staging")
    if len(p["wgrad"]) == 2:
        r.add("weight grad 2 launches")
    r |= {"dPre " + x for x in regimes_nt(p["dpre"])} | {"dX " + x for x in regimes_nt(dx)}
    return r


def store_use_tma(N, out_bf16, row_map, rows_per_tile):
    """gemm_store's use_tma: bf16 chunks leave through the tensor maps for identity rows, whole 64-row tiles and N >= 32."""
    return bool(out_bf16) and not row_map and min(rows_per_tile, kTileM) == kTileM and N >= 32


def store_paths(plan, out_bf16, row_map=False, lo_col0=None):
    """The paths of STORE_PATHS the chunks of every slice take in EpiStore::frag, as (output paths, low-plane paths).  A bf16
    chunk at slice column lc0 is cut (predicated fragment stores) when lc0 + 32 > the slice's columns, else it leaves by TMA
    (use_tma) or as 16-byte row pieces; fp32 leaves as column pairs (lc + 1 < ncols) and, where a slice has an odd column
    count, one scalar.  The low plane takes the bf16 rule for the chunks at or past lo_col0 (None: no low plane)."""
    tma = store_use_tma(plan["N"], out_bf16, row_map, plan["rows_per_tile"])
    out, lo = set(), set()
    for sl in range(plan["n_slices"]):
        col0 = sl * plan["n_stride"]
        ncols = min(plan["n_stride"], plan["N"] - col0)
        for lc0 in range(0, ncols, 32):
            if not out_bf16:
                if ncols - lc0 >= 2:
                    out.add("fp32 pairs")
                if ncols % 2 and lc0 + 32 >= ncols:
                    out.add("fp32 scalar")
                continue
            path = "cut chunk" if lc0 + 32 > ncols else ("TMA" if tma else "row pieces")
            out.add(path)
            if lo_col0 is not None and col0 + lc0 >= lo_col0:
                lo.add(path)
    return out, lo


def lo_chunk_aligned(plan, lo_col0):
    """lo_plane_chunk_aligned (csrc/gemm.cu): no 32-column chunk of a weight slice straddles lo_col0."""
    s = plan["n_stride"]
    return all(not (c0 < lo_col0 < c0 + s and (lo_col0 - c0) % 32) for c0 in range(0, plan["n_slices"] * s, s))


def lo_supported(N, K, lo_col0):
    """gemm_store_lo_supported: the low plane of the columns [lo_col0, N) of an N x K product is chunk aligned under the
    weight slicing of plan_nt (which depends on N and K only)."""
    return 0 <= lo_col0 < N and lo_chunk_aligned(plan_nt(0, N, K), lo_col0)


def store_accepts(option, path):
    """Whether gemm_store takes an option of STORE_OPTIONS on an output path of STORE_PATHS (for "low plane": a path of the
    plane itself).  A row map leaves without TMA; the ones column and the low plane need a bf16 output, += an fp32 one."""
    bf16 = path in ("TMA", "row pieces", "cut chunk")
    if option == "row map":
        return path != "TMA"
    if option in ("ones column", "low plane"):
        return bf16
    if option == "+=":
        return not bf16
    return True
