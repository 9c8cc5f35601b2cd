// Title-level multi-head self-attention, backward and forward (reference src/model/general/attention/multihead_self.py:15-23,
// the backward through autograd) for the news encoder's shape: T = 20 words, d_k = 20, up to 15 heads.
//
//   dA = dCtx V^T;  dS = A (dA - sum A dA)/sqrt(dk);  dQ = dS K;  dK = dS^T Q;  dV = A^T dCtx        (A recomputed from Q, K)
//
// Why a second kernel next to attn.cu: the head-level kernel there moves every 20 x 20 head tile with 8-byte cp.async
// pieces (a 40-byte head row has no 16-byte phase) and is bound by the LSU data pipe -- 418 shared-memory wavefronts per
// head, a third of them the asynchronous copies themselves.  Here a CTA owns
// WHOLE TITLES: one TMA box brings the 20 full Q|K|V rows of a title (all heads, contiguous, sector aligned), a second one
// the 20 dCtx rows, and one TMA store writes the 20 dQ|dK|dV rows back.  Warp h owns head h.  No copy instruction touches
// the LSU pipe; what is left are the ldmatrix fragment loads and a 2.3 KB per-warp scratch for A / dS (126 wavefronts).
//
// The 16-byte phase: with Q | K | V sections at columns 0, sec, 2*sec (sec % 8 == 0, nr_ops.h) head h starts 40*h bytes into
// its section in all four operands: 16-byte aligned for even h, 8 bytes off for odd h.  ldmatrix needs aligned 16-byte row
// pieces, so a head's 20 columns are covered by three aligned 8-column groups starting at gb = 40h - 8*(h & 1):
//     even h:  [0,16) as one k16 step, [16,24) as a k8 step whose columns 20..23 belong to head h+1
//     odd  h:  [-4,4) as a k8 step whose columns -4..-1 belong to head h-1, [4,20) as one k16 step
// Foreign columns are zeroed in the fragment registers (select, so that NaN payloads cannot leak) when they are a
// contraction index and simply not stored when they are an output column.  Every Q|K|V row address goes through a per-lane
// row map (row_offsets): the identity, or over the live tokens' compact rows a title's rank map with the dead rows (and rows
// 20..23) pointed at a bias row in shared memory.  Rows 20..23 of a tile in token order (k8 steps over the title
// rows) are whatever follows the tile in shared memory: the matching fragment lanes are zeroed the same way.
//
// Shared-memory row pitches are (odd multiple of 16) bytes: eight consecutive rows start in eight distinct bank quads, so
// every ldmatrix phase is conflict free; the TMA boxes are simply declared wider than the rows (zero filled / dropped).
#include <algorithm>

#define NR_WATCHDOG_SYMBOL g_attn_dev_error
#include "nr_fused.cuh"
#include "nr_mma.cuh"
#include "nr_ops.h"

namespace nr {

int read_topk_device_error(int* out4);
int read_attn_device_error(int* out4) {
    const int rc = static_cast<int>(cudaMemcpyFromSymbol(out4, fused::g_attn_dev_error, sizeof(int) * 4));
    if (rc != 0 || out4[0] != 0) return rc;
    return read_topk_device_error(out4);  // the top-k kernel keeps its own record (topk.cu)
}

namespace title {

using namespace fused;
using namespace mma;

constexpr int kT = 20;           // words per title
constexpr int kDk = 20;          // head width
constexpr int kMaxHeads = 15;    // compute warps per CTA (+ 1 TMA warp = 512 threads)
constexpr int kIn = 2;           // titles in flight (input stages)
constexpr int kOut = 2;          // result tiles (a TMA store drains one while the warps fill the other)
constexpr int kInHilo = 2;       // input stages of the hi/lo forward variant (a third one measured 3 % slower: the variant is MMA / issue bound)
constexpr int kScrPitch = 48;    // bytes per scratch row: 24 bf16 key columns
constexpr int kScrTile = 24 * kScrPitch;
constexpr int kScrWarp = 2 * kScrTile;  // A | dS of one head

// Shared-memory offsets, from a stage's Q|K|V (or V low plane) tile, of the tile rows lane & 7, 8 + (lane & 7) and
// 16 + (lane & 7): every ldmatrix row address of a lane is one of them.  Token order (mask null): the rows themselves.
// Compact rows (LiveTokens; the tile holds the rows from the title's first compact row on): a live token's rank among the
// title's live tokens, and for a dead token and the rows 20..23 the CTA's copy of the bias row, `to_bias` from the tile.
__device__ __forceinline__ void row_offsets(const uint32_t* mask, int title, uint32_t pitch, uint32_t to_bias, int lane, uint32_t ro[3]) {
    const uint32_t m = mask != nullptr ? __ldg(mask + title) : 0u;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const uint32_t r = 8u * j + static_cast<uint32_t>(lane & 7);
        const bool live = r < kT && ((m >> r) & 1u);
        ro[j] = mask == nullptr ? r * pitch : live ? static_cast<uint32_t>(__popc(m & ((1u << r) - 1u))) * pitch : to_bias;
    }
}
// the bias row (row_bytes) into shared memory, zeros up to pitch bytes; every thread of the block takes part
__device__ __forceinline__ void copy_bias_row(uint8_t* dst, const void* src, uint32_t row_bytes, uint32_t pitch) {
    for (uint32_t i = threadIdx.x; i < pitch / 16u; i += blockDim.x)
        reinterpret_cast<uint4*>(dst)[i] = i < row_bytes / 16u ? __ldg(static_cast<const uint4*>(src) + i) : make_uint4(0, 0, 0, 0);
}

struct Params {
    int n_seq, heads;
    uint32_t sec2;        // section stride in bytes
    uint32_t pq, pc;      // shared-memory row pitch of the Q|K|V tile / the dCtx tile (bytes)
    uint32_t qkv_tile;    // bytes reserved for the Q|K|V tile of a stage (128-byte multiple)
    uint32_t in_stage;    // qkv_tile + dCtx tile
    uint32_t out_stage;   // == qkv_tile
    uint32_t tx;          // bytes one stage's two boxes deliver
    float rs, sc;         // 1/sqrt(dk), log2(e)/sqrt(dk)
    const unsigned char* pad;  // LiveTokens::pad or null
    // with live tokens (mask non-null): title s stores its live rows at rows offset[s] .. of dqkv (pitch ld_out bytes, row_bytes
    // each), and the dead rows' bf16 dQ|dK|dV go into dbias[c * ld_dbias]
    const uint32_t* mask;
    const int* offset;
    char* dqkv;
    uint32_t ld_out, row_bytes;
    float* dbias;
    int ld_dbias;
    // compact (the compact forward's Q|K|V): title s reads its rows from compact row offset[s] on through the row map of
    // row_offsets, a dead token the bias row (LiveTokens::qkv), kept in shared memory behind the barriers
    int compact;
    const void* bias;
};

__device__ __forceinline__ uint32_t sel(bool keep, uint32_t v) { return keep ? v : 0u; }

__global__ void __launch_bounds__((kMaxHeads + 1) * 32, 1)
mhsa_title_bwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_dc,
                      const __grid_constant__ CUtensorMap tm_out, const __grid_constant__ CUtensorMap tm_pad, const Params p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    uint8_t* const base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const uint32_t in_base = base, out_base = base + kIn * p.in_stage, scr_base = out_base + kOut * p.out_stage;
    const uint32_t bar_off = kIn * p.in_stage + kOut * p.out_stage + p.heads * kScrWarp;
    uint64_t* const bars = reinterpret_cast<uint64_t*>(base_ptr + bar_off);
    uint64_t* const full = bars;                 // [kIn]   TMA -> warps
    uint64_t* const empty = bars + kIn;          // [kIn]   warps -> TMA (stage consumed)
    uint64_t* const ofull = bars + 2 * kIn;      // [kOut]  warps -> TMA (results written)
    uint64_t* const oempty = bars + 2 * kIn + kOut;  // [kOut]  TMA -> warps (store has drained the tile)

    // every byte a fragment load can touch is initialised: slack rows / padding columns read finite zeros before the first TMA
    for (uint32_t i = tid; i < bar_off / 16; i += blockDim.x) reinterpret_cast<uint4*>(base_ptr)[i] = make_uint4(0, 0, 0, 0);
    const uint32_t bias_off = bar_off + 128u;
    if (p.compact) copy_bias_row(base_ptr + bias_off, p.bias, 3u * p.sec2, p.pq);
    if (tid == 0) {
        for (int i = 0; i < kIn; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], p.heads);
        }
        for (int i = 0; i < kOut; ++i) {
            mbar_init(&ofull[i], p.heads);
            mbar_init(&oempty[i], 1);
        }
        fence_barrier_init();
    }
    fence_proxy_async();  // the zero fill above is ordered before any TMA write to the same bytes
    __syncthreads();

    const int n_my = (p.n_seq - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);

    if (warp == p.heads) {
        // ---------------- TMA warp: loads two titles ahead, stores each finished tile ----------------
        if (lane == 0) {
            tma_prefetch_desc(&tm_qkv);
            tma_prefetch_desc(&tm_dc);
            tma_prefetch_desc(&tm_out);
            if (p.pad != nullptr) tma_prefetch_desc(&tm_pad);
            auto load = [&](int it) {
                const int s = it % kIn;
                const int title = static_cast<int>(blockIdx.x) + it * static_cast<int>(gridDim.x), row = title * kT;
                const bool pad = p.pad != nullptr && p.pad[title] != 0;  // a padding title reads the shared bias tile
                const bool none = pad && p.compact;                      // compact: its rows are all the bias row
                mbar_arrive_expect_tx(&full[s], none ? p.tx - kT * p.pq : p.tx);
                if (!none) tma_load_2d(base_ptr + s * p.in_stage, pad ? &tm_pad : &tm_qkv, &full[s], 0, pad ? 0 : p.compact ? p.offset[title] : row);
                tma_load_2d(base_ptr + s * p.in_stage + p.qkv_tile, &tm_dc, &full[s], 0, row);
            };
            for (int it = 0; it < kIn && it < n_my; ++it) load(it);
            for (int j = 0; j < n_my; ++j) {
                const int o = j % kOut;
                const int title = static_cast<int>(blockIdx.x) + j * static_cast<int>(gridDim.x);
                const uint32_t tile = out_base + o * p.out_stage;
                uint32_t live = 0;
                char* dst = nullptr;
                if (p.mask != nullptr) {
                    live = p.mask[title];
                    dst = p.dqkv + static_cast<size_t>(p.offset[title]) * p.ld_out;
                }
                f_wait(&ofull[o], (j / kOut) & 1, 70);
                if (p.mask == nullptr) {
                    tma_store_2d(&tm_out, tile, 0, title * kT);
                } else {  // the live rows, one bulk copy each, to consecutive compact rows
                    for (; live != 0; live &= live - 1, dst += p.ld_out) bulk_store_1d(dst, tile + (__ffs(live) - 1) * p.pq, p.row_bytes);
                }
                bulk_commit();
                if (j + kIn < n_my) {
                    f_wait(&empty[j % kIn], (j / kIn) & 1, 71);
                    load(j + kIn);
                }
                bulk_wait_read<0>();
                mbar_arrive(&oempty[o]);
            }
            bulk_wait_all();
        }
        return;
    }

    // ---------------- compute warps: warp h owns head h of every title of this CTA ----------------
    const int h = warp;
    const bool odd = (h & 1) != 0;
    const uint32_t gb = 40u * h - (odd ? 8u : 0u);  // first aligned 8-column group of the head (bytes into the section)
    const uint32_t k16b = gb + (odd ? 16u : 0u);    // the 16-column contraction step
    const uint32_t k8b = gb + (odd ? 0u : 32u);     // the 8-column contraction step (4 live + 4 foreign columns)
    const bool v8 = odd ? (t4 >= 2) : (t4 < 2);     // this lane's two columns of the 8-column step are the head's own
    const bool c0ok = !odd || t4 >= 2;              // output columns of group 0 / group 2 that belong to the head
    const bool c2ok = odd || t4 < 2;
    const bool lo2 = t4 < 2;                        // key columns 16 + 2*t4 (+1) < 20; also: rows 16 + 2*t4 (+1) < 20
    const uint32_t pq = p.pq, pc = p.pc;
    const uint32_t r15c = (lane & 15) * pc, r7c = (lane & 7) * pc;
    const uint32_t hi = (lane >> 4) * 16u, mid = ((lane >> 3) & 1) * 16u;
    const uint32_t ps = scr_base + h * kScrWarp, dsb = ps + kScrTile;  // A | dS scratch of this head
    const uint32_t at0 = ((lane & 7) + (lane >> 4) * 8) * kScrPitch + mid;  // x4.trans, key rows 0..15 as m
    const uint32_t at8 = (16 + (lane & 7)) * kScrPitch;                      // rows 16..23 (the k8 step over query rows)
    const uint32_t at1 = (lane & 15) * kScrPitch + 32u;                      // x2.trans, key rows 16..23 as m
    const uint32_t st_scr = g * kScrPitch + t4 * 4u;
    const float rs = p.rs, sc = p.sc;
    // the dead rows' dQ | dK | dV as stored (bf16), per section, column group and column of the pair: the bias-column term
    float dsum[3][3][2] = {};
    const auto add_dead = [](float* acc, uint32_t packed) {
        const float2 v = unpack_bf16x2(packed);
        acc[0] += v.x;
        acc[1] += v.y;
    };

    for (int it = 0; it < n_my; ++it) {
        const int s = it % kIn, o = it % kOut;
        const uint32_t Q = in_base + s * p.in_stage, K = Q + p.sec2, V = K + p.sec2, G = Q + p.qkv_tile;
        const uint32_t ob = out_base + o * p.out_stage;
        const int title = static_cast<int>(blockIdx.x) + it * static_cast<int>(gridDim.x);
        const uint32_t dead = p.mask != nullptr ? ~__ldg(p.mask + title) : 0u;
        uint32_t ro[3];  // Q|K|V rows lane & 7 (+ 8, + 16) of the tile
        row_offsets(p.compact ? p.mask : nullptr, title, pq, base + bias_off - Q, lane, ro);
        const uint32_t r15 = (lane & 8) ? ro[1] : ro[0];
        f_wait(&full[s], (it / kIn) & 1, 72);

        // ---- phase A (query rows i): A, dS -> scratch; dQ -> result tile ----
        uint32_t kb16[3][2], kb8[3], vb16[3][2], vb8[3], kt16[3][2], kt8[3];
#pragma unroll
        for (int nt = 0; nt < 3; ++nt) {
            lds_x2(kb16[nt], K + k16b + ro[nt] + mid);
            lds_x2(vb16[nt], V + k16b + ro[nt] + mid);
            lds_x1(&kb8[nt], K + k8b + ro[nt]);
            lds_x1(&vb8[nt], V + k8b + ro[nt]);
            kb8[nt] = sel(v8, kb8[nt]);
            vb8[nt] = sel(v8, vb8[nt]);
            lds_x2_t(kt16[nt], K + gb + 16 * nt + r15);
            lds_x1_t(&kt8[nt], K + gb + 16 * nt + ro[2]);
            kt8[nt] = sel(lo2, kt8[nt]);
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            uint32_t aq[4], ag[4], aq8[2], ag8[2];
            if (mt == 0) {
                lds_x4(aq, Q + k16b + r15 + hi);
                lds_x4(ag, G + k16b + r15c + hi);
                lds_x2(aq8, Q + k8b + r15);
                lds_x2(ag8, G + k8b + r15c);
            } else {  // rows 16..23 only: the second half of this row block is dead
                uint32_t t[2];
                lds_x2(t, Q + k16b + ro[2] + mid);
                aq[0] = t[0], aq[1] = 0u, aq[2] = t[1], aq[3] = 0u;
                lds_x2(t, G + k16b + 16 * pc + r7c + mid);
                ag[0] = t[0], ag[1] = 0u, ag[2] = t[1], ag[3] = 0u;
                lds_x1(&aq8[0], Q + k8b + ro[2]);
                lds_x1(&ag8[0], G + k8b + 16 * pc + r7c);
                aq8[1] = ag8[1] = 0u;
            }
            aq8[0] = sel(v8, aq8[0]), aq8[1] = sel(v8, aq8[1]);
            ag8[0] = sel(v8, ag8[0]), ag8[1] = sel(v8, ag8[1]);
            float sm[3][4], dp[3][4];
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                mma_bf16_z(sm[nt], aq, kb16[nt]);   // S  = Q K^T
                mma_bf16_k8(sm[nt], aq8, &kb8[nt]);
                mma_bf16_z(dp[nt], ag, vb16[nt]);   // dA = dCtx V^T
                mma_bf16_k8(dp[nt], ag8, &vb8[nt]);
            }
            // softmax over the 20 live key columns (fp32, exp(S)/(sum exp(S) + 1e-8) in its stable form), then dS
            const bool row0 = mt == 0 || g < 4;  // rows 16 + g < 20
            constexpr float kNegInf = -__builtin_huge_valf();
            float m0 = kNegInf, m1 = kNegInf;
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                const bool ok = nt < 2 || lo2;
#pragma unroll
                for (int e = 0; e < 4; ++e) sm[nt][e] = ok ? sm[nt][e] : kNegInf;
                m0 = fmaxf(m0, fmaxf(sm[nt][0], sm[nt][1]));
                if (mt == 0) m1 = fmaxf(m1, fmaxf(sm[nt][2], sm[nt][3]));
            }
            m0 = quad_max(m0) * sc;
            if (mt == 0) m1 = quad_max(m1) * sc;
            float l0 = 0.f, l1 = 0.f;
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    sm[nt][e] = exp2f(fmaf(sm[nt][e], sc, -m0));
                    l0 += sm[nt][e];
                    if (mt == 0) {
                        sm[nt][2 + e] = exp2f(fmaf(sm[nt][2 + e], sc, -m1));
                        l1 += sm[nt][2 + e];
                    }
                }
            }
            l0 = quad_sum(l0);
            const float i0 = 1.f / (l0 + 1e-8f * exp2f(-m0));
            float i1 = 0.f;
            if (mt == 0) {
                l1 = quad_sum(l1);
                i1 = 1.f / (l1 + 1e-8f * exp2f(-m1));
            }
            float del0 = 0.f, del1 = 0.f;
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                const bool ok = nt < 2 || lo2;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    sm[nt][e] = (ok && row0) ? sm[nt][e] * i0 : 0.f;
                    del0 += ok ? sm[nt][e] * dp[nt][e] : 0.f;
                    if (mt == 0) {
                        sm[nt][2 + e] = ok ? sm[nt][2 + e] * i1 : 0.f;
                        del1 += ok ? sm[nt][2 + e] * dp[nt][2 + e] : 0.f;
                    } else {
                        sm[nt][2 + e] = 0.f;
                    }
                }
            }
            del0 = quad_sum(del0);
            if (mt == 0) del1 = quad_sum(del1);
            uint32_t a16[4], a8[2];
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                const bool ok = nt < 2 || lo2;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    dp[nt][e] = (ok && row0) ? sm[nt][e] * (dp[nt][e] - del0) * rs : 0.f;
                    dp[nt][2 + e] = (mt == 0 && ok) ? sm[nt][2 + e] * (dp[nt][2 + e] - del1) * rs : 0.f;
                }
                const uint32_t p01 = pack_bf16x2(sm[nt][0], sm[nt][1]), d01 = pack_bf16x2(dp[nt][0], dp[nt][1]);
                const uint32_t p23 = pack_bf16x2(sm[nt][2], sm[nt][3]), d23 = pack_bf16x2(dp[nt][2], dp[nt][3]);
                const uint32_t so = st_scr + mt * 16 * kScrPitch + nt * 16;
                sts32(ps + so, p01);   // rows 20..23 are written as zeros: they are contraction indices of phase B
                sts32(dsb + so, d01);
                if (mt == 0) {
                    sts32(ps + so + 8 * kScrPitch, p23);
                    sts32(dsb + so + 8 * kScrPitch, d23);
                }
                if (nt == 0) a16[0] = d01, a16[1] = d23;
                if (nt == 1) a16[2] = d01, a16[3] = d23;
                if (nt == 2) a8[0] = d01, a8[1] = d23;
            }
            // dQ = dS K  (A = dS straight from the registers)
            if (mt == 0 && it >= kOut) f_wait(&oempty[o], ((it / kOut) - 1) & 1, 73);  // the store of title it-2 has drained this tile
#pragma unroll
            for (int nd = 0; nd < 3; ++nd) {
                float dq[4];
                mma_bf16_z(dq, a16, kt16[nd]);
                mma_bf16_k8(dq, a8, &kt8[nd]);
                const bool cok = nd == 1 || (nd == 0 ? c0ok : c2ok);
                const uint32_t oa = ob + (mt * 16 + g) * pq + gb + 16 * nd + 4 * t4;
                if (cok && row0) {
                    const uint32_t v = pack_bf16x2(dq[0], dq[1]);
                    sts32(oa, v);
                    if ((dead >> (mt * 16 + g)) & 1u) add_dead(dsum[0][nd], v);
                }
                if (mt == 0 && cok) {
                    const uint32_t v = pack_bf16x2(dq[2], dq[3]);
                    sts32(oa + 8 * pq, v);
                    if ((dead >> (8 + g)) & 1u) add_dead(dsum[0][nd], v);
                }
            }
        }
        __syncwarp();
        // ---- phase B (key rows j): dK = dS^T Q, dV = A^T dCtx ----
        uint32_t qt16[3][2], qt8[3], gt16[3][2], gt8[3];
#pragma unroll
        for (int nd = 0; nd < 3; ++nd) {
            lds_x2_t(qt16[nd], Q + gb + 16 * nd + r15);
            lds_x2_t(gt16[nd], G + gb + 16 * nd + r15c);
            lds_x1_t(&qt8[nd], Q + gb + 16 * nd + ro[2]);
            lds_x1_t(&gt8[nd], G + gb + 16 * nd + 16 * pc + r7c);
            qt8[nd] = sel(lo2, qt8[nd]);
            gt8[nd] = sel(lo2, gt8[nd]);
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            uint32_t ad[4], ap[4], ad8[2], ap8[2];
            if (mt == 0) {
                lds_x4_t(ad, dsb + at0);
                lds_x4_t(ap, ps + at0);
                lds_x2_t(ad8, dsb + at8 + mid);
                lds_x2_t(ap8, ps + at8 + mid);
            } else {
                uint32_t t[2];
                lds_x2_t(t, dsb + at1);
                ad[0] = t[0], ad[1] = 0u, ad[2] = t[1], ad[3] = 0u;
                lds_x2_t(t, ps + at1);
                ap[0] = t[0], ap[1] = 0u, ap[2] = t[1], ap[3] = 0u;
                lds_x1_t(&ad8[0], dsb + at8 + 32u);
                lds_x1_t(&ap8[0], ps + at8 + 32u);
                ad8[1] = ap8[1] = 0u;
            }
            const bool row0 = mt == 0 || g < 4;
#pragma unroll
            for (int nd = 0; nd < 3; ++nd) {
                float dk[4], dv[4];
                mma_bf16_z(dk, ad, qt16[nd]);
                mma_bf16_k8(dk, ad8, &qt8[nd]);
                mma_bf16_z(dv, ap, gt16[nd]);
                mma_bf16_k8(dv, ap8, &gt8[nd]);
                const bool cok = nd == 1 || (nd == 0 ? c0ok : c2ok);
                const uint32_t oa = ob + p.sec2 + (mt * 16 + g) * pq + gb + 16 * nd + 4 * t4;
                if (cok && row0) {
                    const uint32_t k = pack_bf16x2(dk[0], dk[1]), v = pack_bf16x2(dv[0], dv[1]);
                    sts32(oa, k);
                    sts32(oa + p.sec2, v);
                    if ((dead >> (mt * 16 + g)) & 1u) add_dead(dsum[1][nd], k), add_dead(dsum[2][nd], v);
                }
                if (mt == 0 && cok) {
                    const uint32_t k = pack_bf16x2(dk[2], dk[3]), v = pack_bf16x2(dv[2], dv[3]);
                    sts32(oa + 8 * pq, k);
                    sts32(oa + p.sec2 + 8 * pq, v);
                    if ((dead >> (8 + g)) & 1u) add_dead(dsum[1][nd], k), add_dead(dsum[2][nd], v);
                }
            }
        }
        fence_proxy_async();  // the result tile is read by the TMA store (async proxy)
        __syncwarp();
        if (lane == 0) {
            mbar_arrive(&empty[s]);
            mbar_arrive(&ofull[o]);
        }
    }
    if (p.mask != nullptr) {  // one add per column and CTA: the column sums over the warp's eight row groups g
        const int sec = static_cast<int>(p.sec2 / 2u);
#pragma unroll
        for (int nd = 0; nd < 3; ++nd) {
            const bool cok = nd == 1 || (nd == 0 ? c0ok : c2ok);
            const int col = static_cast<int>(gb / 2u) + 8 * nd + 2 * t4;
#pragma unroll
            for (int sct = 0; sct < 3; ++sct) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float v = dsum[sct][nd][e];
                    v += __shfl_xor_sync(0xffffffffu, v, 4);
                    v += __shfl_xor_sync(0xffffffffu, v, 8);
                    v += __shfl_xor_sync(0xffffffffu, v, 16);
                    if (g == 0 && cok) red_add_f32(p.dbias + static_cast<size_t>(sct * sec + col + e) * p.ld_dbias, v);
                }
            }
        }
    }
}


// ------------------------------------------------------------------------------------------------------------------------
// forward:  S = QK^T/sqrt(dk);  A = exp(S)/(sum exp(S) + 1e-8);  ctx = dropout(A V)      (same CTA / warp decomposition)
// Two CTAs per SM (64 registers): a stage is only the Q|K|V tile, the result tile is the 20 context rows (ones column at d
// and the zero tail are constants of the tile, written once).
// HILO (the accurate mode, DESIGN.md section 4): V arrives as a hi/lo bf16 pair (second TMA box: the low plane the projection
// GEMM wrote), the probabilities are split into a hi/lo pair in registers, ctx = A_hi V_hi + A_lo V_hi + A_hi V_lo in fp32 and
// leaves as a hi/lo pair of planes -- the three bf16 roundings that put the plain path 6e-3 from the fp32 result (V 3.6e-3,
// context 1.9e-3, probabilities 1.1e-3 on the golden case) drop to ~1e-5 each.  One CTA per SM (149 KB of tiles).
// ------------------------------------------------------------------------------------------------------------------------
struct FwdParams {
    int n_seq, heads, ld_ctx;
    uint32_t sec2, pq, pc, pv, qkv_tile, in_stage, out_tile, out_stage, tx;
    float sc;
    Dropout drop;
    const unsigned char* pad;  // PaddingTitles::pad or null
    // compact rows (LiveTokens) or null: title s reads its rows from compact row offset[s] on through the row map of
    // row_offsets (mask[s] == 0: no load at all), a dead token the bias rows bias_q / bias_v, kept in shared memory
    const uint32_t* mask;
    const int* offset;
    const void *bias_q, *bias_v;
};

template <bool HILO>
__global__ void __launch_bounds__((kMaxHeads + 1) * 32, HILO ? 1 : 2)
mhsa_title_fwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_vlo,
                      const __grid_constant__ CUtensorMap tm_ctx, const __grid_constant__ CUtensorMap tm_clo,
                      const __grid_constant__ CUtensorMap tm_pad, const __grid_constant__ CUtensorMap tm_padlo, const FwdParams p) {
    constexpr int kIn = HILO ? kInHilo : title::kIn;  // input stages (one CTA per SM in the hi/lo variant, two otherwise)
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 127u) & ~127u;
    uint8_t* const base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const uint32_t in_base = base, out_base = base + kIn * p.in_stage;
    const uint32_t bar_off = kIn * p.in_stage + kOut * p.out_stage;
    uint64_t* const bars = reinterpret_cast<uint64_t*>(base_ptr + bar_off);
    uint64_t* const full = bars;
    uint64_t* const empty = bars + kIn;
    uint64_t* const ofull = bars + 2 * kIn;
    uint64_t* const oempty = bars + 2 * kIn + kOut;
    for (uint32_t i = tid; i < bar_off / 16; i += blockDim.x) reinterpret_cast<uint4*>(base_ptr)[i] = make_uint4(0, 0, 0, 0);
    const uint32_t bias_q = bar_off + 128u, bias_v = bias_q + p.pq;  // the bias rows behind the barriers
    if (p.mask != nullptr) {
        copy_bias_row(base_ptr + bias_q, p.bias_q, 3u * p.sec2, p.pq);
        if (HILO) copy_bias_row(base_ptr + bias_v, p.bias_v, p.sec2, p.pv);
    }
    __syncthreads();
    if (tid < kOut * kT)  // the ones column of the context rows (bias trick of the pooling GEMM); hi plane only
        *reinterpret_cast<__nv_bfloat16*>(base_ptr + kIn * p.in_stage + (tid / kT) * p.out_stage + (tid % kT) * p.pc + p.heads * kDk * 2) =
            __float2bfloat16_rn(1.0f);
    if (tid == 0) {
        for (int i = 0; i < kIn; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], p.heads);
        }
        for (int i = 0; i < kOut; ++i) {
            mbar_init(&ofull[i], p.heads);
            mbar_init(&oempty[i], 1);
        }
        fence_barrier_init();
    }
    fence_proxy_async();
    __syncthreads();
    const int n_my = (p.n_seq - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);

    if (warp == p.heads) {
        if (lane == 0) {
            tma_prefetch_desc(&tm_qkv);
            tma_prefetch_desc(&tm_ctx);
            if (HILO) {
                tma_prefetch_desc(&tm_vlo);
                tma_prefetch_desc(&tm_clo);
            }
            if (p.pad != nullptr) {
                tma_prefetch_desc(&tm_pad);
                if (HILO) tma_prefetch_desc(&tm_padlo);
            }
            auto load = [&](int it) {
                const int s = it % kIn;
                const int title = static_cast<int>(blockIdx.x) + it * static_cast<int>(gridDim.x);
                const bool pad = p.pad != nullptr && p.pad[title] != 0;  // a padding title reads the shared bias tile
                if (p.mask != nullptr && p.mask[title] == 0) {          // compact: its rows are all the bias rows
                    mbar_arrive(&full[s]);
                    return;
                }
                const int row = pad ? 0 : p.mask != nullptr ? p.offset[title] : title * kT;
                mbar_arrive_expect_tx(&full[s], p.tx);
                tma_load_2d(base_ptr + s * p.in_stage, pad ? &tm_pad : &tm_qkv, &full[s], 0, row);
                if (HILO) tma_load_2d(base_ptr + s * p.in_stage + p.qkv_tile, pad ? &tm_padlo : &tm_vlo, &full[s], 0, row);
            };
            for (int it = 0; it < kIn && it < n_my; ++it) load(it);
            for (int j = 0; j < n_my; ++j) {
                const int o = j % kOut;
                const int row = (static_cast<int>(blockIdx.x) + j * static_cast<int>(gridDim.x)) * kT;
                f_wait(&ofull[o], (j / kOut) & 1, 80);
                tma_store_2d(&tm_ctx, base_ptr + kIn * p.in_stage + o * p.out_stage, 0, row);
                if (HILO) tma_store_2d(&tm_clo, base_ptr + kIn * p.in_stage + o * p.out_stage + p.out_tile, 0, row);
                bulk_commit();
                if (j + kIn < n_my) {
                    f_wait(&empty[j % kIn], (j / kIn) & 1, 81);
                    load(j + kIn);
                }
                bulk_wait_read<0>();
                mbar_arrive(&oempty[o]);
            }
            bulk_wait_all();
        }
        return;
    }

    const int h = warp;
    const bool odd = (h & 1) != 0;
    const uint32_t gb = 40u * h - (odd ? 8u : 0u);
    const uint32_t k16b = gb + (odd ? 16u : 0u), k8b = gb + (odd ? 0u : 32u);
    const bool v8 = odd ? (t4 >= 2) : (t4 < 2);
    const bool c0ok = !odd || t4 >= 2, c2ok = odd || t4 < 2, lo2 = t4 < 2;
    const uint32_t pq = p.pq, pc = p.pc, pv = p.pv;
    const uint32_t hi = (lane >> 4) * 16u, mid = ((lane >> 3) & 1) * 16u;
    const float sc = p.sc;

    for (int it = 0; it < n_my; ++it) {
        const int s = it % kIn, o = it % kOut;
        const uint32_t Q = in_base + s * p.in_stage, K = Q + p.sec2, V = K + p.sec2, VL = Q + p.qkv_tile;
        const uint32_t ob = out_base + o * p.out_stage;
        const int title = static_cast<int>(blockIdx.x) + it * static_cast<int>(gridDim.x);
        const long long row_base = static_cast<long long>(title) * kT;
        uint32_t ro[3], rv[3];  // rows lane & 7 (+ 8, + 16) of the Q|K|V tile and of the V low-plane tile
        row_offsets(p.mask, title, pq, base + bias_q - Q, lane, ro);
        if (HILO) row_offsets(p.mask, title, pv, base + bias_v - VL, lane, rv);
        const uint32_t r15 = (lane & 8) ? ro[1] : ro[0];
        f_wait(&full[s], (it / kIn) & 1, 82);
        uint32_t kb16[3][2], kb8[3], vt16[3][2], vt8[3], vl16[HILO ? 3 : 1][2], vl8[HILO ? 3 : 1];
#pragma unroll
        for (int nt = 0; nt < 3; ++nt) {
            lds_x2(kb16[nt], K + k16b + ro[nt] + mid);
            lds_x1(&kb8[nt], K + k8b + ro[nt]);
            kb8[nt] = sel(v8, kb8[nt]);
            lds_x2_t(vt16[nt], V + gb + 16 * nt + r15);
            lds_x1_t(&vt8[nt], V + gb + 16 * nt + ro[2]);
            vt8[nt] = sel(lo2, vt8[nt]);
            if (HILO) {
                lds_x2_t(vl16[nt], VL + gb + 16 * nt + ((lane & 8) ? rv[1] : rv[0]));
                lds_x1_t(&vl8[nt], VL + gb + 16 * nt + rv[2]);
                vl8[nt] = sel(lo2, vl8[nt]);
            }
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            uint32_t aq[4], aq8[2];
            if (mt == 0) {
                lds_x4(aq, Q + k16b + r15 + hi);
                lds_x2(aq8, Q + k8b + r15);
            } else {
                uint32_t t[2];
                lds_x2(t, Q + k16b + ro[2] + mid);
                aq[0] = t[0], aq[1] = 0u, aq[2] = t[1], aq[3] = 0u;
                lds_x1(&aq8[0], Q + k8b + ro[2]);
                aq8[1] = 0u;
            }
            aq8[0] = sel(v8, aq8[0]), aq8[1] = sel(v8, aq8[1]);
            float sm[3][4];
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                mma_bf16_z(sm[nt], aq, kb16[nt]);
                mma_bf16_k8(sm[nt], aq8, &kb8[nt]);
            }
            const bool row0 = mt == 0 || g < 4;
            constexpr float kNegInf = -__builtin_huge_valf();
            float m0 = kNegInf, m1 = kNegInf;
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                const bool ok = nt < 2 || lo2;
#pragma unroll
                for (int e = 0; e < 4; ++e) sm[nt][e] = ok ? sm[nt][e] : kNegInf;
                m0 = fmaxf(m0, fmaxf(sm[nt][0], sm[nt][1]));
                if (mt == 0) m1 = fmaxf(m1, fmaxf(sm[nt][2], sm[nt][3]));
            }
            m0 = quad_max(m0) * sc;
            if (mt == 0) m1 = quad_max(m1) * sc;
            float l0 = 0.f, l1 = 0.f;
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    sm[nt][e] = exp2f(fmaf(sm[nt][e], sc, -m0));
                    l0 += sm[nt][e];
                    if (mt == 0) {
                        sm[nt][2 + e] = exp2f(fmaf(sm[nt][2 + e], sc, -m1));
                        l1 += sm[nt][2 + e];
                    }
                }
            }
            l0 = quad_sum(l0);
            const float i0 = 1.f / (l0 + 1e-8f * exp2f(-m0));
            float i1 = 0.f;
            if (mt == 0) {
                l1 = quad_sum(l1);
                i1 = 1.f / (l1 + 1e-8f * exp2f(-m1));
            }
            uint32_t a16[4], a8[2], b16[HILO ? 4 : 1], b8[HILO ? 2 : 1];  // probabilities: hi plane, (HILO) lo plane
#pragma unroll
            for (int nt = 0; nt < 3; ++nt) {
                const bool ok = nt < 2 || lo2;
                const float q0 = (ok && row0) ? sm[nt][0] * i0 : 0.f, q1 = (ok && row0) ? sm[nt][1] * i0 : 0.f;
                const float q2 = (mt == 0 && ok) ? sm[nt][2] * i1 : 0.f, q3 = (mt == 0 && ok) ? sm[nt][3] * i1 : 0.f;
                const uint32_t p01 = pack_bf16x2(q0, q1), p23 = pack_bf16x2(q2, q3);
                if (nt == 0) a16[0] = p01, a16[1] = p23;
                if (nt == 1) a16[2] = p01, a16[3] = p23;
                if (nt == 2) a8[0] = p01, a8[1] = p23;
                if (HILO) {
                    const float2 h01 = unpack_bf16x2(p01), h23 = unpack_bf16x2(p23);
                    const uint32_t l01 = pack_bf16x2(q0 - h01.x, q1 - h01.y), l23 = pack_bf16x2(q2 - h23.x, q3 - h23.y);
                    if (nt == 0) b16[0] = l01, b16[1] = l23;
                    if (nt == 1) b16[2] = l01, b16[3] = l23;
                    if (nt == 2) b8[0] = l01, b8[1] = l23;
                }
            }
            if (mt == 0 && it >= kOut) f_wait(&oempty[o], ((it / kOut) - 1) & 1, 83);
#pragma unroll
            for (int nd = 0; nd < 3; ++nd) {
                float c[4];
                if (HILO) {  // small terms first
                    mma_bf16_z(c, b16, vt16[nd]);
                    mma_bf16_k8(c, b8, &vt8[nd]);
                    mma_bf16(c, a16, vl16[nd]);
                    mma_bf16_k8(c, a8, &vl8[nd]);
                    mma_bf16(c, a16, vt16[nd]);
                } else {
                    mma_bf16_z(c, a16, vt16[nd]);
                }
                mma_bf16_k8(c, a8, &vt8[nd]);
                const bool cok = nd == 1 || (nd == 0 ? c0ok : c2ok);
                const uint32_t oa = ob + (mt * 16 + g) * pc + gb + 16 * nd + 4 * t4;
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    if (hf == 1 && mt == 1) continue;
                    if (cok && (hf == 1 || row0)) {
                        const uint32_t hv = pack_bf16x2(c[2 * hf], c[2 * hf + 1]);
                        sts32(oa + hf * 8 * pc, hv);
                        if (HILO) {
                            const float2 hf2 = unpack_bf16x2(hv);
                            sts32(oa + p.out_tile + hf * 8 * pc, pack_bf16x2(c[2 * hf] - hf2.x, c[2 * hf + 1] - hf2.y));
                        }
                    }
                }
            }
        }
        if (p.drop.active()) {
            // dropout acts on the context (multihead_self.py:23 -> news_encoder.py:43): second pass over the head's 20 x 20 block in
            // 8-byte pieces, ONE counter hash per 4 aligned columns (hashing per fragment pair in the loop above costs 3x the
            // hashes and made the kernel issue bound)
            __syncwarp();
            const uint64_t gbase = (static_cast<uint64_t>(row_base) * p.ld_ctx + 20u * h) >> 2;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t i = lane + 32 * k;
                if (i < kT * 5) {
                    const uint32_t r = (i * 205u) >> 10, c4 = i - 5u * r;  // i / 5 for i < 128
                    const uint32_t a = ob + r * pc + 40u * h + 8u * c4;
                    uint32_t u0, u1;
                    asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(u0), "=r"(u1) : "r"(a));
                    float m[4];
                    p.drop.mask4_group(gbase + r * (static_cast<uint32_t>(p.ld_ctx) >> 2) + c4, m);
                    float2 x = unpack_bf16x2(u0), y = unpack_bf16x2(u1);
                    if (HILO) {
                        uint32_t w0, w1;
                        asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(w0), "=r"(w1) : "r"(a + p.out_tile));
                        const float2 xl = unpack_bf16x2(w0), yl = unpack_bf16x2(w1);
                        x.x = (x.x + xl.x) * m[0], x.y = (x.y + xl.y) * m[1], y.x = (y.x + yl.x) * m[2], y.y = (y.y + yl.y) * m[3];
                        const uint32_t h0 = pack_bf16x2(x.x, x.y), h1 = pack_bf16x2(y.x, y.y);
                        const float2 hx = unpack_bf16x2(h0), hy = unpack_bf16x2(h1);
                        asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(a), "r"(h0), "r"(h1) : "memory");
                        asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(a + p.out_tile), "r"(pack_bf16x2(x.x - hx.x, x.y - hx.y)),
                                     "r"(pack_bf16x2(y.x - hy.x, y.y - hy.y)) : "memory");
                    } else {
                        x.x *= m[0], x.y *= m[1], y.x *= m[2], y.y *= m[3];
                        asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(a), "r"(pack_bf16x2(x.x, x.y)), "r"(pack_bf16x2(y.x, y.y)) : "memory");
                    }
                }
            }
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
            mbar_arrive(&empty[s]);
            mbar_arrive(&ofull[o]);
        }
    }
}

static uint32_t odd16_pitch(uint32_t row_bytes) {  // smallest pitch >= row_bytes that is an odd multiple of 16 bytes
    uint32_t q = (row_bytes + 15u) / 16u;
    if ((q & 1u) == 0) ++q;
    return q * 16u;
}

}  // namespace title

bool mhsa_title_bwd_supported(int T, int dk, int heads, int sec, int ld_qkv, int ld_dctx, int ld_dqkv) {
    using namespace title;
    if (T != kT || dk != kDk || heads < 1 || heads > kMaxHeads) return false;
    if (sec % 8 != 0 || sec < heads * dk || ld_qkv % 8 != 0 || ld_dctx % 8 != 0 || ld_dqkv != ld_qkv) return false;
    if (ld_qkv < 3 * sec || ld_dctx < heads * dk) return false;
    return odd16_pitch(static_cast<uint32_t>(3 * sec) * 2u) <= 2048u && odd16_pitch(static_cast<uint32_t>(ld_dctx) * 2u) <= 2048u;
}

int mhsa_title_bwd(const void* qkv, int ld_qkv, int sec, const void* dctx, int ld_dctx, long long n_seq, int heads, void* dqkv,
                   int ld_dqkv, cudaStream_t stream, const TitleBwdLive* live) {
    using namespace title;
    NR_REQUIRE(mhsa_title_bwd_supported(kT, kDk, heads, sec, ld_qkv, ld_dctx, ld_dqkv), "mhsa_title_bwd: unsupported layout");
    NR_REQUIRE(n_seq * kT < (1ll << 31), "mhsa_title_bwd: too many rows");
    if (n_seq == 0) return 0;
    Params p;
    p.n_seq = static_cast<int>(n_seq);
    p.heads = heads;
    p.sec2 = static_cast<uint32_t>(sec) * 2u;
    const uint32_t qkv_row = 3u * p.sec2;                     // bytes of a row that carry sections
    const uint32_t dc_row = static_cast<uint32_t>(ld_dctx) * 2u;
    p.pq = odd16_pitch(qkv_row);
    p.pc = odd16_pitch(dc_row);
    p.qkv_tile = (kT * p.pq + 127u) & ~127u;
    const uint32_t dc_tile = (kT * p.pc + 127u) & ~127u;
    p.in_stage = p.qkv_tile + dc_tile;
    p.out_stage = p.qkv_tile;
    p.tx = kT * p.pq + kT * p.pc;
    p.rs = 1.0f / sqrtf(static_cast<float>(kDk));
    p.sc = p.rs * 1.4426950408889634f;
    const LiveTokens* lt = live != nullptr ? live->tokens : nullptr;
    NR_REQUIRE(live == nullptr || (lt != nullptr && lt->pad && lt->mask && lt->offset && lt->qkv && live->dbias),
               "mhsa_title_bwd: live tokens without their flags, offsets, padding Q|K|V tile or bias column");
    NR_REQUIRE(live == nullptr || (reinterpret_cast<uintptr_t>(dqkv) & 15) == 0, "mhsa_title_bwd: compact rows not 16-byte aligned");
    p.pad = lt != nullptr ? lt->pad : nullptr;
    p.mask = lt != nullptr ? lt->mask : nullptr;
    p.offset = lt != nullptr ? lt->offset : nullptr;
    p.dqkv = static_cast<char*>(dqkv);
    p.ld_out = static_cast<uint32_t>(ld_dqkv) * 2u;
    p.row_bytes = qkv_row;
    p.dbias = live != nullptr ? live->dbias : nullptr;
    p.ld_dbias = live != nullptr ? live->ld_dbias : 0;
    p.compact = live != nullptr && live->compact_qkv ? 1 : 0;
    p.bias = lt != nullptr ? lt->qkv : nullptr;
    const size_t smem = 128 + static_cast<size_t>(kIn) * p.in_stage + static_cast<size_t>(kOut) * p.out_stage +
                       static_cast<size_t>(heads) * kScrWarp + 128 + p.pq + 64;  // barriers | bias row
    NR_REQUIRE(smem <= 227 * 1024, "mhsa_title_bwd: %zu bytes of shared memory", smem);
    const long long rows = n_seq * kT;
    CUtensorMap tq, tc, to, tp;
    NR_PROPAGATE(make_tmap_bytes_2d(&tq, qkv, rows, qkv_row, static_cast<int64_t>(ld_qkv) * 2, static_cast<int>(p.pq), kT));
    NR_PROPAGATE(make_tmap_bytes_2d(&tc, dctx, rows, dc_row, static_cast<int64_t>(ld_dctx) * 2, static_cast<int>(p.pc), kT));
    NR_PROPAGATE(make_tmap_bytes_2d(&to, dqkv, rows, qkv_row, static_cast<int64_t>(ld_dqkv) * 2, static_cast<int>(p.pq), kT));
    if (lt != nullptr)
        NR_PROPAGATE(make_tmap_bytes_2d(&tp, lt->qkv, kT, qkv_row, static_cast<int64_t>(ld_qkv) * 2, static_cast<int>(p.pq), kT));
    else
        tp = tq;
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(mhsa_title_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set = true;
    }
    const int grid = static_cast<int>(std::min<long long>(n_seq, num_sms()));
    mhsa_title_bwd_kernel<<<grid, (heads + 1) * 32, smem, stream>>>(tq, tc, to, tp, p);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

bool mhsa_title_fwd_supported(int T, int dk, int heads, int sec, int ld_qkv, int ld_ctx) {
    using namespace title;
    if (T != kT || dk != kDk || heads < 1 || heads > kMaxHeads) return false;
    if (sec % 8 != 0 || sec < heads * dk || ld_qkv % 8 != 0 || ld_ctx % 8 != 0 || ld_qkv < 3 * sec || ld_ctx < heads * dk + 1) return false;
    return odd16_pitch(static_cast<uint32_t>(3 * sec) * 2u) <= 2048u && odd16_pitch(static_cast<uint32_t>(ld_ctx) * 2u) <= 2048u;
}

// v_lo / ctx_lo both non-null: the accurate (hi/lo) variant.  v_lo bf16 [rows][ld_vlo] = low plane of the V section (column 0
// = first V column); ctx_lo bf16 [rows][ld_ctx] = low plane of the context (no ones column).
int mhsa_title_fwd(const void* qkv, int ld_qkv, int sec, long long n_seq, int heads, void* ctx, int ld_ctx, DropoutCfg drop,
                   cudaStream_t stream, const void* v_lo, int ld_vlo, void* ctx_lo, const PaddingTitles* pad, const LiveTokens* live) {
    using namespace title;
    NR_REQUIRE(mhsa_title_fwd_supported(kT, kDk, heads, sec, ld_qkv, ld_ctx), "mhsa_title_fwd: unsupported layout");
    NR_REQUIRE(n_seq * kT < (1ll << 31), "mhsa_title_fwd: too many rows");
    const bool hilo = v_lo != nullptr || ctx_lo != nullptr;
    NR_REQUIRE(!hilo || (v_lo != nullptr && ctx_lo != nullptr && ld_vlo % 8 == 0 && ld_vlo >= heads * kDk),
               "mhsa_title_fwd: the hi/lo variant needs both low planes (ld_vlo=%d)", ld_vlo);
    if (n_seq == 0) return 0;
    FwdParams p;
    p.n_seq = static_cast<int>(n_seq);
    p.heads = heads;
    p.ld_ctx = ld_ctx;
    p.sec2 = static_cast<uint32_t>(sec) * 2u;
    const uint32_t qkv_row = 3u * p.sec2, ctx_row = static_cast<uint32_t>(ld_ctx) * 2u, vlo_row = static_cast<uint32_t>(ld_vlo) * 2u;
    p.pq = odd16_pitch(qkv_row);
    p.pc = odd16_pitch(ctx_row);
    p.pv = hilo ? odd16_pitch(vlo_row) : 0u;
    p.qkv_tile = (kT * p.pq + 127u) & ~127u;
    p.in_stage = p.qkv_tile + (hilo ? ((kT * p.pv + 127u) & ~127u) : 0u);
    p.out_tile = (kT * p.pc + 127u) & ~127u;
    p.out_stage = (hilo ? 2u : 1u) * p.out_tile;
    p.tx = kT * p.pq + (hilo ? kT * p.pv : 0u);
    p.sc = 1.4426950408889634f / sqrtf(static_cast<float>(kDk));
    p.drop = Dropout::make(drop.p, drop.seed);
    NR_REQUIRE(pad == nullptr || (pad->pad != nullptr && pad->qkv != nullptr && (!hilo || (pad->v_lo != nullptr && ld_vlo == sec))),
               "mhsa_title_fwd: padding titles without their Q|K|V tile (or its V low plane at pitch sec)");
    NR_REQUIRE(live == nullptr || (pad == nullptr && live->pad && live->mask && live->offset && live->qkv && (!hilo || (live->v_lo && ld_vlo == sec))),
               "mhsa_title_fwd: live tokens without their flags, offsets or bias rows (or with padding titles as well)");
    p.pad = pad != nullptr ? pad->pad : nullptr;
    p.mask = live != nullptr ? live->mask : nullptr;
    p.offset = live != nullptr ? live->offset : nullptr;
    p.bias_q = live != nullptr ? live->qkv : nullptr;
    p.bias_v = live != nullptr ? live->v_lo : nullptr;
    // fragment loads of rows 20..23 of a tile run into whatever follows it (the low-plane tile, the next stage, the result
    // tiles): always inside the allocation, always initialised
    const int n_in = hilo ? kInHilo : kIn;
    const size_t smem = 128 + static_cast<size_t>(n_in) * p.in_stage + static_cast<size_t>(kOut) * p.out_stage +
                       128 + p.pq + p.pv + 64;  // barriers | bias rows
    const size_t cap = hilo ? 227 * 1024 : 113 * 1024;
    NR_REQUIRE(smem <= cap, "mhsa_title_fwd: %zu bytes of shared memory", smem);
    const long long rows = n_seq * kT;
    CUtensorMap tq, tc, tv, tl, tp, tpl;
    NR_PROPAGATE(make_tmap_bytes_2d(&tq, qkv, rows, qkv_row, static_cast<int64_t>(ld_qkv) * 2, static_cast<int>(p.pq), kT));
    NR_PROPAGATE(make_tmap_bytes_2d(&tc, ctx, rows, ctx_row, static_cast<int64_t>(ld_ctx) * 2, static_cast<int>(p.pc), kT));
    if (hilo) {
        NR_PROPAGATE(make_tmap_bytes_2d(&tv, v_lo, rows, vlo_row, static_cast<int64_t>(ld_vlo) * 2, static_cast<int>(p.pv), kT));
        NR_PROPAGATE(make_tmap_bytes_2d(&tl, ctx_lo, rows, ctx_row, static_cast<int64_t>(ld_ctx) * 2, static_cast<int>(p.pc), kT));
    } else {
        tv = tq;
        tl = tc;
    }
    tp = tq;
    tpl = tv;
    if (pad != nullptr) {
        NR_PROPAGATE(make_tmap_bytes_2d(&tp, pad->qkv, kT, qkv_row, static_cast<int64_t>(ld_qkv) * 2, static_cast<int>(p.pq), kT));
        if (hilo) NR_PROPAGATE(make_tmap_bytes_2d(&tpl, pad->v_lo, kT, vlo_row, static_cast<int64_t>(ld_vlo) * 2, static_cast<int>(p.pv), kT));
    }
    static bool attr_set = false;
    if (!attr_set) {
        NR_CHECK_CUDA(cudaFuncSetAttribute(mhsa_title_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 113 * 1024));
        NR_CHECK_CUDA(cudaFuncSetAttribute(mhsa_title_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set = true;
    }
    const int grid = static_cast<int>(std::min<long long>(n_seq, (hilo ? 1ll : 2ll) * num_sms()));
    if (hilo)
        mhsa_title_fwd_kernel<true><<<grid, (heads + 1) * 32, smem, stream>>>(tq, tv, tc, tl, tp, tpl, p);
    else
        mhsa_title_fwd_kernel<false><<<grid, (heads + 1) * 32, smem, stream>>>(tq, tv, tc, tl, tp, tpl, p);
    ++g_launches;
    NR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace nr
