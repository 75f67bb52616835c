// Warp-specialised causal varlen prefill attention (wgmma + TMA + mbarrier), second generation of prefill_tc.cu.
//
// Same operator (reference nanovllm/layers/attention.py:64-70: flash_attn_varlen_func, packed or paged K/V, bottom-right
// aligned causal mask), different machine mapping.  prefill_tc.cu's warpgroups load, multiply and exponentiate in turn and
// each CTA stages its own K / V tiles.  Here one CTA owns 64 queries of the TWO q-heads of a GQA group that share a kv head
// (every K / V tile is staged once for both), and the roles are split:
//
//   warps 0-3  ("WG0")  head 0: S = Q K^T (wgmma m64n64k16 x8, fp32 in registers), scale / mask / exponentiate in
//                       registers, P (bf16) fed to O += P V (wgmma m64n128k16 x4, A from registers, V MN-major) straight
//                       from registers; running reference max and row sum, O rescaled in registers when the max moves by > 2^8
//   warps 4-7  ("WG1")  the same for head 1 (idle for the last head of an odd group)
//   warp 8              TMA producer: Q (both heads) once, then a 3-deep ring of K and V tiles (64 keys), paged tiles
//                       page by page through the block table; a slot is refilled once every consumer warp has released it
//
// The two warpgroups run independently on the shared ring, so the tensor pipe works on one head's MMAs while the other
// head is exponentiating.  Shared memory: Q 2 x 16 KB, K 3 x 16 KB, V 3 x 16 KB = 128 KB, one CTA per SM.  Arithmetic and
// rounding points are those of prefill_tc.cu (P rounded to bf16 as the reference's kernel does, fp32 accumulation, one
// rounding of the output); with POLY half of the exponentials run as a polynomial on the FMA pipe.
#include <cstdlib>

#include "tc_common.cuh"

namespace {

using namespace b200tc;

constexpr int BM = 64, BN = 64, D = B200_HEAD_DIM;
constexpr int WS_THREADS = 288;                    // 2 consumer warpgroups + producer warp
constexpr int KV_STAGES = 3;
constexpr uint32_t Q_HALF = BM * 128;              // 8 KB: [64 rows][64 dims]
constexpr uint32_t Q_BYTES = 2 * Q_HALF;           // 16 KB per head
constexpr uint32_t KV_HALF = BN * 128;             // 8 KB
constexpr uint32_t KV_BYTES = 2 * KV_HALF;         // 16 KB: two [64][64] halves
constexpr uint32_t OFF_Q = 0;                                        // 2 heads
constexpr uint32_t OFF_K = OFF_Q + 2 * Q_BYTES;
constexpr uint32_t OFF_V = OFF_K + KV_STAGES * KV_BYTES;
constexpr uint32_t OFF_BAR = OFF_V + KV_STAGES * KV_BYTES;
constexpr uint32_t WS_SMEM = OFF_BAR + 128;
constexpr float RESCALE_THRESHOLD = 8.0f;          // log2 units

// barrier slots (8 bytes each) from OFF_BAR
constexpr uint32_t B_Q = 0;                        // Q tiles landed
constexpr uint32_t B_KFULL = 1, B_VFULL = 4;       // 3 each
constexpr uint32_t B_EMPTY = 7;                    // 3: one arrival per consumer warp once its PV of the slot has retired
constexpr uint32_t B_COUNT = 10;

struct WsParams {
    const int32_t* cu_q;
    const int32_t* cu_k;
    const int32_t* block_tables;   // null => packed k/v
    int bt_stride;
    __nv_bfloat16* out;
    int64_t out_stride;
    int hq, hkv, block_shift;
    int box_rows;                  // rows per TMA box of a paged tile: min(block_size, 64)
    int64_t layer_row0;
    float scale_log2;
};

// 2^x for x <= ~8 on the FMA/ALU pipes instead of the MUFU unit (the softmax is MUFU-bound: one exp2 per score).
// Cody-Waite split x = n + f, f in [0, 1), and a degree-3 minimax polynomial for 2^f (relative error < 1e-4, far inside the
// bf16 rounding P gets anyway); the exponent is added into the float's exponent field.
__device__ __forceinline__ float exp2_poly(float x) {
    const float xc = fmaxf(x, -120.0f);
    const float n = floorf(xc);
    const float f = xc - n;
    float pf = fmaf(f, 0.07790716f, 0.22623319f);      // 2^f ~ c0 + f (c1 + f (c2 + f c3)): relative error < 7.8e-5 on [0, 1)
    pf = fmaf(f, pf, 0.6957771f);
    pf = fmaf(f, pf, 0.99992783f);
    const float y = __int_as_float(__float_as_int(pf) + ((int)n << 23));
    return x < -120.0f ? 0.f : y;                      // masked scores (-inf) must give exactly 0
}

template <bool POLY>
__global__ void __launch_bounds__(WS_THREADS, 1)
prefill_ws_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                  const __grid_constant__ CUtensorMap tm_v, const WsParams p) {
    B200_PDL_SYNC();
    extern __shared__ __align__(1024) uint8_t smem_raw[];   // 128-byte swizzle atoms need 1024-byte alignment
    const uint32_t base = smem_u32(smem_raw);
    if (base & 1023u) __trap();
    const uint32_t bars = base + OFF_BAR;
    auto bar = [&](uint32_t i) { return bars + i * 8; };

    const int seq = blockIdx.z;
    const int g_heads = p.hq / p.hkv;                      // q heads per kv head
    const int pairs_per_kv = (g_heads + 1) / 2;
    const int kvh = blockIdx.y / pairs_per_kv;
    const int head0 = kvh * g_heads + (blockIdx.y % pairs_per_kv) * 2;
    const bool two = (head0 + 1) < (kvh + 1) * g_heads;    // an odd group leaves the second warpgroup of its last pair idle
    const int mb = gridDim.x - 1 - blockIdx.x;             // longest tiles first
    const int q0 = p.cu_q[seq];
    const int len_q = p.cu_q[seq + 1] - q0;
    const int k0 = p.cu_k[seq];
    const int len_k = p.cu_k[seq + 1] - k0;
    if (mb * BM >= len_q) return;
    const int off = len_k - len_q;
    int j_end = mb * BM + BM + off;
    j_end = j_end > len_k ? len_k : j_end;
    const int nblocks = (j_end + BN - 1) / BN;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const bool paged = p.block_tables != nullptr;

    if (tid == 0) {
        for (uint32_t i = 0; i < B_EMPTY; ++i) mbar_init(bar(i), 1);
        for (uint32_t i = B_EMPTY; i < B_COUNT; ++i) mbar_init(bar(i), two ? 8 : 4);
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ---- TMA producer -------------------------------------------------------------------------------------------
        if (lane == 0) {
            mbar_expect_tx(bar(B_Q), two ? 2 * Q_BYTES : Q_BYTES);
            for (int t = 0; t < (two ? 2 : 1); ++t)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    tma_load_2d(base + OFF_Q + t * Q_BYTES + h * Q_HALF, &tm_q, bar(B_Q), (head0 + t) * D + h * 64, q0 + mb * BM);
            auto load_kv = [&](const CUtensorMap* map, uint32_t dst, uint32_t full, int jb) {   // one 64-key tile, both halves
                mbar_expect_tx(full, KV_BYTES);
                if (!paged) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) tma_load_2d(dst + h * KV_HALF, map, full, kvh * D + h * 64, k0 + jb * BN);
                } else {
                    const int R = p.box_rows;
                    for (int s = 0; s < BN / R; ++s) {
                        const int key = jb * BN + s * R;
                        int page = key < len_k ? p.block_tables[(int64_t)seq * p.bt_stride + (key >> p.block_shift)] : 0;
                        page = page < 0 ? 0 : page;
                        const int64_t row = p.layer_row0 + ((((int64_t)page * p.hkv + kvh) << p.block_shift) + (key & ((1 << p.block_shift) - 1)));
#pragma unroll
                        for (int h = 0; h < 2; ++h) tma_load_2d(dst + h * KV_HALF + s * R * 128, map, full, h * 64, (int)row);
                    }
                }
            };
            for (int j = 0; j < nblocks; ++j) {
                const int s = j % KV_STAGES;
                if (j >= KV_STAGES) mbar_wait(bar(B_EMPTY + s), ((j / KV_STAGES) - 1) & 1);
                load_kv(&tm_k, base + OFF_K + s * KV_BYTES, bar(B_KFULL + s), j);
                load_kv(&tm_v, base + OFF_V + s * KV_BYTES, bar(B_VFULL + s), j);
            }
        }
        return;
    }

    // ---- consumer warpgroup t: q-head head0 + t ------------------------------------------------------------------------
    const int t = warp >> 2;
    if (t == 1 && !two) return;
    const int g = lane >> 2, qd = lane & 3;
    const int row_lo = mb * BM + (warp & 3) * 16 + g;      // this thread's two query rows: row_lo, row_lo + 8
    const int rows_w0 = mb * BM + (warp & 3) * 16;
    const uint32_t sQ = base + OFF_Q + t * Q_BYTES;
    float m_ref[2] = {-INFINITY, -INFINITY}, l_sum[2] = {0.f, 0.f};
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;

    mbar_wait(bar(B_Q), 0);
    for (int j = 0; j < nblocks; ++j) {
        const int s = j % KV_STAGES;
        const uint32_t par = (j / KV_STAGES) & 1;

        // ---- S = Q K(j)^T ---------------------------------------------------------------------------------------
        mbar_wait(bar(B_KFULL + s), par);
        float sc[BN / 2];
        const uint32_t kb = base + OFF_K + s * KV_BYTES;
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < D / 16; ++ks)
            wgmma_ss<BN>(sc, make_desc(sQ + (ks >> 2) * Q_HALF + (ks & 3) * 32, 16, 1024),
                         make_desc(kb + (ks >> 2) * KV_HALF + (ks & 3) * 32, 16, 1024), ks > 0 ? 1u : 0u);
        wg_commit();
        wg_wait<0>();
        acc_fence(sc);

        // sc[4c + 2h + e]: row row_lo + 8h, key j*BN + 8c + 2qd + e
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) sc[i] *= p.scale_log2;
        const bool need_mask = (j * BN + BN > len_k) || (j * BN + BN - 1 > rows_w0 + off);
        if (need_mask) {
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) {
                const int jj = j * BN + 8 * (i >> 2) + 2 * qd + (i & 1);
                const int r = row_lo + 8 * ((i >> 1) & 1);
                if (jj >= len_k || jj > r + off) sc[i] = -INFINITY;
            }
        }
        float m_new[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) m_new[(i >> 1) & 1] = fmaxf(m_new[(i >> 1) & 1], sc[i]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            m_new[h] = fmaxf(m_new[h], __shfl_xor_sync(0xffffffffu, m_new[h], 1));
            m_new[h] = fmaxf(m_new[h], __shfl_xor_sync(0xffffffffu, m_new[h], 2));
        }
        if (j == 0) {
#pragma unroll
            for (int h = 0; h < 2; ++h) m_ref[h] = (m_new[h] == -INFINITY) ? 0.f : m_new[h];
        } else if (__any_sync(0xffffffffu, m_new[0] > m_ref[0] + RESCALE_THRESHOLD || m_new[1] > m_ref[1] + RESCALE_THRESHOLD)) {
            float f[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float m_upd = fmaxf(m_ref[h], m_new[h]);
                f[h] = fast_exp2(m_ref[h] - m_upd);
                m_ref[h] = m_upd;
                l_sum[h] *= f[h];
            }
#pragma unroll
            for (int i = 0; i < D / 2; ++i) o[i] *= f[(i >> 1) & 1];
        }

        // ---- P = exp2(S - m_ref) -> bf16 A fragments (k step kk = keys 16 kk .. 16 kk + 15) -------------------
        uint32_t pa[BN / 16][4];
#pragma unroll
        for (int kk = 0; kk < BN / 16; ++kk) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int i = 8 * kk + 2 * r;            // r: (row lo, k lo) (row hi, k lo) (row lo, k hi) (row hi, k hi)
                const int h = r & 1;
                const float p0 = fast_exp2(sc[i] - m_ref[h]);
                const float p1 = POLY ? exp2_poly(sc[i + 1] - m_ref[h]) : fast_exp2(sc[i + 1] - m_ref[h]);
                l_sum[h] += p0 + p1;
                pa[kk][r] = pack_bf16x2(p0, p1);
            }
        }

        mbar_wait(bar(B_VFULL + s), par);
        if (j * BN + BN > len_k) {
            // Tail block: V rows at keys >= len_k are not this sequence's (stale page rows, the next sequence of a packed
            // batch, anything -- possibly NaN/Inf).  Their P is exactly 0, but 0 * NaN would poison the accumulator, so
            // zero those rows of the staged tile (each warpgroup writes the same zeros, then orders them before its MMA).
            const int first = len_k - j * BN;                               // 1..63
            uint8_t* vtile = smem_raw + OFF_V + s * KV_BYTES;
            for (int i = tid & 127; i < (BN - first) * 16; i += 128) {       // 16 chunks of 16 B per row: 2 halves x 8
                const int r = first + (i >> 4), c = i & 15;
                *reinterpret_cast<uint4*>(vtile + (c >> 3) * KV_HALF + r * 128 + ((c & 7) << 4)) = make_uint4(0, 0, 0, 0);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> visible to the MMA
            asm volatile("bar.sync %0, 128;" ::"r"(1 + t) : "memory");        // this warpgroup only
        }

        // ---- O += P V(j) ---------------------------------------------------------------------------------------
        const uint32_t vb = base + OFF_V + s * KV_BYTES;
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < BN / 16; ++kk) wgmma_rs_bmn<D>(o, pa[kk], make_desc(vb + kk * 2048, KV_HALF, 1024), 1u);
        wg_commit();
        wg_wait<0>();
        acc_fence(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(B_EMPTY + s));     // this warp no longer reads slot s
    }

    // ---- epilogue: O / l -> bf16 -> global ------------------------------------------------------------
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float l = l_sum[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = l > 0.f ? 1.f / l : 0.f;
        const int row = row_lo + 8 * h;
        if (row < len_q) {
            __nv_bfloat16* dst = p.out + (int64_t)(q0 + row) * p.out_stride + (head0 + t) * D + 2 * qd;
#pragma unroll
            for (int c = 0; c < D / 8; ++c)
                *reinterpret_cast<uint32_t*>(dst + 8 * c) = pack_bf16x2(o[4 * c + 2 * h] * inv, o[4 * c + 2 * h + 1] * inv);
        }
    }
}

}  // namespace

// Called from b200_paged_prefill / b200_prefill_packed_kv (prefill_attn.cu).  Returns B200_EUNSUPPORTED if TMA descriptors
// cannot be built.
int b200_prefill_ws_launch(b200_ctx* ctx, int layer, const void* q, int64_t q_stride0, const void* k, int64_t k_stride0,
                           const void* v, int64_t v_stride0, const int32_t* cu_q, const int32_t* cu_k,
                           const int32_t* block_tables, int bt_stride, void* out, int64_t out_stride0, int total_q, int total_k,
                           int num_seqs, int max_seqlen_q, int num_q_heads, int num_kv_heads, float scale,
                           cudaStream_t stream) {
    if ((out_stride0 % 8) || ((uintptr_t)out & 15)) return B200_EINVAL;
    CUtensorMap tq, tk, tv;
    if (!make_map(&tq, q, (uint64_t)num_q_heads * D, (uint64_t)total_q, (uint64_t)q_stride0, BM)) return B200_EUNSUPPORTED;
    WsParams prm;
    prm.cu_q = cu_q;
    prm.cu_k = cu_k;
    prm.block_tables = block_tables;
    prm.bt_stride = bt_stride;
    prm.out = static_cast<__nv_bfloat16*>(out);
    prm.out_stride = out_stride0;
    prm.hq = num_q_heads;
    prm.hkv = num_kv_heads;
    prm.scale_log2 = scale * 1.4426950408889634f;
    prm.block_shift = 0;
    prm.box_rows = BN;
    prm.layer_row0 = 0;
    if (block_tables) {
        const uint32_t R = ctx->block_size < BN ? ctx->block_size : BN;
        const uint64_t rows = (uint64_t)ctx->layers * ctx->num_blocks * ctx->num_kv_heads * ctx->block_size;
        if (rows >= (1ull << 31)) return B200_EUNSUPPORTED;
        if (!make_map(&tk, ctx->k_base, D, rows, D, R) || !make_map(&tv, ctx->v_base, D, rows, D, R)) return B200_EUNSUPPORTED;
        prm.block_shift = ctx->block_shift;
        prm.box_rows = (int)R;
        prm.layer_row0 = (int64_t)layer * ctx->num_blocks * ctx->num_kv_heads * ctx->block_size;
    } else {
        if (!make_map(&tk, k, (uint64_t)num_kv_heads * D, (uint64_t)total_k, (uint64_t)k_stride0, BN) ||
            !make_map(&tv, v, (uint64_t)num_kv_heads * D, (uint64_t)total_k, (uint64_t)v_stride0, BN))
            return B200_EUNSUPPORTED;
    }
    // B200_PREFILL_POLY=0 keeps every exponential on the MUFU unit (A/B of the polynomial half)
    static const bool poly = [] { const char* e = getenv("B200_PREFILL_POLY"); return e ? atoi(e) != 0 : true; }();
    static B200SmemOptIn optin_poly, optin_mufu;
    const int g_heads = num_q_heads / num_kv_heads;
    dim3 grid((max_seqlen_q + BM - 1) / BM, num_kv_heads * ((g_heads + 1) / 2), num_seqs);
    if (grid.z > 65535 || grid.y > 65535) return B200_EUNSUPPORTED;
    if (poly) {
        B200_CUDA_CHECK(ctx, optin_poly.ensure(prefill_ws_kernel<true>, WS_SMEM));
        B200_LAUNCH((prefill_ws_kernel<true>), grid, WS_THREADS, WS_SMEM, stream, tq, tk, tv, prm);
    } else {
        B200_CUDA_CHECK(ctx, optin_mufu.ensure(prefill_ws_kernel<false>, WS_SMEM));
        B200_LAUNCH((prefill_ws_kernel<false>), grid, WS_THREADS, WS_SMEM, stream, tq, tk, tv, prm);
    }
    return b200_launch_status(ctx);
}
