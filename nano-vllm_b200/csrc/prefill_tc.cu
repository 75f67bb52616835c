// Causal varlen prefill attention on Hopper's tensor cores (wgmma + TMA + mbarrier).
//
// Replaces the prefill branch of the reference's Attention.forward (nanovllm/layers/attention.py:64-70,
// flash_attn_varlen_func with an optional block_table): packed or paged K/V, bottom-right aligned
// causal mask (query i sees keys j <= i + len_k - len_q).
//
// One CTA = 128 queries of one head, two warpgroups of 64 query rows each, key blocks of 64, two CTAs per SM:
//   * Q, K and V tiles are staged by TMA (cp.async.bulk.tensor, 128-byte swizzle) into shared memory, K and V
//     double-buffered so that the next block's tiles arrive under this block's math; a paged K/V tile is fetched
//     page by page through the block table with the same tensor map;
//   * S = Q K^T : wgmma m64n64k16 x 8 per warpgroup, both operands K-major from shared memory, fp32 in registers;
//   * softmax in registers: a query row is held by the four threads of a quad (row max / row sum: two shuffles);
//     P is rounded to bf16 (as the reference's kernel does) and fed to the next MMA straight from registers (the
//     accumulator layout of S is the A-fragment layout of P);
//   * O += P V : wgmma m64n128k16 x 4, V consumed as an MN-major operand straight from its [key][d] tile; the running
//     reference max only moves (and O is only rescaled) when a row's max grows by more than 2^8.
#include "tc_common.cuh"

namespace {

using namespace b200tc;

constexpr int BM = 128;
constexpr int BN = 64;
constexpr int D = B200_HEAD_DIM;
constexpr int TC_THREADS = 256;                   // two warpgroups
constexpr uint32_t Q_BYTES = BM * D * 2;          // 32 KB: two [128][64] halves
constexpr uint32_t KV_BYTES = BN * D * 2;         // 16 KB: two [64][64] halves
constexpr uint32_t Q_HALF = BM * 128;             // 16 KB
constexpr uint32_t KV_HALF = BN * 128;            // 8 KB
constexpr uint32_t OFF_Q = 0;
constexpr uint32_t OFF_K = OFF_Q + Q_BYTES;       // 2 buffers
constexpr uint32_t OFF_V = OFF_K + 2 * KV_BYTES;  // 2 buffers
constexpr uint32_t OFF_BAR = OFF_V + 2 * KV_BYTES;
constexpr uint32_t TC_SMEM = OFF_BAR + 64;        // 96.1 KB: two CTAs per SM
constexpr float RESCALE_THRESHOLD = 8.0f;         // log2 units

struct TcParams {
    const int32_t* cu_q;
    const int32_t* cu_k;
    const int32_t* block_tables;   // null => packed k/v
    int bt_stride;
    __nv_bfloat16* out;
    int64_t out_stride;
    int hq, hkv, block_shift;
    int box_rows;                  // rows per TMA box of a paged tile: min(block_size, 64)
    int64_t layer_row0;            // first row of this layer in the [rows, 128] view of the cache
    float scale_log2;
};

__global__ void __launch_bounds__(TC_THREADS, 2)
prefill_tc_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                  const __grid_constant__ CUtensorMap tm_v, const TcParams p) {
    B200_PDL_SYNC();
    extern __shared__ __align__(1024) uint8_t smem_raw[];   // 128-byte swizzle atoms need 1024-byte alignment
    const uint32_t base = smem_u32(smem_raw);
    if (base & 1023u) __trap();
    uint8_t* base_ptr = smem_raw;
    const uint32_t sQ = base + OFF_Q, sK = base + OFF_K, sV = base + OFF_V;
    const uint32_t bars = base + OFF_BAR;
    const uint32_t bar_q = bars, bar_k0 = bars + 8, bar_v0 = bars + 24;

    const int seq = blockIdx.z;
    const int head = blockIdx.y;
    const int mb = gridDim.x - 1 - blockIdx.x;      // longest tiles first
    const int q0 = p.cu_q[seq];
    const int len_q = p.cu_q[seq + 1] - q0;
    const int k0 = p.cu_k[seq];
    const int len_k = p.cu_k[seq + 1] - k0;
    if (mb * BM >= len_q) return;
    const int off = len_k - len_q;
    const int kvh = head / (p.hq / p.hkv);
    int j_end = mb * BM + BM + off;
    j_end = j_end > len_k ? len_k : j_end;
    const int nblocks = (j_end + BN - 1) / BN;

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2;                       // warpgroup: query rows [64 wg, 64 wg + 64) of the tile
    const int g = lane >> 2, qd = lane & 3;
    const bool paged = p.block_tables != nullptr;

    if (tid == 0) {
        for (int i = 0; i < 5; ++i) mbar_init(bars + i * 8, 1);
        mbar_fence_init();
    }
    __syncthreads();

    auto load_kv = [&](const CUtensorMap* map, uint32_t dst, uint32_t bar, int jb) {   // one 64-key tile, both halves
        mbar_expect_tx(bar, KV_BYTES);
        if (!paged) {
#pragma unroll
            for (int h = 0; h < 2; ++h) tma_load_2d(dst + h * KV_HALF, map, bar, kvh * D + h * 64, k0 + jb * BN);
        } else {
            const int R = p.box_rows;
            for (int s = 0; s < BN / R; ++s) {
                const int key = jb * BN + s * R;
                int page = key < len_k ? p.block_tables[(int64_t)seq * p.bt_stride + (key >> p.block_shift)] : 0;
                page = page < 0 ? 0 : page;
                const int64_t row = p.layer_row0 + ((((int64_t)page * p.hkv + kvh) << p.block_shift) + (key & ((1 << p.block_shift) - 1)));
#pragma unroll
                for (int h = 0; h < 2; ++h) tma_load_2d(dst + h * KV_HALF + s * R * 128, map, bar, h * 64, (int)row);
            }
        }
    };

    if (tid == 0) {
        mbar_expect_tx(bar_q, Q_BYTES);
#pragma unroll
        for (int h = 0; h < 2; ++h) tma_load_2d(sQ + h * Q_HALF, &tm_q, bar_q, head * D + h * 64, q0 + mb * BM);
        load_kv(&tm_k, sK, bar_k0, 0);
        load_kv(&tm_v, sV, bar_v0, 0);
        if (nblocks > 1) {
            load_kv(&tm_k, sK + KV_BYTES, bar_k0 + 8, 1);
            load_kv(&tm_v, sV + KV_BYTES, bar_v0 + 8, 1);
        }
    }

    // this thread's two query rows (in-sequence indices) and the first row of its warp
    const int row_lo = mb * BM + wg * 64 + (warp & 3) * 16 + g;
    const int rows_w0 = mb * BM + wg * 64 + (warp & 3) * 16;
    float m_ref[2] = {-INFINITY, -INFINITY}, l_sum[2] = {0.f, 0.f};
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    const uint32_t q_wg = sQ + wg * 64 * 128;

    mbar_wait(bar_q, 0);
    for (int j = 0; j < nblocks; ++j) {
        const int b = j & 1;
        const uint32_t par = (j >> 1) & 1;

        // ---- S = Q K(j)^T for this warpgroup's 64 rows ------------------------------------------------
        mbar_wait(bar_k0 + b * 8, par);
        float s[BN / 2];
        const uint32_t kb = sK + b * KV_BYTES;
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < D / 16; ++ks)
            wgmma_ss<BN>(s, make_desc(q_wg + (ks >> 2) * Q_HALF + (ks & 3) * 32, 16, 1024),
                         make_desc(kb + (ks >> 2) * KV_HALF + (ks & 3) * 32, 16, 1024), ks > 0 ? 1u : 0u);
        wg_commit();
        wg_wait<0>();
        acc_fence(s);

        // s[4c + 2h + e]: row row_lo + 8h, key j*BN + 8c + 2qd + e
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) s[i] *= p.scale_log2;
        const bool need_mask = (j * BN + BN > len_k) || (j * BN + BN - 1 > rows_w0 + off);
        if (need_mask) {
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) {
                const int jj = j * BN + 8 * (i >> 2) + 2 * qd + (i & 1);
                const int r = row_lo + 8 * ((i >> 1) & 1);
                if (jj >= len_k || jj > r + off) s[i] = -INFINITY;
            }
        }
        float m_new[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) m_new[(i >> 1) & 1] = fmaxf(m_new[(i >> 1) & 1], s[i]);
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
                const float p0 = fast_exp2(s[i] - m_ref[h]), p1 = fast_exp2(s[i + 1] - m_ref[h]);
                l_sum[h] += p0 + p1;
                pa[kk][r] = pack_bf16x2(p0, p1);
            }
        }

        mbar_wait(bar_v0 + b * 8, par);
        if (j * BN + BN > len_k) {
            // Tail block: V rows at keys >= len_k are not this sequence's (stale page rows, the next sequence of a packed
            // batch, anything -- possibly NaN/Inf).  Their P is exactly 0, but 0 * NaN would poison the accumulator, so
            // zero those rows of the staged tile.  A whole 128-byte row is zeroed, which is swizzle-agnostic.
            const int first = len_k - j * BN;                               // 1..63
            uint8_t* vtile = base_ptr + OFF_V + b * KV_BYTES;
            for (int i = tid; i < (BN - first) * 16; i += TC_THREADS) {     // 16 chunks of 16 B per row: 2 halves x 8
                const int r = first + (i >> 4), c = i & 15;
                *reinterpret_cast<uint4*>(vtile + (c >> 3) * KV_HALF + r * 128 + ((c & 7) << 4)) = make_uint4(0, 0, 0, 0);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> visible to the MMA
            __syncthreads();
        }

        // ---- O += P V(j) ---------------------------------------------------------------------------------
        const uint32_t vb = sV + b * KV_BYTES;
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < BN / 16; ++kk) wgmma_rs_bmn<D>(o, pa[kk], make_desc(vb + kk * 2048, KV_HALF, 1024), 1u);
        wg_commit();
        wg_wait<0>();
        acc_fence(o);

        __syncthreads();                                  // both warpgroups are done with K / V buffer b
        if (tid == 0 && j + 2 < nblocks) {
            load_kv(&tm_k, sK + b * KV_BYTES, bar_k0 + b * 8, j + 2);
            load_kv(&tm_v, sV + b * KV_BYTES, bar_v0 + b * 8, j + 2);
        }
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
            __nv_bfloat16* dst = p.out + (int64_t)(q0 + row) * p.out_stride + head * D + 2 * qd;
#pragma unroll
            for (int c = 0; c < D / 8; ++c)
                *reinterpret_cast<uint32_t*>(dst + 8 * c) = pack_bf16x2(o[4 * c + 2 * h] * inv, o[4 * c + 2 * h + 1] * inv);
        }
    }
}

}  // namespace

// Called from b200_paged_prefill (prefill_attn.cu).  Returns B200_EUNSUPPORTED if TMA descriptors cannot be built.
int b200_prefill_tc_launch(b200_ctx* ctx, int layer, const void* q, int64_t q_stride0, const void* k, int64_t k_stride0,
                           const void* v, int64_t v_stride0, const int32_t* cu_q, const int32_t* cu_k,
                           const int32_t* block_tables, int bt_stride, void* out, int64_t out_stride0, int total_q,
                           int num_seqs, int max_seqlen_q, int num_q_heads, int num_kv_heads, float scale,
                           cudaStream_t stream) {
    const int total_k = total_q;   // packed mode: K/V rows are the step's own tokens (attention.py:67-70 without block_table)
    if ((out_stride0 % 8) || ((uintptr_t)out & 15)) return B200_EINVAL;
    CUtensorMap tq, tk, tv;
    if (!make_map(&tq, q, (uint64_t)num_q_heads * D, (uint64_t)total_q, (uint64_t)q_stride0, BM)) return B200_EUNSUPPORTED;
    TcParams prm;
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
    static B200SmemOptIn optin;
    B200_CUDA_CHECK(ctx, optin.ensure(prefill_tc_kernel, TC_SMEM));
    dim3 grid((max_seqlen_q + BM - 1) / BM, num_q_heads, num_seqs);
    if (grid.z > 65535 || grid.y > 65535) return B200_EUNSUPPORTED;
    B200_LAUNCH((prefill_tc_kernel), grid, TC_THREADS, TC_SMEM, stream, tq, tk, tv, prm);
    return b200_launch_status(ctx);
}
