// Single-token paged decode attention, tensor-core formulation (same contract and same stream-K work
// partition as decode_attn.cu; see that file and DESIGN.md for the scheduling).
//
// What differs is how a warp digests one 16-token chunk:
//   * K and V chunks arrive as 128-byte-swizzled TMA tensor boxes (cp.async.bulk.tensor.2d over a
//     [rows, 128] view of the whole cache, box = 64 columns x 16 rows), so ldmatrix reads them conflict-free;
//   * S = q K^T and O += P V run on warp-level MMA (mma.sync m16n8k16, bf16 in / fp32 accumulate) with the G
//     query heads of the kv head as the first G rows of the 16-row tile: ~150 warp instructions per chunk
//     instead of ~670 for the fp32-FMA formulation, so the kernel is bound by the memory pipeline for every
//     head-group size (G = 1..8) instead of by instruction issue;
//   * softmax statistics live per quad (rows of the C fragment), P is rounded to bf16 for the PV product as in
//     the reference's kernel.
#include <cuda.h>

#include "decode_common.cuh"

using namespace b200dec;

namespace {

constexpr int MMA_WARPS = 8;
constexpr int MMA_STAGES = 2;
constexpr int HALF_BYTES = CHUNK * 128;            // one 64-column half of a chunk: 16 rows x 128 B
constexpr int KV_STAGE = 4 * HALF_BYTES;           // K lo | K hi | V lo | V hi

template <int G>
struct MmaSmem {
    static constexpr int kQBytes = G * ROW_BYTES;
    static constexpr int kQPad = (kQBytes + 1023) / 1024 * 1024;          // keeps every stage 1024-byte aligned
    static constexpr int kStageBytes = KV_STAGE + kQPad;
    static constexpr int kWarpBytes = MMA_STAGES * kStageBytes;
    static constexpr int kOffCum = MMA_WARPS * kWarpBytes;                // int[MAX_BATCH + 1]
    static constexpr int kOffCtx = kOffCum + (MAX_BATCH + 4) * 4;         // int[MAX_BATCH]
    static constexpr int kOffBars = kOffCtx + MAX_BATCH * 4;              // u64[warps][stages]
    static constexpr int kOffWarpTot = kOffBars + MMA_WARPS * MMA_STAGES * 8;
    static constexpr int kTotal = kOffWarpTot + 32 * 4;
};

// K/V are streamed exactly once per launch: the boxes carry an L2 evict_first policy
__device__ __forceinline__ void tma_box(uint32_t dst, const CUtensorMap* map, uint32_t bar, int col, int row, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;" ::
            "r"(dst), "l"(map), "r"(bar), "r"(col), "r"(row), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void ldsm4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm4t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
// rows 8..15 of the A tile are always zero here (at most 8 query heads per kv head)
__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
    const uint32_t z = 0u;
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(z), "r"(a2), "r"(z), "r"(b0), "r"(b1));
}

template <int G>
__global__ void __launch_bounds__(MMA_WARPS * 32, 1)
paged_decode_mma_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                        const DecodeParams p, const long long layer_row0) {
    B200_PDL_TRIGGER();
    using L = MmaSmem<G>;
    constexpr int NWARPS = MMA_WARPS, NSTAGES = MMA_STAGES;
    extern __shared__ __align__(1024) uint8_t smem[];
    if (smem_u32(smem) & 1023u) __trap();
    int* cum = reinterpret_cast<int*>(smem + L::kOffCum);
    int* ctxs = reinterpret_cast<int*>(smem + L::kOffCtx);
    int* warp_tot = reinterpret_cast<int*>(smem + L::kOffWarpTot);

    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int batch = p.batch;
    const int hkv = p.hkv;

    uint8_t* my_stages = smem + warp * L::kWarpBytes;
    const uint32_t my_stages_u32 = smem_u32(my_stages);
    const uint32_t my_bars_u32 = smem_u32(smem + L::kOffBars) + warp * NSTAGES * 8;

    if (lane == 0) {
        for (int s = 0; s < NSTAGES; ++s) mbar_init(my_bars_u32 + s * 8, 1);
        mbar_fence_init();
    }

    // ---- exclusive prefix of per-sequence chunk counts (same as decode_attn.cu) --------------------
    constexpr int NT = NWARPS * 32;
    constexpr int IPT = (MAX_BATCH + NT - 1) / NT;
    {
        int vals[IPT];
        int tsum = 0;
#pragma unroll
        for (int i = 0; i < IPT; ++i) {
            int idx = tid * IPT + i;
            int c = 0;
            if (idx < batch) {
                c = p.context_lens[idx];
                c = c < 0 ? 0 : c;
                ctxs[idx] = c;
            }
            vals[i] = (c + CHUNK - 1) / CHUNK;
            tsum += vals[i];
        }
        int inc = tsum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int nb = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += nb;
        }
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        int woff = 0, total = 0;
#pragma unroll
        for (int w = 0; w < NWARPS; ++w) {
            int t = warp_tot[w];
            if (w < warp) woff += t;
            total += t;
        }
        int excl = woff + inc - tsum;
#pragma unroll
        for (int i = 0; i < IPT; ++i) {
            int idx = tid * IPT + i;
            if (idx < batch) cum[idx] = excl;
            excl += vals[i];
        }
        if (tid == 0) cum[batch] = total;
        __syncthreads();
    }

    // everything above read only step metadata uploaded by the host before the first kernel of the step; q, the KV
    // pages written by this step and the output buffer belong to the previous kernels: wait for them here (PDL flavour)
    B200_PDL_WAIT();
    for (int b = blockIdx.x; b < batch; b += gridDim.x) {     // graph-padding rows produce zeros
        if (ctxs[b] == 0) {
            const int n16 = hkv * G * (B200_HEAD_DIM / 8);
            uint4* o4 = reinterpret_cast<uint4*>(p.out + (int64_t)b * p.out_stride);
            for (int i = tid; i < n16; i += NT) o4[i] = make_uint4(0, 0, 0, 0);
        }
    }

    const long long C = (long long)hkv * cum[batch];
    const int TW = gridDim.x * NWARPS;
    const int gw = warp * gridDim.x + blockIdx.x;
    if (C == 0) return;
    long long TWe = (C + MIN_CHUNKS - 1) / MIN_CHUNKS;
    TWe = TWe < TW ? TWe : (long long)TW;
    if (gw >= TWe) return;
    const long long c_begin = (long long)gw * C / TWe;
    const long long c_end = (long long)(gw + 1) * C / TWe;
    const int n_local = (int)(c_end - c_begin);

    ChunkCursor pi, ci;
    pi.seek(cum, ctxs, batch, hkv, c_begin);
    ci = pi;
    const int bs_mask = (1 << p.block_shift) - 1;

    int pg_next = 0;
    if (lane == 0) pg_next = p.block_tables[(int64_t)pi.b * p.bt_stride + ((pi.ck * CHUNK) >> p.block_shift)];
    const uint64_t l2pol = l2_policy_evict_first();

    auto issue = [&](int i) {
        if (lane == 0) {
            const int slot = i % NSTAGES;
            const int tok0 = pi.ck * CHUNK;
            const long long row = layer_row0 + ((((long long)pg_next * hkv + pi.h) << p.block_shift) + (tok0 & bs_mask));
            const uint32_t bar = my_bars_u32 + slot * 8;
            const uint32_t dst = my_stages_u32 + slot * L::kStageBytes;
            const bool seg_first = (pi.ck == 0) || (i == 0);
            mbar_expect_tx(bar, KV_STAGE + (seg_first ? (uint32_t)L::kQBytes : 0u));
            tma_box(dst, &tm_k, bar, 0, (int)row, l2pol);
            tma_box(dst + HALF_BYTES, &tm_k, bar, 64, (int)row, l2pol);
            tma_box(dst + 2 * HALF_BYTES, &tm_v, bar, 0, (int)row, l2pol);
            tma_box(dst + 3 * HALF_BYTES, &tm_v, bar, 64, (int)row, l2pol);
            if (seg_first)
                bulk_g2s(dst + KV_STAGE, p.q + (int64_t)pi.b * p.q_stride + pi.h * G * B200_HEAD_DIM, L::kQBytes, bar);
        }
        pi.advance(cum, ctxs, batch, hkv);
        if (lane == 0 && i + 1 < n_local)
            pg_next = p.block_tables[(int64_t)pi.b * p.bt_stride + ((pi.ck * CHUNK) >> p.block_shift)];
    };

    __syncwarp();
#pragma unroll 1
    for (int i = 0; i < NSTAGES - 1 && i < n_local; ++i) issue(i);

    const int g_ = lane >> 2;                 // row of the MMA tile this lane's C fragment holds = query head within the group
    const int t4 = lane & 3;
    const bool row_ok = g_ < G;
    const int mi = lane >> 3, r8 = lane & 7;  // ldmatrix: which 8x8 matrix / which of its rows this lane addresses

    uint32_t qa[8][2];                        // A fragments of q (rows 0..7 only), one pair per 16-wide k step
    float o[16][4];                           // C fragments of O: [d tile][..]; entries 2,3 (rows 8..15) stay zero
    float m_run = -INFINITY, l_run = 0.f;
    bool seg_start = true;

#pragma unroll 1
    for (int i = 0; i < n_local; ++i) {
        if (i + NSTAGES - 1 < n_local) issue(i + NSTAGES - 1);

        const int slot = i % NSTAGES;
        mbar_wait(my_bars_u32 + slot * 8, (i / NSTAGES) & 1);
        const uint32_t st = my_stages_u32 + slot * L::kStageBytes;
        uint8_t* st_ptr = my_stages + slot * L::kStageBytes;

        if (seg_start) {
            seg_start = false;
            const uint8_t* qrow = st_ptr + KV_STAGE + (row_ok ? g_ : 0) * ROW_BYTES;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                const uint32_t lo = *reinterpret_cast<const uint32_t*>(qrow + (ks * 16 + 2 * t4) * 2);
                const uint32_t hi = *reinterpret_cast<const uint32_t*>(qrow + (ks * 16 + 8 + 2 * t4) * 2);
                qa[ks][0] = row_ok ? lo : 0u;
                qa[ks][1] = row_ok ? hi : 0u;
            }
#pragma unroll
            for (int n = 0; n < 16; ++n) { o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f; }
            m_run = -INFINITY;
            l_run = 0.f;
        }

        int nvalid = ci.ctx - ci.ck * CHUNK;
        nvalid = nvalid > CHUNK ? CHUNK : nvalid;

        // ---- S = q K^T : 8 k-steps x 2 token tiles -----------------------------------------------------
        float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
        {
            const int row = r8 + (mi >> 1) * 8;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                const int chunk = (ks & 3) * 2 + (mi & 1);
                uint32_t b00, b01, b10, b11;
                ldsm4(st + (ks >> 2) * HALF_BYTES + row * 128 + ((chunk ^ (row & 7)) << 4), b00, b01, b10, b11);
                mma16816(s0, qa[ks][0], qa[ks][1], b00, b01);
                mma16816(s1, qa[ks][0], qa[ks][1], b10, b11);
            }
        }
        // this lane: row g_, tokens 2*t4, 2*t4+1 (s0) and 8+2*t4, 9+2*t4 (s1)
        float v0 = s0[0] * p.scale_log2, v1 = s0[1] * p.scale_log2, v2 = s1[0] * p.scale_log2, v3 = s1[1] * p.scale_log2;
        if (nvalid < CHUNK) {
            if (2 * t4 >= nvalid) v0 = -INFINITY;
            if (2 * t4 + 1 >= nvalid) v1 = -INFINITY;
            if (8 + 2 * t4 >= nvalid) v2 = -INFINITY;
            if (9 + 2 * t4 >= nvalid) v3 = -INFINITY;
            // rows the sequence does not own yet hold stale bytes: zero them in V so that 0 * garbage stays 0
            for (int r = nvalid + (lane >> 4); r < CHUNK; r += 2)
                *reinterpret_cast<uint4*>(st_ptr + 2 * HALF_BYTES + ((lane >> 3) & 1) * HALF_BYTES + r * 128 + ((lane & 7) << 4)) = make_uint4(0, 0, 0, 0);
            __syncwarp();
        }
        float mx = fmaxf(fmaxf(v0, v1), fmaxf(v2, v3));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run, mx);                  // finite: token 0 of every chunk is valid
        const float alpha = fast_exp2(m_run - m_new);
        const float p0 = fast_exp2(v0 - m_new), p1 = fast_exp2(v1 - m_new), p2 = fast_exp2(v2 - m_new), p3 = fast_exp2(v3 - m_new);
        m_run = m_new;
        l_run = l_run * alpha + (p0 + p1) + (p2 + p3);
        const uint32_t pa0 = pack_bf16x2(p0, p1), pa2 = pack_bf16x2(p2, p3);
#pragma unroll
        for (int n = 0; n < 16; ++n) { o[n][0] *= alpha; o[n][1] *= alpha; }

        // ---- O += P V : 16 d-tiles, one 16-token k step -------------------------------------------------
        {
            const int row = r8 + (mi & 1) * 8;
#pragma unroll
            for (int np = 0; np < 8; ++np) {
                const int chunk = 2 * np + (mi >> 1);           // 16-byte column chunk 0..15 over the 128 dims
                uint32_t b0, b1, b2, b3;
                ldsm4t(st + 2 * HALF_BYTES + (chunk >> 3) * HALF_BYTES + row * 128 + (((chunk & 7) ^ (row & 7)) << 4), b0, b1, b2, b3);
                mma16816(o[2 * np], pa0, pa2, b0, b1);
                mma16816(o[2 * np + 1], pa0, pa2, b2, b3);
            }
        }
        if (nvalid < CHUNK) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // our zero stores vs the next TMA box
        __syncwarp();   // every lane is done with this stage

        // ---- end of a segment ----------------------------------------------------------------------------
        const bool pair_done = (ci.ck == ci.n - 1);
        if (pair_done || i == n_local - 1) {
            float l_tot = l_run;
            l_tot += __shfl_xor_sync(0xffffffffu, l_tot, 1);
            l_tot += __shfl_xor_sync(0xffffffffu, l_tot, 2);
            const int pair = ci.b * hkv + ci.h;
            const long long c0 = (long long)hkv * cum[ci.b] + (long long)ci.h * ci.n;
            const long long c1 = c0 + ci.n;
            const int w_first = (int)(((c0 + 1) * TWe - 1) / C);
            const int w_last = (int)((c1 * TWe - 1) / C);
            const int nseg = w_last - w_first + 1;
            __nv_bfloat16* orow = p.out + (int64_t)ci.b * p.out_stride + (ci.h * G + g_) * B200_HEAD_DIM + 2 * t4;
            if (nseg == 1) {
                if (row_ok) {
                    const float inv = 1.f / l_tot;
#pragma unroll
                    for (int n = 0; n < 16; ++n)
                        *reinterpret_cast<uint32_t*>(orow + n * 8) = pack_bf16x2(o[n][0] * inv, o[n][1] * inv);
                }
            } else {
                const int myslot = (gw == w_first) ? TW + pair : gw;
                if (row_ok) {
                    float* po = p.part_o + ((int64_t)myslot * G + g_) * B200_HEAD_DIM + 2 * t4;
#pragma unroll
                    for (int n = 0; n < 16; ++n) *reinterpret_cast<float2*>(po + n * 8) = make_float2(o[n][0], o[n][1]);
                    if (t4 == 0) *reinterpret_cast<float2*>(p.part_ml + ((int64_t)myslot * G + g_) * 2) = make_float2(m_run, l_tot);
                }
                __threadfence();
                __syncwarp();
                int old = 0;
                if (lane == 0) old = atomicAdd(p.counters + pair, 1);
                old = __shfl_sync(0xffffffffu, old, 0);
                if (old == nseg - 1) {
                    __threadfence();
                    if (row_ok) {
                        float M = -INFINITY, Ls = 0.f;
                        float r[32];
#pragma unroll
                        for (int e = 0; e < 32; ++e) r[e] = 0.f;
#pragma unroll 2
                        for (int k = 0; k < nseg; ++k) {
                            const int sl = k == 0 ? TW + pair : w_first + k;
                            const float2 ml = __ldcg(reinterpret_cast<const float2*>(p.part_ml + ((int64_t)sl * G + g_) * 2));
                            const float* src = p.part_o + ((int64_t)sl * G + g_) * B200_HEAD_DIM + 2 * t4;
                            const float Mn = fmaxf(M, ml.x);
                            const float so = fast_exp2(M - Mn), sn = fast_exp2(ml.x - Mn);
                            M = Mn;
                            Ls = Ls * so + ml.y * sn;
#pragma unroll
                            for (int n = 0; n < 16; ++n) {
                                const float2 x = __ldcg(reinterpret_cast<const float2*>(src + n * 8));
                                r[2 * n] = r[2 * n] * so + x.x * sn;
                                r[2 * n + 1] = r[2 * n + 1] * so + x.y * sn;
                            }
                        }
                        const float inv = 1.f / Ls;
#pragma unroll
                        for (int n = 0; n < 16; ++n)
                            *reinterpret_cast<uint32_t*>(orow + n * 8) = pack_bf16x2(r[2 * n] * inv, r[2 * n + 1] * inv);
                    }
                    if (lane == 0) p.counters[pair] = 0;
                }
            }
            seg_start = true;
        }
        ci.advance(cum, ctxs, batch, hkv);
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

bool make_chunk_map(CUtensorMap* m, const void* base, uint64_t rows) {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            return false;
        fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    cuuint64_t dims[2] = {B200_HEAD_DIM, rows};
    cuuint64_t strides[1] = {ROW_BYTES};
    cuuint32_t box[2] = {64, CHUNK};
    cuuint32_t estr[2] = {1, 1};
    return fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int G>
int launch_mma(b200_ctx* ctx, const CUtensorMap& tk, const CUtensorMap& tv, const DecodeParams& prm, long long row0, cudaStream_t st) {
    using L = MmaSmem<G>;
    static_assert(L::kTotal <= 227 * 1024, "decode (mma) shared memory exceeds the sm_90 opt-in limit");
    auto kern = paged_decode_mma_kernel<G>;
    static B200SmemOptIn optin;
    B200_CUDA_CHECK(ctx, optin.ensure(kern, L::kTotal));
    B200_LAUNCH((kern), ctx->sm_count, MMA_WARPS * 32, L::kTotal, st, tk, tv, prm, row0);
    return b200_launch_status(ctx);
}

}  // namespace

// Called from decode_common() in decode_attn.cu.  prm.k_layer / v_layer are ignored: the tensor maps cover the whole
// cache and `layer` selects the rows.
int b200_decode_mma_launch(b200_ctx* ctx, int layer, const DecodeParams& prm, int G, cudaStream_t stream) {
    // the maps depend only on the bound cache: build them once per binding
    static CUtensorMap tk, tv;
    static uint64_t built_for = 0;
    const uint64_t rows = (uint64_t)ctx->layers * ctx->num_blocks * ctx->num_kv_heads * ctx->block_size;
    if (rows >= (1ull << 31)) return B200_EUNSUPPORTED;
    if (built_for != ctx->bind_gen) {
        if (!make_chunk_map(&tk, ctx->k_base, rows) || !make_chunk_map(&tv, ctx->v_base, rows)) return B200_EUNSUPPORTED;
        built_for = ctx->bind_gen;
    }
    const long long row0 = (long long)layer * ctx->num_blocks * ctx->num_kv_heads * ctx->block_size;
    switch (G) {
        case 1: return launch_mma<1>(ctx, tk, tv, prm, row0, stream);
        case 2: return launch_mma<2>(ctx, tk, tv, prm, row0, stream);
        case 4: return launch_mma<4>(ctx, tk, tv, prm, row0, stream);
        case 8: return launch_mma<8>(ctx, tk, tv, prm, row0, stream);
        default: return B200_EUNSUPPORTED;
    }
}
