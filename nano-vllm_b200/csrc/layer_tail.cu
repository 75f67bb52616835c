// The tail of a decoder layer in a decode step as ONE persistent kernel (wgmma + TMA, grid-wide barriers between phases):
//
//     o_proj  ->  residual add + RMSNorm  ->  gate_up_proj + SiluAndMul  ->  down_proj  ->  residual add + RMSNorm
//                                                                                       [ ->  next layer's qkv_proj ]
//
// Replaces, for a batch of <= 256 rows on one GPU, six to seven dependent launches of the step -- RowParallelLinear o_proj
// (reference models/qwen3.py:87, layers/linear.py:131-156), RMSNorm.add_rms_forward (layers/layernorm.py:28-40),
// MergedColumnParallelLinear gate_up_proj + SiluAndMul (models/qwen3.py:91-117, layers/activation.py:8-11), down_proj, the
// next layer's input_layernorm and its QKVParallelLinear (models/qwen3.py:146-159, 72-76).  Why: in a captured decode step
// every one of those kernels costs a launch, a fill and a drain whatever it computes, while the weights they read would
// stream from HBM in a few microseconds for all of them together.  A grid-wide barrier inside a resident kernel is cheaper
// than a launch, and the TMA producer keeps running across it.
//
// Structure: grid = one CTA per SM (all co-resident: cooperative launch), 160 threads:
//   warps 0-3  one warpgroup: wgmma m64n64k16 on both 64-row halves of an item (fp32 accumulator [128][64] in registers),
//              frees ring slots once the MMAs that read them have retired, then epilogue / normalisation
//   warp 4     TMA producer: a ring of 8 x {x tile [128 rows][64 k], W tile [64 n][64 k]} (128-byte swizzle)
// GEMM phases walk "items" = (row block, 64-column block, k split); split-K partial sums go to an fp32 workspace and are
// added IN SPLIT ORDER by the normalisation phase that follows (deterministic; the projection is rounded to bf16 exactly
// where the reference's F.linear output is bf16).  Phase outputs written with ordinary stores are read by later phases
// through TMA: writers issue fence.proxy.async + __threadfence before arriving at the grid barrier.
#include <type_traits>

#include "tc_common.cuh"

namespace {

using namespace b200tc;

constexpr int LT_THREADS = 160;
constexpr int LT_BM = 128, LT_BN = 64, LT_BK = 64;
constexpr uint32_t LT_XT = LT_BM * 128;            // 16 KB
constexpr uint32_t LT_WT = LT_BN * 128;            // 8 KB
constexpr uint32_t LT_STAGE = LT_XT + LT_WT;       // 24 KB
constexpr int LT_STAGES = 8;
constexpr uint32_t LT_OFF_BAR = LT_STAGES * LT_STAGE;
constexpr uint32_t LT_SMEM = LT_OFF_BAR + 256;     // full[8], empty[8], entry generation

enum { LT_EPI_PARTIAL = 0, LT_EPI_SILU = 1, LT_EPI_BF16 = 2 };

struct LtGemm {
    int n_blocks;          // output column blocks (64 accumulator columns each; 32 output columns for SILU)
    int row_blocks;        // ceil(rows / 128)
    int splits;            // k splits (1 unless PARTIAL)
    int k_tiles;           // 64-wide k tiles per split
    int epi;
    int up_row0;           // SILU: first W row of the "up" half
    void* out;             // PARTIAL: fp32 [splits][rows][n]; SILU / BF16: bf16 [rows][out_stride]
    int64_t out_stride;    // elements between output rows
    int wait_barrier;      // grid barrier this phase's x operand depends on (-1: produced by the previous kernel)
};

struct LtParams {
    LtGemm g[4];           // o_proj, gate_up, down, next qkv (n_blocks == 0: absent)
    int rows, hidden;
    float eps;
    __nv_bfloat16* residual;
    const __nv_bfloat16* ln_mid;       // post_attention_layernorm weight
    const __nv_bfloat16* ln_next;      // next layer's input_layernorm (or the final norm) weight
    __nv_bfloat16* xbuf;               // [rows][hidden]: normalised input of gate_up
    __nv_bfloat16* x_next;             // [rows][hidden]: normalised input of the next layer
    const float* partials;             // the PARTIAL phases' output, as read by the normalisation phases
    unsigned int* bar_count;
    unsigned int* bar_gen;
    int* err;
};

__device__ __forceinline__ void tma_load_2d_hint(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;" ::
            "r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "l"(policy)
        : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void epi_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }      // the four epilogue warps

// ---- grid-wide barrier: monotonic generation counter; every CTA arrives exactly once per barrier ------------------------
__device__ __forceinline__ void grid_arrive(const LtParams& p) {
    asm volatile("fence.proxy.async;" ::: "memory");     // this CTA's plain stores, before other SMs' TMA reads of them
    __threadfence();
    if (atomicAdd(p.bar_count, 1u) == gridDim.x - 1) {
        atomicExch(p.bar_count, 0u);
        __threadfence();
        atomicAdd(p.bar_gen, 1u);
    }
}
// waits until `target` barriers (counted from p.bar_gen at kernel entry = base) have completed; bounded, like every spin in
// this library: a CTA that never shows up (a launch that is not fully co-resident) raises *err instead of wedging the GPU
__device__ __forceinline__ void grid_wait(const LtParams& p, unsigned int base, int index) {
    const unsigned int target = base + (unsigned int)index + 1u;
    const long long t0 = clock64();
    while ((int)(ld_acquire_gpu(p.bar_gen) - target) < 0) {
        if (clock64() - t0 > (1ll << 32)) {
            if (p.err) atomicExch(p.err, 1);
            break;
        }
    }
    asm volatile("fence.proxy.async;" ::: "memory");
}

__device__ __forceinline__ void item_coords(const LtGemm& g, int item, int& rb, int& nb, int& s) {
    s = item % g.splits;
    const int t = item / g.splits;
    nb = t % g.n_blocks;
    rb = t / g.n_blocks;
}

// residual <- bf16(h + residual) with h = bf16(sum_s partials[s]) (split order);  out <- bf16((h + residual) * rstd * w)
// RMSNorm.add_rms_forward (layers/layernorm.py:28-40): variance and normalisation use the UN-rounded fp32 sum.  One warp
// per row, two passes over the row (the partials are L2 resident): pass one the sum of squares, pass two the outputs.
__device__ __forceinline__ void lt_row_sum(const float* prow, int64_t split_stride, int splits, const uint4* r4, int idx, float (&v)[8]) {
    float h[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < splits; ++s) {
        const float4* q = reinterpret_cast<const float4*>(prow + s * split_stride) + idx * 2;
        const float4 a = __ldcg(q), b = __ldcg(q + 1);
        h[0] += a.x; h[1] += a.y; h[2] += a.z; h[3] += a.w;
        h[4] += b.x; h[5] += b.y; h[6] += b.z; h[7] += b.w;
    }
    float r[8];
    unpack8(r4[idx], r);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = round_bf16(h[e]) + r[e];
}
__device__ __forceinline__ void norm_rows(const LtParams& p, int splits, const __nv_bfloat16* __restrict__ w, __nv_bfloat16* out,
                                          int warp, int lane) {
    const int cols = p.hidden, nvec = cols >> 3;
    const int64_t split_stride = (int64_t)p.rows * cols;
    const uint4* w4 = reinterpret_cast<const uint4*>(w);
    for (int row = blockIdx.x * 4 + warp; row < p.rows; row += gridDim.x * 4) {
        const float* prow = p.partials + (int64_t)row * cols;
        uint4* r4 = reinterpret_cast<uint4*>(p.residual + (int64_t)row * cols);
        uint4* o4 = reinterpret_cast<uint4*>(out + (int64_t)row * cols);
        float ss = 0.f;
        for (int idx = lane; idx < nvec; idx += 32) {
            float v[8];
            lt_row_sum(prow, split_stride, splits, r4, idx, v);
#pragma unroll
            for (int e = 0; e < 8; ++e) ss = fmaf(v[e], v[e], ss);
        }
        ss = warp_sum(ss);
        const float rstd = 1.0f / sqrtf(ss / (float)cols + p.eps);
        for (int idx = lane; idx < nvec; idx += 32) {
            float v[8], wf[8], y[8];
            lt_row_sum(prow, split_stride, splits, r4, idx, v);      // the old residual: each vector is rewritten only below
            unpack8(w4[idx], wf);
#pragma unroll
            for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(__fmul_rn(v[e], rstd), wf[e]);
            r4[idx] = pack8(v);
            o4[idx] = pack8(y);
        }
    }
}

__global__ void __launch_bounds__(LT_THREADS, 1)
layer_tail_kernel(const __grid_constant__ CUtensorMap tm_x0, const __grid_constant__ CUtensorMap tm_w0,
                  const __grid_constant__ CUtensorMap tm_x1, const __grid_constant__ CUtensorMap tm_w1,
                  const __grid_constant__ CUtensorMap tm_x2, const __grid_constant__ CUtensorMap tm_w2,
                  const __grid_constant__ CUtensorMap tm_x3, const __grid_constant__ CUtensorMap tm_w3, const LtParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t base = smem_u32(smem_raw);
    if (base & 1023u) __trap();
    const uint32_t bars = base + LT_OFF_BAR;                   // full[i] = bars + 8 i, empty[i] = bars + 64 + 8 i

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    volatile uint32_t* gen_slot = reinterpret_cast<volatile uint32_t*>(smem_raw + LT_OFF_BAR + 152);

    if (tid == 0) {
        // the barrier generation at kernel entry, read ONCE per CTA before the set-up __syncthreads (hence before this
        // CTA's first arrival, so no barrier of this launch can have completed) and shared through smem: a thread that
        // read it on its own, later, could already see barrier 0 completed and would wait for one barrier too many
        *gen_slot = ld_acquire_gpu(p.bar_gen);
        for (int i = 0; i < LT_STAGES; ++i) mbar_init(bars + i * 8, 1);
        for (int i = LT_STAGES; i < 2 * LT_STAGES; ++i) mbar_init(bars + i * 8, 4);     // one arrival per MMA warp
        mbar_fence_init();
    }
    __syncthreads();
    const unsigned int gen0 = *gen_slot;

    const CUtensorMap* const mx[4] = {&tm_x0, &tm_x1, &tm_x2, &tm_x3};
    const CUtensorMap* const mw[4] = {&tm_w0, &tm_w1, &tm_w2, &tm_w3};

    if (warp == 4) {
        // ---- TMA producer --------------------------------------------------------------------------------------------
        if (lane == 0) {
            const uint64_t pol = l2_policy_evict_first();
            uint32_t pc = 0;                                    // k tiles produced so far (all phases)
            for (int ph = 0; ph < 4; ++ph) {
                const LtGemm& g = p.g[ph];
                if (g.n_blocks == 0) continue;
                if (g.wait_barrier >= 0) grid_wait(p, gen0, g.wait_barrier);
                const int items = g.row_blocks * g.n_blocks * g.splits;
                for (int item = blockIdx.x; item < items; item += gridDim.x) {
                    int rb, nb, s;
                    item_coords(g, item, rb, nb, s);
                    for (int kt = 0; kt < g.k_tiles; ++kt, ++pc) {
                        const int slot = pc % LT_STAGES;
                        if (pc >= (uint32_t)LT_STAGES) mbar_wait(bars + 64 + slot * 8, ((pc / LT_STAGES) - 1) & 1);
                        const uint32_t full = bars + slot * 8;
                        const uint32_t xs = base + slot * LT_STAGE, ws = xs + LT_XT;
                        const int kc = (s * g.k_tiles + kt) * LT_BK;
                        mbar_expect_tx(full, LT_STAGE);
                        if (g.epi == LT_EPI_SILU) {
                            tma_load_2d_hint(ws, mw[ph], full, kc, nb * 32, pol);
                            tma_load_2d_hint(ws + 32 * 128, mw[ph], full, kc, g.up_row0 + nb * 32, pol);
                        } else {
                            tma_load_2d_hint(ws, mw[ph], full, kc, nb * LT_BN, pol);
                        }
                        tma_load_2d(xs, mx[ph], full, kc, rb * LT_BM);
                    }
                }
            }
        }
    } else {
        // ---- MMA + epilogue + normalisation warpgroup (warps 0-3) --------------------------------------------------------
        // acc[h][4c + 2r + e] = D[64 h + 16 warp + g + 8 r][8 c + 2 qd + e]
        const int g8 = lane >> 2, qd = lane & 3;
        uint32_t cc = 0;                                        // k tiles consumed (all phases)
        int next_barrier = 0;
        for (int ph = 0; ph < 4; ++ph) {
            const LtGemm& g = p.g[ph];
            if (g.n_blocks == 0) continue;
            const int items = g.row_blocks * g.n_blocks * g.splits;
            for (int item = blockIdx.x; item < items; item += gridDim.x) {
                int rb, nb, s;
                item_coords(g, item, rb, nb, s);
                const bool two_halves = p.rows - rb * LT_BM > 64;
                float acc[2][LT_BN / 2];
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int c = 0; c < LT_BN / 2; ++c) acc[h][c] = 0.f;
                // the row-half decision is taken once, outside the MMA loop, so that every wgmma sequence is straight-line code
                auto consume = [&](auto two) {
                    constexpr bool TWO = decltype(two)::value;
                    for (int kt = 0; kt < g.k_tiles; ++kt, ++cc) {
                        const int slot = cc % LT_STAGES;
                        mbar_wait(bars + slot * 8, (cc / LT_STAGES) & 1);
                        const uint32_t xs = base + slot * LT_STAGE, ws = xs + LT_XT;
                        wg_fence();
#pragma unroll
                        for (int ks = 0; ks < LT_BK / 16; ++ks) {
                            const uint64_t bdesc = make_desc(ws + ks * 32, 16, 1024);
                            wgmma_ss<LT_BN>(acc[0], make_desc(xs + ks * 32, 16, 1024), bdesc, 1u);
                            if constexpr (TWO) wgmma_ss<LT_BN>(acc[1], make_desc(xs + 64 * 128 + ks * 32, 16, 1024), bdesc, 1u);
                        }
                        wg_commit();
                        wg_wait<0>();
                        __syncwarp();
                        if (lane == 0) mbar_arrive(bars + 64 + slot * 8);
                    }
                };
                if (two_halves) consume(std::true_type{});
                else consume(std::false_type{});
                acc_fence(acc[0]);
                acc_fence(acc[1]);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const int row = rb * LT_BM + 64 * h + 16 * warp + g8 + 8 * r;
                        if (row >= p.rows) continue;
                        if (g.epi == LT_EPI_PARTIAL) {
                            float* dst = static_cast<float*>(g.out) + ((int64_t)s * p.rows + row) * g.out_stride + nb * LT_BN + 2 * qd;
#pragma unroll
                            for (int c = 0; c < LT_BN / 8; ++c)
                                *reinterpret_cast<float2*>(dst + 8 * c) = make_float2(acc[h][4 * c + 2 * r], acc[h][4 * c + 2 * r + 1]);
                        } else if (g.epi == LT_EPI_SILU) {
                            __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(g.out) + (int64_t)row * g.out_stride + nb * 32 + 2 * qd;
#pragma unroll
                            for (int c = 0; c < 4; ++c) {
                                float y[2];
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    const float gt = round_bf16(acc[h][4 * c + 2 * r + e]), up = round_bf16(acc[h][4 * (c + 4) + 2 * r + e]);
                                    y[e] = __fmul_rn(gt / (1.0f + expf(-gt)), up);
                                }
                                *reinterpret_cast<uint32_t*>(dst + 8 * c) = pack_bf16x2(y[0], y[1]);
                            }
                        } else {
                            __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(g.out) + (int64_t)row * g.out_stride + nb * LT_BN + 2 * qd;
#pragma unroll
                            for (int c = 0; c < LT_BN / 8; ++c)
                                *reinterpret_cast<uint32_t*>(dst + 8 * c) = pack_bf16x2(acc[h][4 * c + 2 * r], acc[h][4 * c + 2 * r + 1]);
                        }
                    }
                }
            }
            if (ph == 3) break;                                 // the qkv phase is the last one: nothing waits for it in this kernel
            // this CTA's share of the phase is written: arrive, then (after o_proj and after down_proj) normalise.  Every
            // writer orders its own plain stores before later async-proxy (TMA) reads of them by other SMs.
            asm volatile("fence.proxy.async;" ::: "memory");
            epi_sync();
            // A CTA never arrives at barrier k+1 before barrier k has completed: the arrival counter is reset by the
            // last arriver of k, and an early arrival for k+1 could fall between its last increment and that reset.
            if (tid == 0) {
                if (next_barrier > 0) grid_wait(p, gen0, next_barrier - 1);
                grid_arrive(p);
            }
            const int b_written = next_barrier++;
            if (ph == 0 || ph == 2) {
                if (tid == 0) grid_wait(p, gen0, b_written);
                epi_sync();
                norm_rows(p, g.splits, ph == 0 ? p.ln_mid : p.ln_next, ph == 0 ? p.xbuf : p.x_next, warp, lane);
                asm volatile("fence.proxy.async;" ::: "memory");
                epi_sync();
                if (tid == 0) grid_arrive(p);                   // barrier b_written has completed (waited for above)
                next_barrier++;
            }
        }
    }
}

}  // namespace

// linear_tc.cu owns the tensor-map cache
bool b200_cached_tensor_map(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t stride, uint32_t box_rows);

extern "C" size_t b200_layer_tail_workspace_bytes(int max_rows, int hidden, int inter, int max_splits) {
    if (max_rows <= 0 || hidden <= 0 || inter <= 0 || max_splits <= 0) return 0;
    size_t b = 256;                                                        // barrier count, generation, error flag
    b += (size_t)max_splits * max_rows * hidden * 4;                       // fp32 split-K partials (o_proj and down_proj in turn)
    b += (size_t)max_rows * hidden * 2;                                    // xbuf
    b += (size_t)max_rows * inter * 2;                                     // act
    return (b + 255) / 256 * 256;
}

extern "C" int b200_layer_tail(b200_ctx* ctx, const void* attn_out, int64_t attn_stride0, void* residual, const void* w_o, const void* ln_mid,
                               const void* w_gate_up, const void* w_down, const void* ln_next, void* x_next, const void* w_qkv_next,
                               void* qkv_out, int64_t qkv_stride0, int qkv_n, void* workspace, size_t workspace_bytes, int rows, int hidden,
                               int q_size, int inter, float eps, int splits_o, int splits_down, void* stream) {
    if (!ctx || !attn_out || !residual || !w_o || !ln_mid || !w_gate_up || !w_down || !ln_next || !x_next || !workspace) return B200_EINVAL;
    if (rows < 0 || hidden <= 0 || q_size <= 0 || inter <= 0 || splits_o < 1 || splits_down < 1) return B200_EINVAL;
    if (rows == 0) return B200_OK;
    if (hidden % 64 || q_size % 64 || inter % 64 || (inter % 32) || rows > 1024) return B200_EUNSUPPORTED;
    if ((q_size / 64) % splits_o || (inter / 64) % splits_down) return B200_EUNSUPPORTED;
    if ((attn_stride0 % 8) || ((uintptr_t)attn_out & 15) || ((uintptr_t)residual & 15) || ((uintptr_t)x_next & 15) || ((uintptr_t)workspace & 255))
        return B200_EINVAL;
    if (w_qkv_next && (!qkv_out || qkv_n <= 0 || qkv_n % 64 || (qkv_stride0 % 8) || ((uintptr_t)qkv_out & 15))) return B200_EINVAL;
    const int max_splits = splits_o > splits_down ? splits_o : splits_down;
    if (workspace_bytes < b200_layer_tail_workspace_bytes(rows, hidden, inter, max_splits)) return B200_EWORKSPACE;

    uint8_t* ws = static_cast<uint8_t*>(workspace);
    unsigned int* bar = reinterpret_cast<unsigned int*>(ws);
    float* partials = reinterpret_cast<float*>(ws + 256);
    __nv_bfloat16* xbuf = reinterpret_cast<__nv_bfloat16*>(ws + 256 + (size_t)max_splits * rows * hidden * 4);
    __nv_bfloat16* act = xbuf + (size_t)rows * hidden;

    CUtensorMap m[8];
    const int rb = (rows + LT_BM - 1) / LT_BM;
    bool ok = b200_cached_tensor_map(&m[0], attn_out, (uint64_t)q_size, (uint64_t)rows, (uint64_t)attn_stride0, LT_BM) &&
              b200_cached_tensor_map(&m[1], w_o, (uint64_t)q_size, (uint64_t)hidden, (uint64_t)q_size, LT_BN) &&
              b200_cached_tensor_map(&m[2], xbuf, (uint64_t)hidden, (uint64_t)rows, (uint64_t)hidden, LT_BM) &&
              b200_cached_tensor_map(&m[3], w_gate_up, (uint64_t)hidden, (uint64_t)2 * inter, (uint64_t)hidden, 32) &&
              b200_cached_tensor_map(&m[4], act, (uint64_t)inter, (uint64_t)rows, (uint64_t)inter, LT_BM) &&
              b200_cached_tensor_map(&m[5], w_down, (uint64_t)inter, (uint64_t)hidden, (uint64_t)inter, LT_BN);
    if (ok && w_qkv_next)
        ok = b200_cached_tensor_map(&m[6], x_next, (uint64_t)hidden, (uint64_t)rows, (uint64_t)hidden, LT_BM) &&
             b200_cached_tensor_map(&m[7], w_qkv_next, (uint64_t)hidden, (uint64_t)qkv_n, (uint64_t)hidden, LT_BN);
    if (!ok) return B200_EUNSUPPORTED;
    if (!w_qkv_next) { m[6] = m[2]; m[7] = m[1]; }

    LtParams p = {};
    p.g[0] = {hidden / LT_BN, rb, splits_o, q_size / 64 / splits_o, LT_EPI_PARTIAL, 0, partials, hidden, -1};
    p.g[1] = {inter / 32, rb, 1, hidden / 64, LT_EPI_SILU, inter, act, inter, 1};          // x = xbuf: after the first normalisation
    p.g[2] = {hidden / LT_BN, rb, splits_down, inter / 64 / splits_down, LT_EPI_PARTIAL, 0, partials, hidden, 2};
    p.g[3] = {w_qkv_next ? qkv_n / LT_BN : 0, rb, 1, hidden / 64, LT_EPI_BF16, 0, qkv_out, qkv_stride0, 4};
    p.rows = rows;
    p.hidden = hidden;
    p.eps = eps;
    p.residual = static_cast<__nv_bfloat16*>(residual);
    p.ln_mid = static_cast<const __nv_bfloat16*>(ln_mid);
    p.ln_next = static_cast<const __nv_bfloat16*>(ln_next);
    p.xbuf = xbuf;
    p.x_next = static_cast<__nv_bfloat16*>(x_next);
    p.partials = partials;
    p.bar_count = bar;
    p.bar_gen = bar + 1;
    p.err = reinterpret_cast<int*>(bar + 2);

    static B200SmemOptIn optin;
    B200_CUDA_CHECK(ctx, optin.ensure(layer_tail_kernel, LT_SMEM));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(ctx->sm_count);
    cfg.blockDim = dim3(LT_THREADS);
    cfg.dynamicSmemBytes = LT_SMEM;
    cfg.stream = static_cast<cudaStream_t>(stream);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;          // all CTAs co-resident: the grid barriers cannot deadlock
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    B200_CUDA_CHECK(ctx, cudaLaunchKernelEx(&cfg, layer_tail_kernel, m[0], m[1], m[2], m[3], m[4], m[5], m[6], m[7], p));
    return b200_launch_status(ctx);
}
