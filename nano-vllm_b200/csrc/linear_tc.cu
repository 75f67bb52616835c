// Small-batch linear layers y = x W^T on Hopper's tensor cores (wgmma), with the op that follows fused in.
//
// On the product path for o_proj / down_proj of decode batches <= 128 rows (split-K) and for all four projections of the
// two-stream decode step (models/qwen3.py::_forward_dual), where a shallow ring lets these CTAs share an SM with the
// attention kernel.
//
// Why: in a decode step the four projections of a layer (reference layers/linear.py:51,73,153 -> F.linear -> cuBLAS)
// cost several microseconds each whatever the batch is, well above the time their weights need to stream from HBM, and
// the elementwise kernels between them sit at the floor of a tiny launch.  The levers are
//   * weights do not depend on the previous kernel: each CTA starts streaming its W tiles before
//     griddepcontrol.wait (programmatic dependent launch), so the HBM-bound part runs under the predecessor;
//   * SiluAndMul (layers/activation.py:8-11) becomes the epilogue of the gate_up projection: a CTA owns BN/2 gate
//     columns and the matching BN/2 up columns, so the [rows, 2*inter] intermediate never exists;
//   * the two N = hidden projections (o_proj, down_proj) split K over CTAs so that all SMs stream weights; the
//     fp32 partials are summed IN ORDER (deterministic) by the add+RMSNorm that follows anyway
//     (b200_add_rmsnorm_partials), which rounds the sum to bf16 exactly where the reference's GEMM output is bf16.
//
// Kernel: one CTA = 128 rows of x (two wgmma m64 halves; rows beyond `rows` are zero-filled by TMA and never stored, and
// the second half is skipped when the CTA has <= 64 rows) x BN output columns x a contiguous range of 64-wide k tiles.
// Warp 4 / lane 0 feeds a STAGES-deep ring of {x tile [128][64], W tile [BN][64]} by TMA (128-byte swizzle, W with an
// L2 evict_first policy: read once per step); warps 0-3 (one warpgroup) issue wgmma (both operands K-major, fp32
// accumulator in registers), release ring slots once the MMAs that read them have retired, and run the epilogue.
#include <mutex>
#include <type_traits>
#include <unordered_map>

#include "sample_common.cuh"
#include "tc_common.cuh"

namespace {

using namespace b200tc;

constexpr int LM = 128;                   // rows of x per CTA (two wgmma m64 halves)
constexpr int LK = 64;                    // k extent of a ring slot: one 128-byte swizzle atom of bf16
constexpr int L_THREADS = 160;            // warpgroup 0 = MMA + epilogue, warp 4 = TMA producer
constexpr uint32_t X_TILE = LM * 128;     // 16 KB
constexpr uint32_t X_HALF = 64 * 128;     // 8 KB: rows [64, 128) of the x tile

enum { EPI_BF16 = 0, EPI_SILU = 1, EPI_PARTIAL = 2, EPI_SAMPLE = 3 };

// DEEP: as many ring slots as one CTA per SM allows (all of a short K in flight).  !DEEP: 4 slots for block_n <= 64, so
// that two CTAs fit an SM and a dependent kernel launched early (PDL) finds room to prefetch its weights.
template <int BN, bool DEEP>
struct Cfg {
    static constexpr uint32_t W_TILE = BN * 128;
    static constexpr uint32_t STAGE = X_TILE + W_TILE;
    static constexpr int STAGES = !DEEP ? (BN <= 64 ? 4 : 3) : (BN <= 32 ? 8 : (BN <= 64 ? 6 : 4));
    static constexpr uint32_t SMEM = STAGES * STAGE + 256;   // ring, then full[S], empty[S]
    // The ring depth actually used by a launch is LinParams::stages <= STAGES (b200_linear flags bits 4-7): the dynamic
    // shared memory of that launch is stages * STAGE + 256, so a shallow launch fits beside another kernel's CTA.
};

struct LinParams {
    void* out;                // bf16 [rows, n_out] (EPI_BF16 / EPI_SILU) or fp32 [splits, rows, n_out] (EPI_PARTIAL)
    int64_t out_stride;       // elements between rows of out
    int rows;                 // M
    int up_row0;              // EPI_SILU: first W row of the "up" half (= inter)
    int k_tiles;              // 64-wide k tiles per split (gridDim.z splits)
    int stages;               // ring slots of this launch (2 .. Cfg::STAGES)
    // EPI_SAMPLE (fused LM head + sampling): nothing of size [rows, vocab] is ever written
    int n_valid;                          // columns of this vocabulary shard (the last column block may be ragged)
    const float* temperatures;            // [rows] or null (greedy)
    int64_t index_offset;                 // first vocabulary id of the shard
    uint64_t seed, step;
    const int64_t* step_dev;              // optional device-side addend to step (CUDA-graph replays)
    unsigned long long* keys;             // [rows] running maximum of packed (score, token) keys; zero = empty
};

__device__ __forceinline__ void tma_load_2d_hint(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;" ::
            "r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "l"(policy)
        : "memory");
}
// x tile shared by the CL CTAs of a cluster (neighbouring column blocks, same rows of x): each CTA fetches 128 / CL rows
// and multicasts them into the same ring slot of every CTA of the cluster; each copy signals the mbarrier at the same
// offset in its destination CTA.  Cuts the L2 -> SM traffic of x by CL.
__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::
            "r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// ring slot `slot` is free again in this CTA's view: one arrival per consumer warp of every CTA that received multicast
// data in it (the producer of each CTA waits for all of them before it overwrites the slot everywhere)
template <int CL>
__device__ __forceinline__ void release_slot(uint32_t empty_bar, int lane) {
    __syncwarp();
    if constexpr (CL == 1) {
        if (lane == 0) mbar_arrive(empty_bar);
    } else {
        if (lane < CL) mbar_arrive_cluster(empty_bar, (uint32_t)lane);
    }
}

template <int BN, int EPI, bool DEEP, int CL>
__global__ void __launch_bounds__(L_THREADS, 1)
linear_tc_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w, const LinParams p) {
    using C = Cfg<BN, DEEP>;
    constexpr uint16_t CL_MASK = (uint16_t)((1u << CL) - 1);
    constexpr int X_ROWS = LM / CL;                            // rows of x this CTA fetches (and multicasts when CL > 1)
    const int S = p.stages;
    constexpr int BOUT = EPI == EPI_SILU ? BN / 2 : BN;       // output columns of this CTA
    extern __shared__ __align__(1024) uint8_t smem_raw[];     // 128-byte swizzle atoms need 1024-byte alignment
    const uint32_t base = smem_u32(smem_raw);
    if (base & 1023u) __trap();
    const uint32_t off_bar = (uint32_t)S * C::STAGE;
    const uint32_t bars = base + off_bar;                      // full[i] = bars + 8 i, empty[i] = bars + 8 (S + i)

    // let the next kernel of the stream start its own prologue (and weight prefetch) now; it still waits for this
    // grid to finish before it touches anything this grid writes (its own griddepcontrol.wait)
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int m0 = blockIdx.y * LM;
    const int kt0 = blockIdx.z * p.k_tiles;
    const int nk = p.k_tiles;
    const bool two_halves = p.rows - m0 > 64;                 // rows [64, 128) of this CTA exist

    const uint32_t crank = CL > 1 ? cluster_ctarank() : 0;
    if (tid == 0) {
        for (int i = 0; i < S; ++i) mbar_init(bars + i * 8, 1);                  // full: this CTA's own expect_tx arrival
        for (int i = S; i < 2 * S; ++i) mbar_init(bars + i * 8, 4 * CL);        // empty: every consumer warp of the cluster
        mbar_fence_init();
    }
    if constexpr (CL > 1) cluster_sync_all();      // peers' barriers exist before anything is multicast at them
    else __syncthreads();

    float acc[2][BN / 2];
    if (warp == 4) {
        // ---- TMA producer --------------------------------------------------------------------------------
        if (lane == 0) {
            const uint64_t pol = l2_policy_evict_first();
            auto load_w = [&](int slot, int kt) {
                const uint32_t dst = base + slot * C::STAGE + X_TILE;
                if constexpr (EPI == EPI_SILU) {
                    tma_load_2d_hint(dst, &tm_w, bars + slot * 8, kt * LK, blockIdx.x * BOUT, pol);
                    tma_load_2d_hint(dst + BOUT * 128, &tm_w, bars + slot * 8, kt * LK, p.up_row0 + blockIdx.x * BOUT, pol);
                } else {
                    tma_load_2d_hint(dst, &tm_w, bars + slot * 8, kt * LK, blockIdx.x * BN, pol);
                }
            };
            auto load_x = [&](int slot, int kt) {
                if constexpr (CL > 1)
                    tma_load_2d_mc(base + slot * C::STAGE + crank * (X_ROWS * 128), &tm_x, bars + slot * 8, kt * LK, m0 + (int)crank * X_ROWS, CL_MASK);
                else
                    tma_load_2d(base + slot * C::STAGE, &tm_x, bars + slot * 8, kt * LK, m0);
            };
            const int pre = nk < S ? nk : S;
            for (int i = 0; i < pre; ++i) {                      // weights first: they do not depend on the predecessor
                mbar_expect_tx(bars + i * 8, C::STAGE);
                load_w(i, kt0 + i);
            }
            asm volatile("griddepcontrol.wait;" ::: "memory");   // x is the previous kernel's output
            for (int i = 0; i < pre; ++i) load_x(i, kt0 + i);
            for (int i = pre; i < nk; ++i) {
                const int slot = i % S, round = i / S;
                mbar_wait(bars + (S + slot) * 8, (round - 1) & 1);            // the MMAs that read this slot have retired
                mbar_expect_tx(bars + slot * 8, C::STAGE);
                load_w(slot, kt0 + i);
                load_x(slot, kt0 + i);
            }
        }
    } else {
        // ---- MMA warpgroup: one k tile in flight while the previous one retires ------------------------------------
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int c = 0; c < BN / 2; ++c) acc[h][c] = 0.f;
        // the row-half decision is taken once, outside the MMA loop, so that every wgmma sequence is straight-line code
        auto consume = [&](auto two) {
            constexpr bool TWO = decltype(two)::value;
            for (int i = 0; i < nk; ++i) {
                const int slot = i % S, round = i / S;
                mbar_wait(bars + slot * 8, round & 1);
                const uint32_t xs = base + slot * C::STAGE, ws = xs + X_TILE;
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < LK / 16; ++ks) {
                    const uint64_t bdesc = make_desc(ws + ks * 32, 16, 1024);
                    wgmma_ss<BN>(acc[0], make_desc(xs + ks * 32, 16, 1024), bdesc, 1u);
                    if constexpr (TWO) wgmma_ss<BN>(acc[1], make_desc(xs + X_HALF + ks * 32, 16, 1024), bdesc, 1u);
                }
                wg_commit();
                wg_wait<1>();                                  // k tile i - 1 has been read: its slot is free
                if (i > 0) release_slot<CL>(bars + (S + (i - 1) % S) * 8, lane);
            }
            wg_wait<0>();
        };
        if (two_halves) consume(std::true_type{});
        else consume(std::false_type{});
        acc_fence(acc[0]);
        acc_fence(acc[1]);
        if (nk > 0) release_slot<CL>(bars + (S + (nk - 1) % S) * 8, lane);
    }

    // ---- epilogue (warpgroup 0): acc[h][4c + 2r + e] = D[64 h + 16 warp + g + 8 r][8 c + 2 qd + e] ---------------------
    if (warp < 4) {
        const int g = lane >> 2, qd = lane & 3;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int row = m0 + 64 * h + 16 * warp + g + 8 * r;
                if constexpr (EPI == EPI_SAMPLE) {
                    // LM head + Sampler.forward in one pass (layers/embed_head.py:56-66, layers/sampler.py:7-12): this thread
                    // holds BN/4 logits of its row; they are rounded to bf16 (the reference's logits are the bf16 output of
                    // F.linear), scored (greedy: the logit; otherwise the exponential race) and only the best (score, token)
                    // key of the quad's BN columns leaves the SM.
                    unsigned long long key = 0ull;
                    if (row < p.rows) {
                        const uint64_t step = p.step + (p.step_dev ? (uint64_t)*p.step_dev : 0ull);
                        const b200sample::RowSampler rs(p.temperatures ? p.temperatures[row] : 0.f, p.seed, step, row);
                        b200sample::Best best{-INFINITY, 0x7fffffff};
                        const int n0 = blockIdx.x * BN + 2 * qd;
#pragma unroll
                        for (int c = 0; c < BN / 8; ++c)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int col = n0 + 8 * c + e;
                                if (col < p.n_valid) b200sample::take(best, rs.score(round_bf16(acc[h][4 * c + 2 * r + e]), p.index_offset + col), col);
                            }
                        if (best.i != 0x7fffffff) key = b200sample::pack_key(best.v, (uint32_t)(p.index_offset + best.i));
                    }
                    key = max(key, __shfl_xor_sync(0xffffffffu, key, 1));
                    key = max(key, __shfl_xor_sync(0xffffffffu, key, 2));
                    if (qd == 0 && key != 0ull) atomicMax(p.keys + row, key);
                } else if (row < p.rows) {
                    if constexpr (EPI == EPI_PARTIAL) {
                        float* dst = static_cast<float*>(p.out) + ((int64_t)blockIdx.z * p.rows + row) * p.out_stride + blockIdx.x * BN + 2 * qd;
#pragma unroll
                        for (int c = 0; c < BN / 8; ++c) *reinterpret_cast<float2*>(dst + 8 * c) = make_float2(acc[h][4 * c + 2 * r], acc[h][4 * c + 2 * r + 1]);
                    } else {
                        __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(p.out) + (int64_t)row * p.out_stride + blockIdx.x * BOUT + 2 * qd;
#pragma unroll
                        for (int c = 0; c < BOUT / 8; ++c) {
                            float y[2];
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                if constexpr (EPI == EPI_SILU) {
                                    // the reference rounds the projection to bf16 before SiluAndMul sees it (F.linear output)
                                    const float gt = round_bf16(acc[h][4 * c + 2 * r + e]), up = round_bf16(acc[h][4 * (c + BOUT / 8) + 2 * r + e]);
                                    y[e] = __fmul_rn(gt / (1.0f + expf(-gt)), up);
                                } else {
                                    y[e] = acc[h][4 * c + 2 * r + e];
                                }
                            }
                            *reinterpret_cast<uint32_t*>(dst + 8 * c) = pack_bf16x2(y[0], y[1]);
                        }
                    }
                }
            }
        }
    }
    __syncwarp();                                  // the producer warp's lanes reconverge before the .aligned cluster barrier
    if constexpr (CL > 1) cluster_sync_all();      // nobody leaves while a peer may still signal its barriers
}

// RMSNorm.add_rms_forward (layers/layernorm.py:28-40) on a split-K projection: x = bf16(sum over splits, in order).
constexpr int PN_THREADS = 128;
constexpr int PN_MAXV = 8;
__global__ void __launch_bounds__(PN_THREADS) add_rmsnorm_partials_kernel(const float* __restrict__ parts, int splits, int64_t split_stride,
                                                                          __nv_bfloat16* residual, const __nv_bfloat16* __restrict__ w,
                                                                          __nv_bfloat16* out, int cols, float eps) {
    __shared__ float red[4];
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int row = blockIdx.x;
    const int nvec = cols >> 3;
    const float* prow = parts + (int64_t)row * cols;
    uint4* r4 = reinterpret_cast<uint4*>(residual + (int64_t)row * cols);
    const uint4* w4 = reinterpret_cast<const uint4*>(w);
    uint4* o4 = reinterpret_cast<uint4*>(out + (int64_t)row * cols);
    float v[PN_MAXV][8];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < PN_MAXV; ++k) {
        const int idx = threadIdx.x + k * PN_THREADS;
        if (idx < nvec) {
            float h[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            for (int s = 0; s < splits; ++s) {
                const float4* q = reinterpret_cast<const float4*>(prow + s * split_stride) + idx * 2;
                const float4 a = q[0], b = q[1];
                h[0] += a.x; h[1] += a.y; h[2] += a.z; h[3] += a.w;
                h[4] += b.x; h[5] += b.y; h[6] += b.z; h[7] += b.w;
            }
            float r[8];
            unpack8(r4[idx], r);
#pragma unroll
            for (int e = 0; e < 8; ++e) v[k][e] = round_bf16(h[e]) + r[e];
            r4[idx] = pack8(v[k]);
#pragma unroll
            for (int e = 0; e < 8; ++e) ss = fmaf(v[k][e], v[k][e], ss);
        }
    }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    const float rstd = 1.0f / sqrtf((red[0] + red[1] + red[2] + red[3]) / (float)cols + eps);
#pragma unroll
    for (int k = 0; k < PN_MAXV; ++k) {
        const int idx = threadIdx.x + k * PN_THREADS;
        if (idx < nvec) {
            float wf[8], y[8];
            unpack8(w4[idx], wf);
#pragma unroll
            for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(__fmul_rn(v[k][e], rstd), wf[e]);
            o4[idx] = pack8(y);
        }
    }
}

// keys -> token ids (and the signed keys of the vocab-parallel combine); leaves the key array empty for the next step
__global__ void sample_finalize_kernel(unsigned long long* keys, int64_t* out, int64_t* out_keys, int64_t index_offset, int rows) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= rows) return;
    const unsigned long long key = keys[row];
    keys[row] = 0ull;
    if (out) out[row] = key ? (int64_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull)) : index_offset;
    if (out_keys) out_keys[row] = (int64_t)(key ^ 0x8000000000000000ull);
}

// ---- host side ------------------------------------------------------------------------------------------------
// Tensor maps depend only on (base, shape, stride, box); weights never move and activations cycle through a few
// allocator blocks, so encoded maps are cached (cuTensorMapEncodeTiled costs ~1 us of host time).
struct MapKey {
    const void* base; uint64_t cols, rows, stride; uint32_t box_rows;
    bool operator==(const MapKey& o) const { return base == o.base && cols == o.cols && rows == o.rows && stride == o.stride && box_rows == o.box_rows; }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        uint64_t h = (uint64_t)(uintptr_t)k.base * 0x9E3779B97F4A7C15ull;
        h ^= (k.cols + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
        h ^= (k.rows + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
        h ^= (k.stride * 31 + k.box_rows + (h << 6) + (h >> 2));
        return (size_t)h;
    }
};
bool cached_map(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t stride, uint32_t box_rows) {
    static std::mutex mu;
    static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
    const MapKey key{base, cols, rows, stride, box_rows};
    std::lock_guard<std::mutex> lock(mu);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return true; }
    if (!make_map(out, base, cols, rows, stride, box_rows)) return false;
    if (cache.size() > 4096) cache.clear();
    cache.emplace(key, *out);
    return true;
}

}  // namespace

// shared with layer_tail.cu
bool b200_cached_tensor_map(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t stride, uint32_t box_rows) {
    return cached_map(out, base, cols, rows, stride, box_rows);
}

namespace {

template <int BN, int EPI, bool DEEP, int CL>
int launch_linear(const CUtensorMap& tx, const CUtensorMap& tw, LinParams prm, dim3 grid, bool pdl, cudaStream_t stream) {
    using C = Cfg<BN, DEEP>;
    if (prm.stages <= 0 || prm.stages > C::STAGES) prm.stages = C::STAGES;      // 0: this configuration's full ring
    if (prm.stages < 2) prm.stages = 2;
    static B200SmemOptIn optin;
    if (cudaError_t e = optin.ensure(linear_tc_kernel<BN, EPI, DEEP, CL>, C::SMEM); e != cudaSuccess) {
        b200_tls_cuda_error() = cudaGetErrorString(e);
        return B200_ECUDA;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(L_THREADS);
    cfg.dynamicSmemBytes = (size_t)prm.stages * C::STAGE + 256;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (pdl) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    if (CL > 1) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = CL;
        attr[na].val.clusterDim.y = 1;
        attr[na].val.clusterDim.z = 1;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    if (cudaLaunchKernelEx(&cfg, linear_tc_kernel<BN, EPI, DEEP, CL>, tx, tw, prm) != cudaSuccess) return B200_ECUDA;
    return B200_OK;
}

template <int EPI, bool DEEP, int CL>
int dispatch_bn(int bn, const CUtensorMap& tx, const CUtensorMap& tw, const LinParams& prm, dim3 grid, bool pdl, cudaStream_t stream) {
    switch (bn) {
        case 16: if constexpr (EPI == EPI_SILU) return B200_EUNSUPPORTED; else return launch_linear<16, EPI, DEEP, CL>(tx, tw, prm, grid, pdl, stream);
        case 32: return launch_linear<32, EPI, DEEP, CL>(tx, tw, prm, grid, pdl, stream);
        case 64: return launch_linear<64, EPI, DEEP, CL>(tx, tw, prm, grid, pdl, stream);
        case 128: return launch_linear<128, EPI, DEEP, CL>(tx, tw, prm, grid, pdl, stream);
        default: return B200_EUNSUPPORTED;
    }
}
template <int EPI>
int dispatch_depth(bool deep, int cluster, int bn, const CUtensorMap& tx, const CUtensorMap& tw, const LinParams& prm, dim3 grid, bool pdl, cudaStream_t stream) {
    if (cluster == 2) return dispatch_bn<EPI, true, 2>(bn, tx, tw, prm, grid, pdl, stream);       // multicast variants: deep ring only
    if (cluster == 4) return dispatch_bn<EPI, true, 4>(bn, tx, tw, prm, grid, pdl, stream);
    return deep ? dispatch_bn<EPI, true, 1>(bn, tx, tw, prm, grid, pdl, stream) : dispatch_bn<EPI, false, 1>(bn, tx, tw, prm, grid, pdl, stream);
}

}  // namespace

extern "C" int b200_linear(const void* x, int64_t x_stride0, const void* w, void* out, int64_t out_stride0, int rows, int n_out,
                           int k, int epilogue, int block_n, int k_splits, int flags, void* stream) {
    if (!x || !w || !out || rows < 0 || n_out <= 0 || k <= 0) return B200_EINVAL;
    if (((uintptr_t)x & 15) || ((uintptr_t)w & 15) || ((uintptr_t)out & 15) || (x_stride0 % 8) || (out_stride0 % 8)) return B200_EINVAL;
    if (epilogue < EPI_BF16 || epilogue > EPI_PARTIAL || k_splits < 1) return B200_EINVAL;
    if (k % LK) return B200_EUNSUPPORTED;
    const int k_tiles_total = k / LK;
    if (k_tiles_total % k_splits) return B200_EUNSUPPORTED;
    if (k_splits > 1 && epilogue != EPI_PARTIAL) return B200_EINVAL;
    const int bout = epilogue == EPI_SILU ? block_n / 2 : block_n;        // output columns per CTA
    if (bout <= 0 || n_out % bout) return B200_EUNSUPPORTED;
    if (rows == 0) return B200_OK;
    const int w_rows = epilogue == EPI_SILU ? 2 * n_out : n_out;
    const int cluster = 1 << ((flags >> 2) & 3);                         // flags bits 2-3: log2 of the cluster size
    if (cluster > 4 || (cluster > 1 && (flags & 2))) return B200_EUNSUPPORTED;
    if ((n_out / bout) % cluster) return B200_EUNSUPPORTED;
    CUtensorMap tx, tw;
    if (!cached_map(&tx, x, (uint64_t)k, (uint64_t)rows, (uint64_t)x_stride0, LM / cluster)) return B200_EUNSUPPORTED;
    if (!cached_map(&tw, w, (uint64_t)k, (uint64_t)w_rows, (uint64_t)k, (uint32_t)bout)) return B200_EUNSUPPORTED;
    LinParams prm = {};
    prm.out = out;
    prm.out_stride = out_stride0;
    prm.rows = rows;
    prm.up_row0 = n_out;
    prm.k_tiles = k_tiles_total / k_splits;
    prm.stages = (flags >> 4) & 15;                                      // 0: the configuration's own depth
    dim3 grid(n_out / bout, (rows + LM - 1) / LM, k_splits);
    if (grid.y > 65535 || grid.z > 65535) return B200_EUNSUPPORTED;
    const bool pdl = (flags & 1) != 0;
    const bool deep = (flags & 2) == 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc;
    if (epilogue == EPI_BF16) rc = dispatch_depth<EPI_BF16>(deep, cluster, block_n, tx, tw, prm, grid, pdl, st);
    else if (epilogue == EPI_SILU) rc = dispatch_depth<EPI_SILU>(deep, cluster, block_n, tx, tw, prm, grid, pdl, st);
    else rc = dispatch_depth<EPI_PARTIAL>(deep, cluster, block_n, tx, tw, prm, grid, pdl, st);
    if (rc != B200_OK) return rc;
    return b200_launch_status(nullptr);
}

extern "C" int b200_lm_head_sample(const void* hidden, int64_t hidden_stride0, const void* lm_head, int rows, int vocab, int k,
                                   const float* temperatures, int64_t index_offset, uint64_t seed, uint64_t step,
                                   const int64_t* step_dev, void* key_workspace, int64_t* out, int64_t* out_keys, int block_n,
                                   int flags, void* stream) {
    if (!hidden || !lm_head || !key_workspace || (!out && !out_keys) || rows < 0 || vocab <= 0 || k <= 0 || index_offset < 0) return B200_EINVAL;
    if (((uintptr_t)hidden & 15) || ((uintptr_t)lm_head & 15) || ((uintptr_t)key_workspace & 7) || (hidden_stride0 % 8)) return B200_EINVAL;
    if (index_offset + vocab > 0xffffffffll || (k % LK)) return B200_EUNSUPPORTED;
    if (rows == 0) return B200_OK;
    const int cluster = 1 << ((flags >> 2) & 3);
    if (cluster > 4 || (cluster > 1 && (flags & 2))) return B200_EUNSUPPORTED;
    if (block_n <= 0) return B200_EUNSUPPORTED;
    const int n_tiles = (vocab + block_n - 1) / block_n;
    if (n_tiles % cluster) return B200_EUNSUPPORTED;
    CUtensorMap tx, tw;
    if (!cached_map(&tx, hidden, (uint64_t)k, (uint64_t)rows, (uint64_t)hidden_stride0, LM / cluster)) return B200_EUNSUPPORTED;
    if (!cached_map(&tw, lm_head, (uint64_t)k, (uint64_t)vocab, (uint64_t)k, (uint32_t)block_n)) return B200_EUNSUPPORTED;
    LinParams prm = {};
    prm.rows = rows;
    prm.k_tiles = k / LK;
    prm.n_valid = vocab;
    prm.temperatures = temperatures;
    prm.index_offset = index_offset;
    prm.seed = seed;
    prm.step = step;
    prm.step_dev = step_dev;
    prm.keys = static_cast<unsigned long long*>(key_workspace);
    prm.stages = (flags >> 4) & 15;
    dim3 grid(n_tiles, (rows + LM - 1) / LM, 1);
    if (grid.y > 65535) return B200_EUNSUPPORTED;
    const bool pdl = (flags & 1) != 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = dispatch_depth<EPI_SAMPLE>((flags & 2) == 0, cluster, block_n, tx, tw, prm, grid, pdl, st);
    if (rc != B200_OK) return rc;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((rows + 127) / 128);
    cfg.blockDim = dim3(128);
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    if (cudaLaunchKernelEx(&cfg, sample_finalize_kernel, prm.keys, out, out_keys, index_offset, rows) != cudaSuccess) return B200_ECUDA;
    return b200_launch_status(nullptr);
}

extern "C" int b200_add_rmsnorm_partials(const float* partials, int splits, void* residual, const void* weight, void* out, int rows,
                                         int cols, float eps, int flags, void* stream) {
    if (!partials || !residual || !weight || !out || rows < 0 || splits < 1) return B200_EINVAL;
    if (cols <= 0 || cols % 8 || cols > PN_THREADS * PN_MAXV * 8) return B200_EUNSUPPORTED;
    if (((uintptr_t)partials & 15) || ((uintptr_t)residual & 15) || ((uintptr_t)weight & 15) || ((uintptr_t)out & 15)) return B200_EINVAL;
    if (rows == 0) return B200_OK;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(rows);
    cfg.blockDim = dim3(PN_THREADS);
    cfg.stream = static_cast<cudaStream_t>(stream);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (flags & 1) ? 1 : 0;
    if (cudaLaunchKernelEx(&cfg, add_rmsnorm_partials_kernel, partials, splits, (int64_t)rows * cols, static_cast<__nv_bfloat16*>(residual),
                           static_cast<const __nv_bfloat16*>(weight), static_cast<__nv_bfloat16*>(out), cols, eps) != cudaSuccess)
        return B200_ECUDA;
    return b200_launch_status(nullptr);
}
