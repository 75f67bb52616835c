// Single-token paged decode attention for sm_90a.
//
// Replaces the decode branch of the reference's Attention.forward (nanovllm/layers/attention.py:71-74,
// flash_attn_with_kvcache over paged K/V).  HBM-bandwidth bound: every K/V byte of every live
// context token is read exactly once per layer per step.
//
// Design (DESIGN.md "decode kernel"):
//   * one persistent launch, one CTA per SM, NWARPS independent warps per CTA;
//   * the step's work is the list of 16-token chunks ordered by (sequence, kv head, chunk);
//     it is cut into equal contiguous ranges, one per warp ("stream-K" over KV pages), so the
//     load is balanced to one chunk whatever the mix of context lengths;
//   * each warp streams its chunks through a private NSTAGES-deep ring in shared memory with
//     1-D bulk async copies (TMA engine, cp.async.bulk -> SASS UBLKCP) completing on mbarriers;
//     a (page, kv head) tile is contiguous in HBM so every copy is one linear 4 KB burst;
//   * QK^T and PV run on the fp32 FMA pipe with all G q-heads of the kv head sharing each K/V
//     read; softmax statistics via warp shuffles;
//   * a kv-head's context that straddles several warps leaves (m, l, O) partials in a small
//     workspace; the last warp to arrive (per-pair counter) merges them in fixed order, so the
//     result is deterministic and no second launch is needed.
//
// This file holds the fp32-FMA formulation, used for head groups G <= 2 (Qwen3-0.6B), where it reads HBM at
// 6.1 TB/s (93 % of the measured copy peak).  decode_mma.cu is the warp-level tensor-core formulation of the same
// schedule for G >= 4.  The FUSED template flag (b200_paged_decode_fused) makes the kernel take the raw qkv
// projection and do q/k-norm, RoPE and the KV append itself.  K/V bulk copies carry an L2 evict_first policy.
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "decode_common.cuh"

using namespace b200dec;

namespace {

constexpr int CS_BYTES = B200_HEAD_DIM * 4;        // one cos|sin row of the rotary table

template <int G, int NWARPS, int NSTAGES, bool FUSED = false>
struct DecodeSmem {
    static constexpr int kQBytes = G * ROW_BYTES;                        // the G query heads of one kv head
    static constexpr int kStageBytes = 2 * CHUNK_BYTES + kQBytes + (FUSED ? CS_BYTES : 0);   // [K][V][q][cos|sin]
    static constexpr int kWarpBytes = NSTAGES * kStageBytes;
    static constexpr int kOffStages = 0;
    static constexpr int kOffCum = NWARPS * kWarpBytes;                 // int[MAX_BATCH + 1]
    static constexpr int kOffCtx = kOffCum + (MAX_BATCH + 4) * 4;       // int[MAX_BATCH]
    static constexpr int kOffBars = kOffCtx + MAX_BATCH * 4;            // u64[NWARPS][NSTAGES]
    static constexpr int kOffP = kOffBars + NWARPS * NSTAGES * 8;       // float[NWARPS][G][16]
    static constexpr int kOffWarpTot = kOffP + NWARPS * G * 16 * 4;     // int[NWARPS]
    static constexpr int kTotal = kOffWarpTot + 32 * 4;
};

template <int G, int NWARPS, int NSTAGES, bool FUSED>
__global__ void __launch_bounds__(NWARPS * 32, 1) paged_decode_kernel(const DecodeParams p) {
    B200_PDL_TRIGGER();
    using L = DecodeSmem<G, NWARPS, NSTAGES, FUSED>;
    extern __shared__ __align__(128) uint8_t smem[];
    int* cum = reinterpret_cast<int*>(smem + L::kOffCum);
    int* ctxs = reinterpret_cast<int*>(smem + L::kOffCtx);
    int* warp_tot = reinterpret_cast<int*>(smem + L::kOffWarpTot);

    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int batch = p.batch;
    const int hkv = p.hkv;

    uint8_t* my_stages = smem + L::kOffStages + warp * L::kWarpBytes;
    const uint32_t my_stages_u32 = smem_u32(my_stages);
    const uint32_t my_bars_u32 = smem_u32(smem + L::kOffBars) + warp * NSTAGES * 8;
    float* pbuf = reinterpret_cast<float*>(smem + L::kOffP) + warp * G * 16;

    // ---- per-warp ring setup -----------------------------------------------------------------------
    if (lane == 0) {
        for (int s = 0; s < NSTAGES; ++s) mbar_init(my_bars_u32 + s * 8, 1);
        mbar_fence_init();
    }

    // ---- exclusive prefix of per-sequence chunk counts ------------------------------------------
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
    // ---- rows without context (CUDA-graph padding) produce zeros --------------------------------
    for (int b = blockIdx.x; b < batch; b += gridDim.x) {
        if (ctxs[b] == 0) {
            const int n16 = hkv * G * (B200_HEAD_DIM / 8);
            uint4* o4 = reinterpret_cast<uint4*>(p.out + (int64_t)b * p.out_stride);
            for (int i = tid; i < n16; i += NT) o4[i] = make_uint4(0, 0, 0, 0);
        }
    }

    // ---- this warp's contiguous chunk range -----------------------------------------------------
    const long long C = (long long)hkv * cum[batch];
    const int TW = gridDim.x * NWARPS;
    // logical worker id: consecutive workers sit on different SMs, so a small step still spreads over the chip
    const int gw = warp * gridDim.x + blockIdx.x;
    if (C == 0) return;
    // workers that get work: each at least MIN_CHUNKS chunks (a sequence cut into too many segments pays
    // for it in the merge), never more than there are warps
    long long TWe = (C + MIN_CHUNKS - 1) / MIN_CHUNKS;
    TWe = TWe < TW ? TWe : (long long)TW;
    if (gw >= TWe) return;
    const long long c_begin = (long long)gw * C / TWe;
    const long long c_end = (long long)(gw + 1) * C / TWe;
    const int n_local = (int)(c_end - c_begin);

    ChunkCursor pi, ci;                                   // producer (issue) / consumer cursors
    pi.seek(cum, ctxs, batch, hkv, c_begin);
    ci = pi;

    const int hw = lane >> 4;                             // which token of a pair this half-warp owns
    const int j = lane & 15;                              // which 8-wide slice of head_dim
    const int bs_mask = (1 << p.block_shift) - 1;

    // lane 0 keeps the page id of the next chunk to issue one step ahead, so the dependent
    // block-table load never sits on the issue path
    int pg_next = 0;
    if (lane == 0) pg_next = p.block_tables[(int64_t)pi.b * p.bt_stride + ((pi.ck * CHUNK) >> p.block_shift)];
    const uint64_t l2pol = l2_policy_evict_first();

    auto issue = [&](int i) {                             // chunk i of this warp's range
        if (lane == 0) {
            const int slot = i % NSTAGES;
            const int tok0 = pi.ck * CHUNK;
            const int page = pg_next;
            int valid = pi.ctx - tok0;
            valid = valid > CHUNK ? CHUNK : valid;
            if (FUSED && pi.ck == pi.n - 1) --valid;              // the newest token is not in the cache yet
            const uint32_t bytes = (uint32_t)valid * ROW_BYTES;
            const int64_t row = (((int64_t)page * hkv + pi.h) << p.block_shift) + (tok0 & bs_mask);
            const uint32_t bar = my_bars_u32 + slot * 8;
            const uint32_t dst = my_stages_u32 + slot * L::kStageBytes;
            const bool seg_first = (pi.ck == 0) || (i == 0);      // the consumer starts a segment on this chunk
            mbar_expect_tx(bar, 2 * bytes + (seg_first ? (uint32_t)(L::kQBytes + (FUSED ? CS_BYTES : 0)) : 0u));
            if (bytes) {
                if (p.l2_hint) {
                    bulk_g2s_hint(dst, p.k_layer + row * B200_HEAD_DIM, bytes, bar, l2pol);
                    bulk_g2s_hint(dst + CHUNK_BYTES, p.v_layer + row * B200_HEAD_DIM, bytes, bar, l2pol);
                } else {
                    bulk_g2s(dst, p.k_layer + row * B200_HEAD_DIM, bytes, bar);
                    bulk_g2s(dst + CHUNK_BYTES, p.v_layer + row * B200_HEAD_DIM, bytes, bar);
                }
            }
            if (seg_first) {
                bulk_g2s(dst + 2 * CHUNK_BYTES, p.q + (int64_t)pi.b * p.q_stride + pi.h * G * B200_HEAD_DIM, L::kQBytes, bar);
                if (FUSED)
                    bulk_g2s(dst + 2 * CHUNK_BYTES + L::kQBytes, p.cos_sin + (int64_t)(pi.ctx - 1) * B200_HEAD_DIM, CS_BYTES, bar);
            }
        }
        pi.advance(cum, ctxs, batch, hkv);
        if (lane == 0 && i + 1 < n_local)
            pg_next = p.block_tables[(int64_t)pi.b * p.bt_stride + ((pi.ck * CHUNK) >> p.block_shift)];
    };

    __syncwarp();
#pragma unroll 1
    for (int i = 0; i < NSTAGES - 1 && i < n_local; ++i) issue(i);

    float qf[G][8];
    float o[G][8];
    float m[G], l[G];
    bool seg_start = true;
    // fused mode: this lane's slice of the q/k norm weights (whole kernel) and of the cos|sin row (per segment)
    float qw[8], kw[8], cosr[8], sinr[8];
    if (FUSED) {
        unpack8(*reinterpret_cast<const uint4*>(p.q_norm_w + j * 8), qw);
        unpack8(*reinterpret_cast<const uint4*>(p.k_norm_w + j * 8), kw);
    }
    // RMSNorm over head_dim (the 16 lanes of a half-warp hold one head) -> bf16 -> NeoX rotation -> bf16, the
    // arithmetic of qknorm_rope_store_kernel (models/qwen3.py:82-85)
    auto norm_rope = [&](float (&x)[8], const float (&w)[8]) {
        float ss = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) ss = fmaf(x[e], x[e], ss);
#pragma unroll
        for (int o2 = 8; o2 > 0; o2 >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o2);
        const float rstd = 1.0f / sqrtf(ss / (float)B200_HEAD_DIM + p.eps);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float y = round_bf16(__fmul_rn(__fmul_rn(x[e], rstd), w[e]));
            const float other = __shfl_xor_sync(0xffffffffu, y, 8);          // element d +- 64
            const float r = (j < 8) ? __fsub_rn(__fmul_rn(y, cosr[e]), __fmul_rn(other, sinr[e]))
                                    : __fadd_rn(__fmul_rn(y, cosr[e]), __fmul_rn(other, sinr[e]));
            x[e] = round_bf16(r);
        }
    };

#pragma unroll 1
    for (int i = 0; i < n_local; ++i) {
        if (i + NSTAGES - 1 < n_local) issue(i + NSTAGES - 1);

        const int slot = i % NSTAGES;
        mbar_wait(my_bars_u32 + slot * 8, (i / NSTAGES) & 1);
        const uint8_t* ks = my_stages + slot * L::kStageBytes;
        const uint8_t* vs = ks + CHUNK_BYTES;

        // fused mode: the raw K / V row of the newest token is needed after the last chunk of the kv head;
        // start its loads now so they fly under the chunk's math
        const bool last_chunk = FUSED && (ci.ck == ci.n - 1);
        uint4 k_raw = make_uint4(0, 0, 0, 0), v_raw = make_uint4(0, 0, 0, 0);
        if (last_chunk) {
            const __nv_bfloat16* rowp = p.q + (int64_t)ci.b * p.q_stride + j * 8;
            k_raw = *reinterpret_cast<const uint4*>(rowp + (hkv * G + ci.h) * B200_HEAD_DIM);
            v_raw = *reinterpret_cast<const uint4*>(rowp + (hkv * G + hkv + ci.h) * B200_HEAD_DIM);
        }

        if (seg_start) {                                  // q arrived with this chunk
            seg_start = false;
            if (FUSED) {
                const float* cs = reinterpret_cast<const float*>(ks + 2 * CHUNK_BYTES + L::kQBytes) + (j & 7) * 8;
                const float4 c0 = *reinterpret_cast<const float4*>(cs), c1 = *reinterpret_cast<const float4*>(cs + 4);
                const float4 s0 = *reinterpret_cast<const float4*>(cs + 64), s1 = *reinterpret_cast<const float4*>(cs + 68);
                cosr[0] = c0.x; cosr[1] = c0.y; cosr[2] = c0.z; cosr[3] = c0.w; cosr[4] = c1.x; cosr[5] = c1.y; cosr[6] = c1.z; cosr[7] = c1.w;
                sinr[0] = s0.x; sinr[1] = s0.y; sinr[2] = s0.z; sinr[3] = s0.w; sinr[4] = s1.x; sinr[5] = s1.y; sinr[6] = s1.z; sinr[7] = s1.w;
            }
#pragma unroll
            for (int g = 0; g < G; ++g) {
                const uint4 w = *reinterpret_cast<const uint4*>(ks + 2 * CHUNK_BYTES + g * ROW_BYTES + j * 16);
                unpack8(w, qf[g]);
                if (FUSED) norm_rope(qf[g], qw);
#pragma unroll
                for (int e = 0; e < 8; ++e) { qf[g][e] *= p.scale_log2; o[g][e] = 0.f; }
                m[g] = -INFINITY;
                l[g] = 0.f;
            }
        }

        int nvalid = ci.ctx - ci.ck * CHUNK;
        nvalid = nvalid > CHUNK ? CHUNK : nvalid;
        if (last_chunk) --nvalid;                         // the newest token is handled from registers below
        if (nvalid > 0) {

        // ---- S = q K^T : half-warp per token, 16 lanes x 8 dims ---------------------------------
        float acc[G][8];
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            const uint4 w = *reinterpret_cast<const uint4*>(ks + (2 * it + hw) * ROW_BYTES + j * 16);
            float kf[8];
            unpack8(w, kf);
#pragma unroll
            for (int g = 0; g < G; ++g) {
                float a = qf[g][0] * kf[0];
#pragma unroll
                for (int e = 1; e < 8; ++e) a = fmaf(qf[g][e], kf[e], a);
                acc[g][it] = a;
            }
        }
        // reduce over the 16 dim-slices, scattering tokens over lanes: 8 -> 4 -> 2 -> 1 values
#pragma unroll
        for (int g = 0; g < G; ++g) {
#pragma unroll
            for (int x = 0; x < 4; ++x) {
                const float send = (j & 8) ? acc[g][x] : acc[g][x + 4];
                const float keep = (j & 8) ? acc[g][x + 4] : acc[g][x];
                acc[g][x] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
            }
#pragma unroll
            for (int x = 0; x < 2; ++x) {
                const float send = (j & 4) ? acc[g][x] : acc[g][x + 2];
                const float keep = (j & 4) ? acc[g][x + 2] : acc[g][x];
                acc[g][x] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
            {
                const float send = (j & 2) ? acc[g][0] : acc[g][1];
                const float keep = (j & 2) ? acc[g][1] : acc[g][0];
                acc[g][0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
            }
            acc[g][0] += __shfl_xor_sync(0xffffffffu, acc[g][0], 1);
        }
        // this lane now holds the score of token  t = 2*it + hw,  it = bits (3,2,1) of j
        const int my_it = ((j >> 3) & 1) * 4 + ((j >> 2) & 1) * 2 + ((j >> 1) & 1);
        const int my_t = 2 * my_it + hw;
        const bool tok_ok = my_t < nvalid;

        // ---- online softmax ---------------------------------------------------------------------
#pragma unroll
        for (int g = 0; g < G; ++g) {
            const float s = tok_ok ? acc[g][0] : -INFINITY;
            const float m_new = fmaxf(m[g], warp_max(s));
            const float alpha = fast_exp2(m[g] - m_new);
            const float pv = fast_exp2(s - m_new);
            m[g] = m_new;
            l[g] = l[g] * alpha + ((j & 1) ? 0.f : pv);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[g][e] *= alpha;
            if (!(j & 1)) pbuf[g * 16 + hw * 8 + my_it] = pv;
        }
        __syncwarp();

        // ---- O += P V ---------------------------------------------------------------------------
        float pr[G][8];
#pragma unroll
        for (int g = 0; g < G; ++g) {
            const float4 a = *reinterpret_cast<const float4*>(pbuf + g * 16 + hw * 8);
            const float4 c4 = *reinterpret_cast<const float4*>(pbuf + g * 16 + hw * 8 + 4);
            pr[g][0] = a.x; pr[g][1] = a.y; pr[g][2] = a.z; pr[g][3] = a.w;
            pr[g][4] = c4.x; pr[g][5] = c4.y; pr[g][6] = c4.z; pr[g][7] = c4.w;
        }
        // Rows beyond the context in the last chunk of a sequence were not copied: the stage still holds
        // whatever an earlier chunk left there (or uninitialised shared memory); their p is 0 but 0 * NaN
        // is NaN, so that chunk takes a path that zeroes them.
        auto pv = [&](auto partial) {
#pragma unroll
            for (int it = 0; it < 8; ++it) {
                uint4 w = *reinterpret_cast<const uint4*>(vs + (2 * it + hw) * ROW_BYTES + j * 16);
                if constexpr (decltype(partial)::value) {
                    if (2 * it + hw >= nvalid) w = make_uint4(0, 0, 0, 0);
                }
                float vf[8];
                unpack8(w, vf);
#pragma unroll
                for (int g = 0; g < G; ++g) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) o[g][e] = fmaf(pr[g][it], vf[e], o[g][e]);
                }
            }
        };
        if (nvalid == CHUNK) pv(std::false_type{}); else pv(std::true_type{});
        }   // nvalid > 0

        if (last_chunk) {
            // ---- the step's own token: k = rope(norm(k_raw)), v = v_raw, appended to the cache and attended ----
            float kn[8], vn[8];
            unpack8(k_raw, kn);
            unpack8(v_raw, vn);
            norm_rope(kn, kw);
            const int tok = ci.ctx - 1;
            const int page = p.block_tables[(int64_t)ci.b * p.bt_stride + (tok >> p.block_shift)];
            const int64_t crow = (((int64_t)page * hkv + ci.h) << p.block_shift) + (tok & bs_mask);
            if (hw == 0) {
                *reinterpret_cast<uint4*>(p.k_layer_w + crow * B200_HEAD_DIM + j * 8) = pack8(kn);
                *reinterpret_cast<uint4*>(p.v_layer_w + crow * B200_HEAD_DIM + j * 8) = v_raw;
            }
#pragma unroll
            for (int g = 0; g < G; ++g) {
                float sc = qf[g][0] * kn[0];
#pragma unroll
                for (int e = 1; e < 8; ++e) sc = fmaf(qf[g][e], kn[e], sc);
#pragma unroll
                for (int o2 = 8; o2 > 0; o2 >>= 1) sc += __shfl_xor_sync(0xffffffffu, sc, o2);
                const float m_new = fmaxf(m[g], sc);
                const float alpha = fast_exp2(m[g] - m_new);
                const float pn = fast_exp2(sc - m_new);
                m[g] = m_new;
                l[g] = l[g] * alpha + (lane == 0 ? pn : 0.f);
                const float pv0 = hw == 0 ? pn : 0.f;        // the two half-warps' partial O are summed at the end
#pragma unroll
                for (int e = 0; e < 8; ++e) o[g][e] = fmaf(pv0, vn[e], o[g][e] * alpha);
            }
        }
        __syncwarp();   // every lane is done with this stage and with pbuf

        // ---- end of a segment (kv head exhausted, or this warp's range ends) ---------------------
        const bool pair_done = (ci.ck == ci.n - 1);
        if (pair_done || i == n_local - 1) {
#pragma unroll
            for (int g = 0; g < G; ++g) {
                l[g] = warp_sum(l[g]);
#pragma unroll
                for (int e = 0; e < 8; ++e) o[g][e] += __shfl_xor_sync(0xffffffffu, o[g][e], 16);
            }
            const int pair = ci.b * hkv + ci.h;
            const long long c0 = (long long)hkv * cum[ci.b] + (long long)ci.h * ci.n;
            const long long c1 = c0 + ci.n;
            const int w_first = (int)(((c0 + 1) * TWe - 1) / C);
            const int w_last = (int)((c1 * TWe - 1) / C);
            const int nseg = w_last - w_first + 1;
            __nv_bfloat16* orow = p.out + (int64_t)ci.b * p.out_stride + (ci.h * G) * B200_HEAD_DIM + j * 8;
            if (nseg == 1) {
                if (hw == 0) {
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        const float inv = 1.f / l[g];
                        float r[8];
#pragma unroll
                        for (int e = 0; e < 8; ++e) r[e] = o[g][e] * inv;
                        *reinterpret_cast<uint4*>(orow + g * B200_HEAD_DIM) = pack8(r);
                    }
                }
            } else {
                const int myslot = (gw == w_first) ? TW + pair : gw;
                float* po = p.part_o + (int64_t)myslot * (G * B200_HEAD_DIM) + j * 8;
                if (hw == 0) {
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        float4* d4 = reinterpret_cast<float4*>(po + g * B200_HEAD_DIM);
                        d4[0] = make_float4(o[g][0], o[g][1], o[g][2], o[g][3]);
                        d4[1] = make_float4(o[g][4], o[g][5], o[g][6], o[g][7]);
                    }
                }
                if (lane == 0) {
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        p.part_ml[((int64_t)myslot * G + g) * 2 + 0] = m[g];
                        p.part_ml[((int64_t)myslot * G + g) * 2 + 1] = l[g];
                    }
                }
                __threadfence();
                __syncwarp();
                int old = 0;
                if (lane == 0) old = atomicAdd(p.counters + pair, 1);
                old = __shfl_sync(0xffffffffu, old, 0);
                if (old == nseg - 1) {               // last segment in: merge, in an order fixed by the data
                    __threadfence();
                    // half-warp hw folds segments k = hw, hw+2, ... with a running maximum, then the halves meet
                    float M[G], Ls[G], r[G][8];
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        M[g] = -INFINITY; Ls[g] = 0.f;
#pragma unroll
                        for (int e = 0; e < 8; ++e) r[g][e] = 0.f;
                    }
#pragma unroll 2
                    for (int k = hw; k < nseg; k += 2) {
                        const int sl = k == 0 ? TW + pair : w_first + k;
#pragma unroll
                        for (int g = 0; g < G; ++g) {
                            const float2 ml = __ldcg(reinterpret_cast<const float2*>(p.part_ml + ((int64_t)sl * G + g) * 2));
                            const float4* s4 = reinterpret_cast<const float4*>(
                                p.part_o + ((int64_t)sl * G + g) * B200_HEAD_DIM + j * 8);
                            const float4 a = __ldcg(s4), c4 = __ldcg(s4 + 1);
                            const float Mn = fmaxf(M[g], ml.x);
                            const float so = fast_exp2(M[g] - Mn), sn = fast_exp2(ml.x - Mn);
                            M[g] = Mn;
                            Ls[g] = Ls[g] * so + ml.y * sn;
                            r[g][0] = r[g][0] * so + a.x * sn; r[g][1] = r[g][1] * so + a.y * sn;
                            r[g][2] = r[g][2] * so + a.z * sn; r[g][3] = r[g][3] * so + a.w * sn;
                            r[g][4] = r[g][4] * so + c4.x * sn; r[g][5] = r[g][5] * so + c4.y * sn;
                            r[g][6] = r[g][6] * so + c4.z * sn; r[g][7] = r[g][7] * so + c4.w * sn;
                        }
                    }
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        const float Mo = __shfl_xor_sync(0xffffffffu, M[g], 16);
                        const float Lo = __shfl_xor_sync(0xffffffffu, Ls[g], 16);
                        const float Mn = fmaxf(M[g], Mo);                       // nseg >= 2: both halves saw a segment
                        const float sa = fast_exp2(M[g] - Mn), sb = fast_exp2(Mo - Mn);
                        const float inv = 1.f / (Ls[g] * sa + Lo * sb);
                        float res[8];
#pragma unroll
                        for (int e = 0; e < 8; ++e) {
                            const float ro = __shfl_xor_sync(0xffffffffu, r[g][e], 16);
                            res[e] = (r[g][e] * sa + ro * sb) * inv;
                        }
                        if (hw == 0) *reinterpret_cast<uint4*>(orow + g * B200_HEAD_DIM) = pack8(res);
                    }
                    if (lane == 0) p.counters[pair] = 0;   // leave the workspace clean for the next launch
                }
            }
            seg_start = true;
        }
        ci.advance(cum, ctxs, batch, hkv);
    }
}

constexpr int kMaxWarps = 16;   // workspace is sized for the widest variant

// (warps per CTA, ring depth) variants; B200_DECODE_CFG=<warps>x<stages> picks one at first use (tuning knob).
template <int G, int NW, int NS, bool FUSED>
int launch_variant(b200_ctx* ctx, const DecodeParams& prm, cudaStream_t stream) {
    using L = DecodeSmem<G, NW, NS, FUSED>;
    if constexpr (L::kTotal > 227 * 1024) {
        return B200_EUNSUPPORTED;
    } else {
        auto kern = paged_decode_kernel<G, NW, NS, FUSED>;
        static B200SmemOptIn optin;
        B200_CUDA_CHECK(ctx, optin.ensure(kern, L::kTotal));
        B200_LAUNCH((kern), ctx->sm_count, NW * 32, L::kTotal, stream, prm);
        return b200_launch_status(ctx);
    }
}

int decode_variant() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("B200_DECODE_CFG");
        v = 0;
        if (e && !strcmp(e, "12x2")) v = 1;
        if (e && !strcmp(e, "10x2")) v = 2;
        if (e && !strcmp(e, "8x3")) v = 3;
        if (e && !strcmp(e, "6x2")) v = 4;
    }
    return v;
}

template <int G, bool FUSED>
int launch_decode(b200_ctx* ctx, const DecodeParams& prm, cudaStream_t stream) {
    static_assert(G <= 2, "the fp32-FMA formulation is issue-bound beyond 2 query heads per kv head: use decode_mma.cu");
    if constexpr (FUSED) {
        return launch_variant<G, 8, 2, true>(ctx, prm, stream);
    } else {
        switch (decode_variant()) {
            case 1: return launch_variant<G, 12, 2, false>(ctx, prm, stream);
            case 2: return launch_variant<G, 10, 2, false>(ctx, prm, stream);
            case 3: return launch_variant<G, 8, 3, false>(ctx, prm, stream);
            case 4: return launch_variant<G, 6, 2, false>(ctx, prm, stream);
            default: return launch_variant<G, 8, 2, false>(ctx, prm, stream);
        }
    }
}

}  // namespace

struct WsLayout {
    size_t off_ml, off_o, total;
};
// [counters: MAX_BATCH*hkv ints -- fixed place whatever the batch, they persist (as zeros) between
//  launches][part_ml][part_o]; the two scratch regions may move with the batch size.
static WsLayout ws_layout(int sm_count, int batch, int hkv, int G) {
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    const size_t slots = (size_t)sm_count * kMaxWarps + (size_t)batch * hkv;
    WsLayout w;
    size_t off = al((size_t)MAX_BATCH * hkv * sizeof(int));
    w.off_ml = off;
    off += al(slots * G * 2 * sizeof(float));
    w.off_o = off;
    off += al(slots * G * B200_HEAD_DIM * sizeof(float));
    w.total = off;
    return w;
}

extern "C" size_t b200_decode_workspace_bytes(const b200_ctx* ctx, int max_batch, int num_q_heads) {
    if (!ctx || ctx->num_kv_heads <= 0 || max_batch <= 0 || num_q_heads % ctx->num_kv_heads) return 0;
    return ws_layout(ctx->sm_count, max_batch, ctx->num_kv_heads, num_q_heads / ctx->num_kv_heads).total;
}

int b200_decode_mma_launch(b200_ctx* ctx, int layer, const DecodeParams& prm, int G, cudaStream_t stream);

static bool use_mma_decode() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("B200_DECODE");
        v = (e && !strcmp(e, "mma")) ? 1 : 0;
    }
    return v == 1;
}

static int decode_common(b200_ctx* ctx, int layer, const void* q, int64_t q_stride0, const int32_t* block_tables,
                         int bt_stride, const int32_t* context_lens, void* out, int64_t out_stride0, int batch,
                         int num_q_heads, float scale, void* workspace, size_t workspace_bytes, void* stream,
                         const void* q_norm_w, const void* k_norm_w, const float* cos_sin, float eps, bool fused) {
    if (!ctx || !q || !out || !block_tables || !context_lens || !workspace) return B200_EINVAL;
    if (!ctx->k_base) return B200_ENOTBOUND;
    if (layer < 0 || layer >= ctx->layers || batch < 0) return B200_EINVAL;
    if (batch == 0) return B200_OK;
    if (batch > MAX_BATCH) return B200_EUNSUPPORTED;
    const int hkv = ctx->num_kv_heads;
    if (num_q_heads % hkv) return B200_EINVAL;
    const int G = num_q_heads / hkv;
    if (G != 1 && G != 2 && G != 4 && G != 8) return B200_EUNSUPPORTED;
    if ((q_stride0 % 8) || (out_stride0 % 8) || ((uintptr_t)q % 16) || ((uintptr_t)out % 16)) return B200_EINVAL;
    if (fused && (!q_norm_w || !k_norm_w || !cos_sin || ((uintptr_t)q_norm_w % 16) || ((uintptr_t)k_norm_w % 16) ||
                  ((uintptr_t)cos_sin % 16)))
        return B200_EINVAL;
    const WsLayout w = ws_layout(ctx->sm_count, batch, hkv, G);
    if (workspace_bytes < w.total) return B200_EWORKSPACE;

    DecodeParams prm;
    prm.q = static_cast<const __nv_bfloat16*>(q);
    prm.q_stride = q_stride0;
    prm.out = static_cast<__nv_bfloat16*>(out);
    prm.out_stride = out_stride0;
    prm.k_layer = ctx->k_layer(layer);
    prm.v_layer = ctx->v_layer(layer);
    prm.k_layer_w = ctx->k_layer(layer);
    prm.v_layer_w = ctx->v_layer(layer);
    prm.block_tables = block_tables;
    prm.bt_stride = bt_stride;
    prm.context_lens = context_lens;
    prm.batch = batch;
    prm.hkv = hkv;
    prm.block_shift = ctx->block_shift;
    prm.scale_log2 = scale * 1.4426950408889634f;
    prm.q_norm_w = static_cast<const __nv_bfloat16*>(q_norm_w);
    prm.k_norm_w = static_cast<const __nv_bfloat16*>(k_norm_w);
    prm.cos_sin = cos_sin;
    prm.eps = eps;
    {
        static int hint = -1;
        // measured on the benchmark's decode steps: 97.8 -> 96.1 us at batch 256, 91.2 -> 90.0 at 126, 46.0 -> 45.0 at 37
        if (hint < 0) { const char* e = getenv("B200_DECODE_L2HINT"); hint = (e && e[0] == '0') ? 0 : 1; }
        prm.l2_hint = hint;
    }
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    prm.counters = reinterpret_cast<int*>(ws);
    prm.part_ml = reinterpret_cast<float*>(ws + w.off_ml);
    prm.part_o = reinterpret_cast<float*>(ws + w.off_o);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // Kernel choice by head-group size (measured on the benchmark's batch-256 step, same KV bytes):
    //   G = 2: FMA 97.6 us, MMA 99.4 us      G = 4: FMA 121.6, MMA 101.9      G = 8: FMA 215.7, MMA 104.2
    if (fused) {
        if (G > 2) return B200_EUNSUPPORTED;
        return G == 1 ? launch_decode<1, true>(ctx, prm, st) : launch_decode<2, true>(ctx, prm, st);
    }
    if (G > 2 || use_mma_decode()) return b200_decode_mma_launch(ctx, layer, prm, G, st);
    return G == 1 ? launch_decode<1, false>(ctx, prm, st) : launch_decode<2, false>(ctx, prm, st);
}

extern "C" int b200_paged_decode(b200_ctx* ctx, int layer, const void* q, int64_t q_stride0,
                                 const int32_t* block_tables, int bt_stride,
                                 const int32_t* context_lens, void* out, int64_t out_stride0,
                                 int batch, int num_q_heads, float scale, void* workspace,
                                 size_t workspace_bytes, void* stream) {
    return decode_common(ctx, layer, q, q_stride0, block_tables, bt_stride, context_lens, out, out_stride0, batch,
                         num_q_heads, scale, workspace, workspace_bytes, stream, nullptr, nullptr, nullptr, 0.f, false);
}

extern "C" int b200_paged_decode_fused(b200_ctx* ctx, int layer, const void* qkv, int64_t qkv_stride0,
                                       const void* q_norm_weight, const void* k_norm_weight,
                                       const float* cos_sin, float eps, const int32_t* block_tables,
                                       int bt_stride, const int32_t* context_lens, void* out,
                                       int64_t out_stride0, int batch, int num_q_heads, float scale,
                                       void* workspace, size_t workspace_bytes, void* stream) {
    return decode_common(ctx, layer, qkv, qkv_stride0, block_tables, bt_stride, context_lens, out, out_stride0, batch,
                         num_q_heads, scale, workspace, workspace_bytes, stream, q_norm_weight, k_norm_weight, cos_sin,
                         eps, true);
}
