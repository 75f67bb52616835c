// Tensor-parallel exchange fused with the op that always follows it, over NVLink peer memory (sm_90a).
//
// Replaces, for a decode step, the pair
//     dist.all_reduce(y)                          RowParallelLinear.forward, reference layers/linear.py:152-156
//     x, residual = add_rms_forward(y, residual)  RMSNorm, reference layers/layernorm.py:28-40
// by ONE kernel: every rank's partial GEMM output sits in its own slice of a symmetric (peer-mapped) allocation;
// after a flag handshake through peer memory each rank reads all partials directly over NVLink (ld.global on
// mapped peer pointers), sums them in fp32 in rank order (so all ranks produce identical bits), adds the
// residual, writes bf16(residual') and the normalised row.  One-shot all-reduce: the messages are <= 512 KB, so
// the exchange is latency bound and redundant reads (world x rows x cols) cost less than a second pass.
//
// Synchronisation: epoch counters.  flags_of(p)[r] holds the last epoch rank r has announced to rank p (written
// by r with st.release.sys); a launch at epoch e announces e+1 and waits until every peer has announced e+1,
// which also proves the peers have finished READING this rank's other data buffer (two buffers alternate), so the
// next GEMM may overwrite it.  The last CTA of a launch advances the local epoch (device memory, so a captured
// CUDA graph keeps counting across replays).
#include "common.cuh"

namespace {

constexpr int AR_THREADS = 128;
constexpr int AR_MAXV = 8;          // uint4 per thread -> cols <= 8192
constexpr int AR_MAX_WORLD = 8;

__device__ __forceinline__ void st_release_sys(int* p, int v) {
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// In-switch reduction (NVLS): one multimem load returns the sum over all ranks of the 8 bf16 at a multicast address,
// accumulated in fp32 inside the NVSwitch and rounded to bf16 once -- the rounding point of the reference's
// dist.all_reduce on bf16 tensors.  Every rank then moves `data` bytes over its links instead of world x data.
__device__ __forceinline__ uint4 multimem_sum_bf16x8(const void* mc_addr) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc_addr) : "memory");
    return v;
}

template <bool NVLS>
__global__ void __launch_bounds__(AR_THREADS) allreduce_add_rmsnorm_kernel(
    void* const* __restrict__ bases, const uint8_t* mc_base, uint64_t data_off, uint64_t flag_off, int* epoch, unsigned int* done, int* err, int rank,
    int world, __nv_bfloat16* residual, const __nv_bfloat16* __restrict__ w, __nv_bfloat16* out, int cols, float eps) {
    B200_PDL_SYNC();
    __shared__ float red[4];
    __shared__ int s_epoch;
    const int row = blockIdx.x;
    // epoch only advances when the LAST CTA of a launch has passed its wait, so every thread of every CTA reads the same value
    const int e = *reinterpret_cast<volatile int*>(epoch);
    if (threadIdx.x == 0) s_epoch = e;
    if (blockIdx.x == 0 && threadIdx.x < world && threadIdx.x != rank) {
        // Announce to every peer AT ONCE, one thread per peer: a release store at system scope cannot complete before the
        // writes ahead of it are performed, so a loop of world-1 of them in one thread is a chain of world-1 NVLink round
        // trips in front of every exchange (the reason 8 ranks were slower than 4).  Each thread orders this rank's
        // partials (previous kernel) before its own flag store.
        __threadfence_system();
        st_release_sys(reinterpret_cast<int*>(static_cast<uint8_t*>(bases[threadIdx.x]) + flag_off) + rank, e + 1);
    }
    if (threadIdx.x < world && threadIdx.x != rank) {
        // One thread per peer polls that peer's flag, so the system-scope acquire loads overlap instead of forming a chain of
        // world-1 round trips in front of every exchange (56 exchanges per decode step).
        // A peer that never shows up (a rank died, a mis-wired handle) must not wedge the GPU: after 2^35 cycles
        // (~18 s, far beyond any skew between lock-stepped ranks) the launch gives up and raises *err; the
        // start-up self-test (engine/peer_reduce.py) then switches every rank to NCCL.
        const int* mine = reinterpret_cast<const int*>(static_cast<const uint8_t*>(bases[rank]) + flag_off) + threadIdx.x;
        const long long t0 = clock64();
        while (ld_acquire_sys(mine) - (e + 1) < 0) {
            if (clock64() - t0 > (1ll << 35)) {
                if (err) atomicExch(err, 1);
                break;
            }
        }
    }
    __syncthreads();

    const int nvec = cols >> 3;
    const uint4* src[AR_MAX_WORLD];
#pragma unroll
    for (int p = 0; p < AR_MAX_WORLD; ++p)
        src[p] = p < world ? reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(bases[p]) + data_off) + (int64_t)row * nvec : nullptr;
    uint4* r4 = reinterpret_cast<uint4*>(residual + (int64_t)row * cols);
    const uint4* w4 = reinterpret_cast<const uint4*>(w);
    uint4* o4 = reinterpret_cast<uint4*>(out + (int64_t)row * cols);

    float v[AR_MAXV][8];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < AR_MAXV; ++k) {
        const int idx = threadIdx.x + k * AR_THREADS;
        if (idx < nvec) {
            unpack8(r4[idx], v[k]);                   // residual, then the partials in rank order
            if constexpr (NVLS) {
                float t[8];
                unpack8(multimem_sum_bf16x8(mc_base + data_off + ((int64_t)row * nvec + idx) * 16), t);
#pragma unroll
                for (int e = 0; e < 8; ++e) v[k][e] += t[e];
            } else {
#pragma unroll
                for (int p = 0; p < AR_MAX_WORLD; ++p) {
                    if (p < world) {
                        float t[8];
                        unpack8(__ldcv(src[p] + idx), t);
#pragma unroll
                        for (int e = 0; e < 8; ++e) v[k][e] += t[e];
                    }
                }
            }
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
    for (int k = 0; k < AR_MAXV; ++k) {
        const int idx = threadIdx.x + k * AR_THREADS;
        if (idx < nvec) {
            float wf[8], y[8];
            unpack8(w4[idx], wf);
#pragma unroll
            for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(__fmul_rn(v[k][e], rstd), wf[e]);
            o4[idx] = pack8(y);
        }
    }
    // the last CTA to get here advances the epoch for the next launch
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(done, 1u) == gridDim.x - 1) {
            *done = 0;
            *reinterpret_cast<volatile int*>(epoch) = s_epoch + 1;
        }
    }
}

}  // namespace

extern "C" int b200_allreduce_add_rmsnorm(const void* peer_bases_dev, uint64_t data_offset, uint64_t flag_offset,
                                          int* epoch, unsigned int* done, int* err_flag, int rank, int world,
                                          void* residual, const void* weight, void* out, int rows, int cols, float eps,
                                          void* stream) {
    if (!peer_bases_dev || !epoch || !done || !residual || !weight || !out || rows < 0) return B200_EINVAL;
    if (world < 2 || world > AR_MAX_WORLD || rank < 0 || rank >= world) return B200_EINVAL;
    if (cols <= 0 || cols % 8 || cols > AR_THREADS * AR_MAXV * 8 || (data_offset & 15) || (flag_offset & 3)) return B200_EUNSUPPORTED;
    if (rows == 0) return B200_OK;
    B200_LAUNCH((allreduce_add_rmsnorm_kernel<false>), rows, AR_THREADS, 0, static_cast<cudaStream_t>(stream), 
        static_cast<void* const*>(peer_bases_dev), nullptr, data_offset, flag_offset, epoch, done, err_flag, rank, world,
        static_cast<__nv_bfloat16*>(residual), static_cast<const __nv_bfloat16*>(weight), static_cast<__nv_bfloat16*>(out), cols, eps);
    return b200_launch_status(nullptr);
}

// Same exchange with the reduction done inside the NVSwitch (default from 4 ranks; validated at 2, 4 and 8 ranks in round 2).  `multicast_base` is the
// multicast mapping of the same symmetric allocation (torch symmetric memory: handle.multicast_ptr).
extern "C" int b200_allreduce_add_rmsnorm_nvls(const void* peer_bases_dev, const void* multicast_base, uint64_t data_offset,
                                               uint64_t flag_offset, int* epoch, unsigned int* done, int* err_flag, int rank,
                                               int world, void* residual, const void* weight, void* out, int rows, int cols,
                                               float eps, void* stream) {
    if (!peer_bases_dev || !multicast_base || !epoch || !done || !residual || !weight || !out || rows < 0) return B200_EINVAL;
    if (world < 2 || world > AR_MAX_WORLD || rank < 0 || rank >= world) return B200_EINVAL;
    if (cols <= 0 || cols % 8 || cols > AR_THREADS * AR_MAXV * 8 || (data_offset & 15) || (flag_offset & 3) || ((uintptr_t)multicast_base & 15))
        return B200_EUNSUPPORTED;
    if (rows == 0) return B200_OK;
    B200_LAUNCH((allreduce_add_rmsnorm_kernel<true>), rows, AR_THREADS, 0, static_cast<cudaStream_t>(stream), 
        static_cast<void* const*>(peer_bases_dev), static_cast<const uint8_t*>(multicast_base), data_offset, flag_offset, epoch, done, err_flag,
        rank, world, static_cast<__nv_bfloat16*>(residual), static_cast<const __nv_bfloat16*>(weight), static_cast<__nv_bfloat16*>(out), cols, eps);
    return b200_launch_status(nullptr);
}
