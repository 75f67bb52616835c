// Shared device helpers and the context struct behind include/b200_paged_attn.h.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>
#include <string>

#include "b200_paged_attn.h"

#define B200_HEAD_DIM 128

struct b200_ctx {
    int device = 0;
    int sm_count = 0;
    size_t smem_optin = 0;
    // bound KV cache (layout [layers][num_blocks][num_kv_heads][block_size][head_dim])
    __nv_bfloat16* k_base = nullptr;
    __nv_bfloat16* v_base = nullptr;
    int layers = 0;
    int64_t num_blocks = 0;
    int block_size = 0;
    int block_shift = 0;
    int num_kv_heads = 0;
    int head_dim = 0;
    std::string last_cuda_error;
    uint64_t bind_gen = 0;          // set by every b200_kv_bind, unique within the process (cached TMA descriptors key on it)
    // b200_kv_bind_fp8: the cache holds e4m3 bytes, element = e4m3_satfinite_rn(x / scale), read back as float(e) * scale.
    // k_base / v_base then point at bytes: use the *_layer8 accessors, never k_layer / v_layer.
    bool kv_fp8 = false;
    float k_scale = 1.f, v_scale = 1.f;

    size_t layer_elems() const {
        return (size_t)num_blocks * num_kv_heads * block_size * head_dim;
    }
    __nv_bfloat16* k_layer(int l) const { return k_base + (size_t)l * layer_elems(); }
    __nv_bfloat16* v_layer(int l) const { return v_base + (size_t)l * layer_elems(); }
    uint8_t* k_layer8(int l) const { return reinterpret_cast<uint8_t*>(k_base) + (size_t)l * layer_elems(); }
    uint8_t* v_layer8(int l) const { return reinterpret_cast<uint8_t*>(v_base) + (size_t)l * layer_elems(); }
};

#define B200_CUDA_CHECK(ctx, expr)                                   \
    do {                                                              \
        cudaError_t _e = (expr);                                      \
        if (_e != cudaSuccess) {                                      \
            if (ctx) (ctx)->last_cuda_error = cudaGetErrorString(_e); \
            return B200_ECUDA;                                        \
        }                                                             \
    } while (0)

// Text of the last CUDA error seen by an entry point that has no b200_ctx (b200_rmsnorm, b200_linear, ...): kept per
// host thread and returned by b200_last_cuda_error(NULL).
inline std::string& b200_tls_cuda_error() {
    static thread_local std::string text;
    return text;
}

static inline int b200_launch_status(b200_ctx* ctx) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        if (ctx) ctx->last_cuda_error = cudaGetErrorString(e);
        else b200_tls_cuda_error() = cudaGetErrorString(e);
        return B200_ECUDA;
    }
    return B200_OK;
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-DEVICE property of a kernel: remember the opt-in per device
// ordinal, so that a process that drives several GPUs configures each of them (a process-wide flag would leave the second
// device without the opt-in and its launches would fail).
constexpr int B200_MAX_DEVICES = 64;
struct B200SmemOptIn {
    bool done[B200_MAX_DEVICES] = {};
    template <typename K>
    cudaError_t ensure(K kernel, size_t bytes) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        if (dev < 0 || dev >= B200_MAX_DEVICES) return cudaErrorInvalidDevice;
        if (done[dev]) return cudaSuccess;
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        // Ask for the largest shared-memory carve-out: a kernel of ANOTHER stream can only join this one on an SM if the
        // SM's current L1/shared split already has room for both (the split is not changed under a running CTA).  The
        // two-stream decode step (models/qwen3.py::_forward_dual) relies on it: wgmma projections of one half batch
        // run in the shared memory that the attention kernel of the other half leaves free.  A hint; none of these
        // kernels leans on L1.
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e == cudaSuccess) done[dev] = true;
        return e;
    }
};

// ------------------------------------------------------------------------------------------
// bf16 <-> fp32 on packed words.  A bf16 is the high half of an fp32, so unpacking is one
// shift / one mask (ALU pipe), leaving the FMA pipe to the dot products.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float bf16lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);  // .x = lo (low 16 bits)
    return *reinterpret_cast<uint32_t*>(&p);
}

__device__ __forceinline__ float round_bf16(float x) {
    return __bfloat162float(__float2bfloat16_rn(x));
}

__device__ __forceinline__ void unpack8(const uint4& w, float (&f)[8]) {
    f[0] = bf16lo(w.x); f[1] = bf16hi(w.x);
    f[2] = bf16lo(w.y); f[3] = bf16hi(w.y);
    f[4] = bf16lo(w.z); f[5] = bf16hi(w.z);
    f[6] = bf16lo(w.w); f[7] = bf16hi(w.w);
}

__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    uint4 w;
    w.x = pack_bf16x2(f[0], f[1]);
    w.y = pack_bf16x2(f[2], f[3]);
    w.z = pack_bf16x2(f[4], f[5]);
    w.w = pack_bf16x2(f[6], f[7]);
    return w;
}

// ------------------------------------------------------------------------------------------
// e4m3 cache elements (b200_kv_bind_fp8).  Quantize: e4m3_satfinite_rn(x / scale), one F2FP per pair (low byte = first
// element).  Dequantize: every e4m3 value is exact in fp16, so one F2FP per pair gives the exact value.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t quant4_e4m3(float a, float b, float c, float d, float scale) {
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(a, scale), __fdiv_rn(b, scale)), __NV_SATFINITE, __NV_E4M3);
    const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(c, scale), __fdiv_rn(d, scale)), __NV_SATFINITE, __NV_E4M3);
    return lo | (hi << 16);
}
// 8 bf16 (one 16-byte word) -> 8 e4m3 (one 8-byte word)
__device__ __forceinline__ uint2 quant8_e4m3(const uint4& w, float scale) {
    float f[8];
    unpack8(w, f);
    return make_uint2(quant4_e4m3(f[0], f[1], f[2], f[3], scale), quant4_e4m3(f[4], f[5], f[6], f[7], scale));
}
// two e4m3 (low byte first) -> f16x2 (low half first)
__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint32_t two) {
    const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(two & 0xffffu), __NV_E4M3);
    return (uint32_t)h.x | ((uint32_t)h.y << 16);
}

// ------------------------------------------------------------------------------------------
// warp reductions
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ------------------------------------------------------------------------------------------
// mbarrier + bulk async copy (TMA engine, SASS: UBLKCP / SYNCS)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    // make the inits visible to the async proxy before any bulk copy signals them
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(bar), "r"(parity)
        : "memory");
}
// 1-D bulk copy global -> shared, completion counted in bytes on `bar`.
// size must be a multiple of 16, both addresses 16-byte aligned.
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes,
                                         uint32_t bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
            "r"(dst_smem), "l"(src), "r"(bytes), "r"(bar)
        : "memory");
}

// Same copy with an L2 eviction-priority hint (streamed-once data: evict_first keeps it from displacing the rest).
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
            "r"(dst_smem), "l"(src), "r"(bytes), "r"(bar), "l"(policy)
        : "memory");
}

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// ------------------------------------------------------------------------------------------
// Programmatic dependent launch, compiled in with -DB200_PDL (the Makefile's default; `make NOPDL=1` builds the plain
// flavour as libb200attn_nopdl.so).  With it every kernel starts with launch_dependents + wait (a no-op for a launch
// without the attribute) and every launch carries cudaLaunchAttributeProgrammaticStreamSerialization, so inside a
// captured step the next kernel's blocks are scheduled while the previous kernel drains; kernels with a host-metadata
// prologue (the decode attention kernels) wait only after it.  Without the define both macros expand to nothing / a
// plain <<<>>> launch.
// ------------------------------------------------------------------------------------------
#define B200_UNPAREN(...) __VA_ARGS__
// Per host thread: launches made while this is set carry NO programmatic-serialization attribute (b200_set_pdl).  Used for
// the first kernel after a cross-stream event wait and for the kernel that follows an attention launch in the two-stream
// decode step, where an early-launched dependent would sit on the shared memory the other stream's kernels need.
inline bool& b200_tls_pdl_off() {
    static thread_local bool off = false;
    return off;
}
#ifdef B200_PDL
#define B200_PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")
#define B200_PDL_WAIT() asm volatile("griddepcontrol.wait;" ::: "memory")
#define B200_PDL_SYNC()     \
    do {                    \
        B200_PDL_TRIGGER(); \
        B200_PDL_WAIT();    \
    } while (0)
template <typename... KArgs, typename... Args>
static inline void b200_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = b200_tls_pdl_off() ? 0 : 1;
    cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);      // errors surface through cudaGetLastError()
}
#define B200_LAUNCH(kernel_in_parens, grid, block, smem, stream, ...) \
    b200_launch_pdl(B200_UNPAREN kernel_in_parens, dim3(grid), dim3(block), smem, stream, __VA_ARGS__)
#else
#define B200_PDL_TRIGGER() \
    do {                   \
    } while (0)
#define B200_PDL_WAIT() \
    do {                \
    } while (0)
#define B200_PDL_SYNC() \
    do {                \
    } while (0)
#define B200_LAUNCH(kernel_in_parens, grid, block, smem, stream, ...) \
    B200_UNPAREN kernel_in_parens<<<grid, block, smem, stream>>>(__VA_ARGS__)
#endif

// SM count of the current device, for the grid heuristics of the context-less entry points (cached per device ordinal;
// an attribute query, so it is legal while a stream is being captured)
static inline int b200_current_sm_count() {
    static int cached[B200_MAX_DEVICES] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= B200_MAX_DEVICES) return 132;
    if (!cached[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
        cached[dev] = n;
    }
    return cached[dev];
}

static inline int ilog2_exact(int v) {
    int s = 0;
    while ((1 << s) < v) ++s;
    return ((1 << s) == v) ? s : -1;
}
