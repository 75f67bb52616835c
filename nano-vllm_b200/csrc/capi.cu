// Context lifetime and KV binding behind include/b200_paged_attn.h.
#include <atomic>
#include <cmath>

#include "common.cuh"

// Source of b200_ctx::bind_gen.  Process-wide, so that a binding of a new context (or of a context created after
// b200_destroy) never reuses the generation of an earlier binding: the tensor maps the tensor-core decode caches per
// generation (decode_mma.cu) would otherwise describe the earlier cache.
static std::atomic<uint64_t> g_bind_generation{0};

extern "C" int b200_abi_version(void) { return 2; }

extern "C" const char* b200_strerror(int code) {
    switch (code) {
        case B200_OK: return "ok";
        case B200_EINVAL: return "invalid argument";
        case B200_EUNSUPPORTED: return "unsupported shape (head_dim must be 128, q/kv head ratio in {1,2,4,8}, block_size a power of two in [16,256])";
        case B200_ECUDA: return "CUDA runtime error (see b200_last_cuda_error)";
        case B200_ENOTBOUND: return "KV cache not bound (call b200_kv_bind)";
        case B200_EWORKSPACE: return "workspace too small (see b200_decode_workspace_bytes)";
        case B200_EARCH: return "device is not compute capability 9.0 (this library is sm_90a only)";
        default: return "unknown error";
    }
}

extern "C" int b200_init(int device, b200_ctx** out) {
    if (!out) return B200_EINVAL;
    *out = nullptr;
    cudaDeviceProp prop;
    cudaError_t e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) return B200_ECUDA;
    if (prop.major != 9 || prop.minor != 0) return B200_EARCH;
    e = cudaSetDevice(device);
    if (e != cudaSuccess) return B200_ECUDA;
    b200_ctx* ctx = new b200_ctx();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    *out = ctx;
    return B200_OK;
}

extern "C" void b200_destroy(b200_ctx* ctx) { delete ctx; }

extern "C" const char* b200_last_cuda_error(b200_ctx* ctx) {
    return ctx ? ctx->last_cuda_error.c_str() : b200_tls_cuda_error().c_str();   // NULL: this thread's context-less calls
}

extern "C" int b200_sm_count(const b200_ctx* ctx) { return ctx ? ctx->sm_count : 0; }

extern "C" int b200_set_pdl(int enabled) {
    const int was = b200_tls_pdl_off() ? 0 : 1;
    b200_tls_pdl_off() = (enabled == 0);
    return was;
}

static int kv_bind(b200_ctx* ctx, void* k_base, void* v_base, int layers, int64_t num_blocks, int block_size,
                   int num_kv_heads, int head_dim, bool fp8, float k_scale, float v_scale) {
    if (!ctx || !k_base || !v_base || layers <= 0 || num_blocks <= 0 || num_kv_heads <= 0) return B200_EINVAL;
    if (head_dim != B200_HEAD_DIM) return B200_EUNSUPPORTED;
    const int shift = ilog2_exact(block_size);
    if (shift < 4 || shift > 8) return B200_EUNSUPPORTED;
    if (((uintptr_t)k_base & 127) || ((uintptr_t)v_base & 127)) return B200_EINVAL;
    ctx->k_base = static_cast<__nv_bfloat16*>(k_base);
    ctx->v_base = static_cast<__nv_bfloat16*>(v_base);
    ctx->layers = layers;
    ctx->num_blocks = num_blocks;
    ctx->block_size = block_size;
    ctx->block_shift = shift;
    ctx->num_kv_heads = num_kv_heads;
    ctx->head_dim = head_dim;
    ctx->kv_fp8 = fp8;
    ctx->k_scale = k_scale;
    ctx->v_scale = v_scale;
    ctx->bind_gen = ++g_bind_generation;
    return B200_OK;
}

extern "C" int b200_kv_bind(b200_ctx* ctx, void* k_base, void* v_base, int layers,
                            int64_t num_blocks, int block_size, int num_kv_heads, int head_dim) {
    return kv_bind(ctx, k_base, v_base, layers, num_blocks, block_size, num_kv_heads, head_dim, false, 1.f, 1.f);
}

extern "C" int b200_kv_bind_fp8(b200_ctx* ctx, void* k_base, void* v_base, int layers, int64_t num_blocks,
                                int block_size, int num_kv_heads, int head_dim, float k_scale, float v_scale) {
    if (!(std::isfinite(k_scale) && k_scale > 0.f) || !(std::isfinite(v_scale) && v_scale > 0.f)) return B200_EINVAL;
    return kv_bind(ctx, k_base, v_base, layers, num_blocks, block_size, num_kv_heads, head_dim, true, k_scale, v_scale);
}
