// Helpers shared by the kernels that are fed by TMA (the Tensor Memory Accelerator: gemm_tc.cu, flash_attn.cu, refiner_fused.cu,
// dwconv_tma.cu); gp.cu, refiner.cu and local_corr_tile.cu use the named barriers, the shared-memory opt-in or the SM count.
//   device: mbarrier, cp.async.bulk.tensor and named-barrier PTX wrappers;
//   host:   the tensor-map encoder, the one-time-per-device dynamic shared-memory opt-in and the cached SM count.
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>

namespace rb {

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n" : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

__device__ __forceinline__ void bar_named(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int nthreads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// cuTensorMapEncodeTiled, resolved through the runtime once per process (nullptr when the driver does not provide it)
inline PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
    static const PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && ptr;
        return ok ? reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr) : nullptr;
    }();
    return fn;
}

// tensor-map element type of a dtype code (RB_F16S: each of its two planes is fp16)
inline CUtensorMapDataType tma_dtype(int code) {
    return code == RB_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : (code == RB_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
}

// Tiled tensor map of `rank` dimensions over `base`: dims[rank], byte strides[rank - 1] of dimensions 1.., box[rank]; dense
// element strides, 256-byte L2 promotion, zero fill out of bounds.  Errors are reported as "<what>: ...".
inline int encode_tiled(CUtensorMap* map, const char* what, CUtensorMapDataType dtype, int rank, const void* base, const cuuint64_t* dims,
                        const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle) {
    const PFN_cuTensorMapEncodeTiled_v12000 enc = tensor_map_encoder();
    RB_REQUIRE(enc, "%s: cuTensorMapEncodeTiled not available (driver too old?)", what);
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    const CUresult r = enc(map, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    RB_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled failed with %d (dims %llu x %llu x ..., pitch %llu bytes)", what, (int)r,
               (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)strides[0]);
    return 0;
}

// Opts Kernel in to `bytes` of dynamic shared memory, once per device (function attributes are per device, and several engines on
// different GPUs may share the process).  The flags belong to the kernel itself, so kernels of the same signature do not share them;
// a kernel is always given the same `bytes`.
template <auto Kernel>
inline int ensure_smem(int bytes, const char* what) {
    static bool configured[64] = {};
    const int dev = current_device() & 63;
    if (!configured[dev]) {
        const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
        RB_REQUIRE(e == cudaSuccess, "%s: cannot set %d bytes of dynamic shared memory: %s", what, bytes, cudaGetErrorString(e));
        configured[dev] = true;
    }
    return 0;
}

// multiprocessors of the current device, queried once per device
inline int sm_count() {
    static int n[64] = {};
    const int dev = current_device() & 63;
    if (!n[dev]) {
        cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
        if (n[dev] <= 0) n[dev] = 132;
    }
    return n[dev];
}

// L2 cache bytes of the current device, queried once per device
inline int64_t l2_bytes() {
    static int n[64] = {};
    const int dev = current_device() & 63;
    if (!n[dev]) {
        cudaDeviceGetAttribute(&n[dev], cudaDevAttrL2CacheSize, dev);
        if (n[dev] <= 0) n[dev] = 50 << 20;
    }
    return n[dev];
}

}  // namespace rb
