// C-ABI glue: error reporting, device check, GEMM back-end dispatch.
#include "common.cuh"
#include <string.h>

namespace rb {

static thread_local char g_error[512] = "";
static unsigned long long g_launches = 0;     // kernels launched by this library (every launch goes through check_launch)

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

int check_launch(const char* what) {
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
        return 1;
    }
    return 0;
}

}  // namespace rb

extern "C" int romab200_abi_version(void) { return ROMAB200_ABI_VERSION; }
extern "C" const char* romab200_last_error(void) { return rb::g_error; }
extern "C" unsigned long long romab200_launch_count(void) { return rb::g_launches; }

extern "C" int romab200_device_ok(void) {
    int dev = 0;
    cudaDeviceProp prop;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
        rb::set_error("no CUDA device");
        cudaGetLastError();
        return 0;
    }
    return prop.major == 9 && prop.minor == 0 ? 1 : 0;
}

extern "C" int romab200_gemm(const rb_gemm_args* a, void* stream) {
    using namespace rb;
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a && a->A && a->B && a->C, "gemm: null operand");
    // the epilogues of both back-ends convert the output and the residual at run time
    if (a->dtype_c != RB_F16S && check_dtype<float, __half, __nv_bfloat16>(a->dtype_c, "gemm")) return 1;
    if (a->R && check_dtype<float, __half, __nv_bfloat16>(a->dtype_r, "gemm")) return 1;
    int backend = a->backend;
    if (backend == RB_BACKEND_AUTO) backend = a->dtype_ab == RB_F32 ? RB_BACKEND_SIMT : RB_BACKEND_TCGEN05;
    if (backend == RB_BACKEND_SIMT) return gemm_simt(a, st);
    return gemm_tc(a, st);
}
