// racinglmpc_b200/csrc/ftocp_launch.cuh — what the two translation units of the QP kernels share: the bulk-copy helpers, the
// launch arguments, the resident-warp bounds and the instantiated (horizon, safe-set size) grid.
//   lmpc_b200.cu  : ftocp_kernel, parameters of the whole launch in the constant bank (handles without parameter sets)
//   ftocp_sets.cu : ftocp_sets_kernel, each instance's parameters from a table (lmpc_set_param_sets)
// The variant lives in its own translation unit so that the compiler treats the uniform kernels exactly as before: with both
// kernels calling the same inlined solver in one unit, the uniform instantiations were scheduled differently.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "ftocp_pdip.cuh"

using namespace lmpc;

// ------------------------------------------------------------------------------------------------
// device helpers: mbarrier + bulk async copy (PTX ISA: cp.async.bulk, sm_90+)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}

struct FtocpArgs {
    int batch;
    const double* x0;     // [B,6]
    const double* uOld;   // [B,2]
    const double* abc;    // stage model
    long long abc_inst_stride, abc_stage_stride;   // doubles
    const double* SS;     // [B,6,M]
    const double* Qfun;   // [B,M]
    const double* SuccSS; // [B,6,M] or null
    const double* SuccU;  // [B,2,M] or null
    double* xPred;        // [B,N+1,6]
    double* uPred;        // [B,N,2]
    double* slack;        // [B,N*NCX] or null
    double* lambd;        // [B,M] or null
    double* slackT;       // [B,6] or null
    double* zt;           // [B,6] or null
    double* ztu;          // [B,2] or null
    int* status;
    int* iters;
    double* resid;        // [B,3]
    unsigned long long* late;   // counter of instances accepted by the late-acceptance rule (ftocp_pdip.cuh), or null
    double* warm;         // [B][warm_stride] warm-start records (ftocp_pdip.cuh), or null = cold start
    int* warm_valid;      // [B]
    long long warm_stride;
    const int* set_idx;   // [B] parameter set of each instance (lmpc_set_param_sets), or null = the handle's own parameters
};

// One row of the per-controller parameter table: cp.async.bulk moves whole 16 B units, so the rows are padded to a multiple of 16 B
struct alignas(16) FtocpConstRec {
    FtocpConst c;
};
static_assert(sizeof(FtocpConstRec) % 16 == 0, "bulk copies need 16 B multiples");

// resident CTAs (= warps) per SM the register allocation is held to: horizons up to 14 are bounded by registers and shared
// memory alike; longer horizons by shared memory only
#ifndef LMPC_LB_MPC
#define LMPC_LB_MPC 16
#endif
#ifndef LMPC_LB_LMPC
#define LMPC_LB_LMPC 12
#endif
// what shared memory allows (about 992 B per stage + 3.5 KB for a safe set + 1 KB reserved per CTA + `extra`), capped by the
// register target
constexpr int ftocp_min_blocks(int N, int M, int extra = 0) {
    const int by_smem = 227 * 1024 / ((lmpc::stream_model(N) ? 560 : 992) * N + (M > 0 ? 74 * M : 0) + 448 + 1024 + extra);
    const int by_regs = M > 0 ? LMPC_LB_LMPC : LMPC_LB_MPC;
    return by_smem < 1 ? 1 : (by_smem < by_regs ? by_smem : by_regs);
}

// The supported (horizon, safe-set size) grid: one instantiation of the solver per pair.
// Horizons 4..48 with and without the reference's 48-point safe set (initControllerParameters.py:43-44), and other safe-set
// sizes (numSS_it x even points per lap) at the reference's and BASELINE's horizons.
#define LMPC_FOR_EACH_CASE(X) \
    X(4, 0) X(6, 0) X(8, 0) X(10, 0) X(12, 0) X(14, 0) X(16, 0) X(20, 0) X(24, 0) X(32, 0) X(48, 0) \
    X(4, 48) X(6, 48) X(8, 48) X(10, 48) X(12, 48) X(14, 48) X(16, 48) X(20, 48) X(24, 48) X(32, 48) X(48, 48) \
    X(12, 24) X(12, 32) X(12, 64) X(12, 96) X(14, 24) X(14, 32) X(14, 64) X(14, 96)
#define LMPC_GRID_TEXT "N in {4,6,8,10,12,14,16,20,24,32,48} with numSS_Points in {0,48}; N in {12,14} also with numSS_Points in {24,32,64,96}"

// ftocp_sets.cu: opt the variant's (N, M) and (N, 0) instantiations into their shared-memory size on the current device, and launch
// one; both return a CUDA error code (cudaErrorInvalidValue for a pair outside the grid)
cudaError_t ftocp_sets_configure(int N, int M);
cudaError_t ftocp_sets_launch(int N, int M, const FtocpConstRec* table, const FtocpArgs& a, cudaStream_t st);
