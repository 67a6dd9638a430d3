// racinglmpc_b200/csrc/ftocp_sets.cu — the QP kernel for handles with per-controller parameters (lmpc_set_param_sets):
// ftocp_kernel<..., true>.  A separate translation unit from lmpc_b200.cu, so that each unit instantiates only its own variant
// (see ftocp_launch.cuh).
#include "ftocp_launch.cuh"

template <int N, int M>
static cudaError_t sets_configure_t() {
    return cudaFuncSetAttribute(ftocp_kernel<N, M, 2, 4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)sizeof(KernelSmem<N, M, 2, 4, true>));
}

cudaError_t ftocp_sets_configure(int N, int M) {
    cudaError_t e = cudaErrorInvalidValue;
#define SCASE(n, m) if (N == n && (m == 0 || m == M)) { e = sets_configure_t<n, m>(); if (e != cudaSuccess) return e; }
    LMPC_FOR_EACH_CASE(SCASE)
#undef SCASE
    return e;
}

cudaError_t ftocp_sets_launch(int N, int M, const FtocpConstRec* table, FtocpArgs a, cudaStream_t st) {
    a.sets = table;
#define LCASE(n, m)                                                                                               \
    if (N == n && M == m) {                                                                                       \
        ftocp_kernel<n, m, 2, 4, true><<<a.batch, 32, sizeof(KernelSmem<n, m, 2, 4, true>), st>>>({}, a);        \
        return cudaGetLastError();                                                                                \
    }
    LMPC_FOR_EACH_CASE(LCASE)
#undef LCASE
    return cudaErrorInvalidValue;
}
