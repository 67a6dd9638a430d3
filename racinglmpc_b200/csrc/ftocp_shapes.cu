// racinglmpc_b200/csrc/ftocp_shapes.cu — the QP kernel for handles with per-controller horizons and safe-set sizes
// (lmpc_set_shapes).  A kernel and a translation unit of its own, so that the uniform and parameter-set kernels keep their code
// (see ftocp_launch.cuh).
#include "ftocp_launch.cuh"

// ftocp_kernel<N, M, NCX, NCU, true> for the controllers s.inst[0 .. gridDim.x) of shape (N, M): the same staging, solve and
// unpack, with the instance taken from the launch's list and every per-controller buffer addressed with the handle's strides
// (s.N, s.M).  A controller of shape (N, M) reads and writes the leading part of its regions: N stages of abc, N + 1 rows of xPred,
// N rows of uPred and the lane slacks, the row-major [6, M] / [2, M] blocks and M entries of Qfun and lambd (include/lmpc_b200.h,
// lmpc_set_shapes).  Shapes are refused on warm-start handles, so every solve starts cold.
template <int N, int M, int NCX, int NCU>
__global__ void __launch_bounds__(32, ftocp_min_blocks(N, M, (int)sizeof(FtocpConstRec)))
    ftocp_shaped_kernel(const __grid_constant__ ShapedLaunch s, const FtocpArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using KS = KernelSmem<N, M, NCX, NCU, true>;
    KS& ks = *reinterpret_cast<KS*>(smem_raw);
    auto& w = ks.w;
    const int b = s.inst[blockIdx.x];
    if (a.retire.retired(b)) return;       // before the mbarrier exists and before any bulk copy is in flight
    const int lane = threadIdx.x;
    const long long SN = s.N, SM = s.M;

    // ---- stage the instance's parameters, model and safe set into shared memory (TMA 1-D bulk copies) ----
    if (lane == 0) {
        mbar_init(&ks.bar, 1);
        constexpr bool STREAM = Work<N, M, NCX, NCU>::STREAM;
        uint32_t bytes = (STREAM ? 0 : N * 54 * 8) + (M > 0 ? (6 * M + M) * 8 : 0) + (uint32_t)sizeof(FtocpConstRec);
        mbar_expect_tx(&ks.bar, bytes);
        bulk_g2s(&ks.c, a.sets + (a.set_idx ? a.set_idx[b] : 0), sizeof(FtocpConstRec), &ks.bar);
        const double* src = a.abc + (long long)b * a.abc_inst_stride;
        w.gabc = src;
        w.gstage = (int)a.abc_stage_stride;
        if (STREAM) {
        } else if (a.abc_stage_stride == 54) {
            bulk_g2s(&w.ABC[0][0], src, N * 54 * 8, &ks.bar);
        } else {
            for (int k = 0; k < N; ++k) bulk_g2s(&w.ABC[k][0], src + (long long)k * a.abc_stage_stride, 54 * 8, &ks.bar);
        }
        if (M > 0) {
            bulk_g2s(&w.SS[0], a.SS + (long long)b * 6 * SM, 6 * M * 8, &ks.bar);
            bulk_g2s(&w.Qfun[0], a.Qfun + (long long)b * SM, M * 8, &ks.bar);
        }
    }
    double x0[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) x0[i] = a.x0[(long long)b * 6 + i];
    if (lane < 2) w.uOld[lane] = a.uOld[(long long)b * 2 + lane];
    __syncwarp();
    mbar_wait(&ks.bar, 0);

    // ---- solve ----
    SolveInfo info;
    Pdip<N, M, NCX, NCU>::solve(w, ks.c.c, x0, info, (M > 0) ? w.d4i : nullptr, a.slack ? a.slack + (long long)b * SN * NCX : nullptr,
                                nullptr, nullptr);

    // ---- unpack (PC.py:364-384) ----
    for (int e = lane; e < (N + 1) * 6; e += 32) a.xPred[(long long)b * (SN + 1) * 6 + e] = w.x[e];
    for (int e = lane; e < N * 2; e += 32) a.uPred[(long long)b * SN * 2 + e] = w.u[e];
    if (M > 0) {
        const double* lam = w.d4i;   // solve() left lambda here
        if (a.lambd)
            for (int e = lane; e < M; e += 32) a.lambd[(long long)b * SM + e] = lam[e];
        for (int e = lane; e < 14; e += 32) {
            double v = 0.0;
            if (e < 6) {           // slackTerminal = SS lam - x_N
                if (a.slackT) {
                    for (int l = 0; l < M; ++l) v += w.SS[e * M + l] * lam[l];
                    a.slackT[(long long)b * 6 + e] = v - w.x[N * 6 + e];
                }
            } else if (e < 12) {   // zt = Succ_SS lam
                if (a.zt && a.SuccSS) {
                    const double* S = a.SuccSS + (long long)b * 6 * SM + (e - 6) * M;
                    for (int l = 0; l < M; ++l) v += S[l] * lam[l];
                    a.zt[(long long)b * 6 + (e - 6)] = v;
                }
            } else {               // zt_u = Succ_uSS lam
                if (a.ztu && a.SuccU) {
                    const double* S = a.SuccU + (long long)b * 2 * SM + (e - 12) * M;
                    for (int l = 0; l < M; ++l) v += S[l] * lam[l];
                    a.ztu[(long long)b * 2 + (e - 12)] = v;
                }
            }
        }
    }
    if (lane == 0) {
        a.status[b] = info.status;
        a.iters[b] = info.iters;
        a.resid[(long long)b * 3 + 0] = info.r_prim;
        a.resid[(long long)b * 3 + 1] = info.r_dual;
        a.resid[(long long)b * 3 + 2] = info.gap;
        if (info.late && a.late) atomicAdd(a.late, 1ull);
    }
}

template <int N, int M>
static cudaError_t shaped_configure_t() {
    return cudaFuncSetAttribute(ftocp_shaped_kernel<N, M, 2, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)sizeof(KernelSmem<N, M, 2, 4, true>));
}

cudaError_t ftocp_shaped_configure(int N, int M) {
    cudaError_t e = cudaErrorInvalidValue;
#define SCASE(n, m) if (N == n && (m == 0 || m == M)) { e = shaped_configure_t<n, m>(); if (e != cudaSuccess) return e; }
    LMPC_FOR_EACH_CASE(SCASE)
#undef SCASE
    return e;
}

cudaError_t ftocp_shaped_launch(int N, int M, const FtocpConstRec* table, ShapedLaunch s, int n, FtocpArgs a, cudaStream_t st) {
    a.sets = table;
#define LCASE(n_, m_)                                                                                             \
    if (N == n_ && M == m_) {                                                                                     \
        ftocp_shaped_kernel<n_, m_, 2, 4><<<n, 32, sizeof(KernelSmem<n_, m_, 2, 4, true>), st>>>(s, a);           \
        return cudaGetLastError();                                                                                \
    }
    LMPC_FOR_EACH_CASE(LCASE)
#undef LCASE
    return cudaErrorInvalidValue;
}
