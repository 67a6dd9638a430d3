// racinglmpc_b200/csrc/ftocp_sets.cu — the QP kernel for handles with per-controller parameters (lmpc_set_param_sets).
// A separate translation unit from lmpc_b200.cu: see ftocp_launch.cuh.
#include "ftocp_launch.cuh"

// the same plus the instance's own parameter record (ftocp_sets_kernel)
template <int N, int M, int NCX, int NCU>
struct KernelSmemSets {
    Work<N, M, NCX, NCU> w;
    FtocpConstRec c;
    alignas(8) uint64_t bar;
};

// Handles with per-controller parameters (lmpc_set_param_sets): ftocp_kernel with the parameters read from the instance's row
// table[set_idx[b]], which lane 0 bulk-copies into shared memory on the same mbarrier as the stage model (sizeof(FtocpConstRec)
// more shared memory per warp).  Pdip::solve is the same code; only the address space of c differs.  The uniform ftocp_kernel
// (lmpc_b200.cu) stays the headline path (parameters in the constant bank, no copy) and is kept textually separate: moving the
// shared body into one inlined function changed the instruction schedule of all 30 uniform instantiations.  The body below is
// ftocp_kernel's plus exactly three edits (the KernelSmemSets layout, the record's bulk copy and its bytes on the mbarrier, and
// `c` bound to the staged record); tests/test_param_sets.py checks that correspondence, so the two cannot drift apart.
template <int N, int M, int NCX, int NCU>
__global__ void __launch_bounds__(32, ftocp_min_blocks(N, M, (int)sizeof(FtocpConstRec)))
    ftocp_sets_kernel(const FtocpConstRec* __restrict__ table, const FtocpArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using KS = KernelSmemSets<N, M, NCX, NCU>;
    KS& ks = *reinterpret_cast<KS*>(smem_raw);
    auto& w = ks.w;
    const int b = blockIdx.x;
    if (b >= a.batch) return;
    const int lane = threadIdx.x;

    // ---- stage the instance's model into shared memory (TMA 1-D bulk copies) ----
    if (lane == 0) {
        mbar_init(&ks.bar, 1);
        constexpr bool STREAM = Work<N, M, NCX, NCU>::STREAM;   // long horizons read the stage model in place (ftocp_pdip.cuh)
        uint32_t bytes = (STREAM ? 0 : N * 54 * 8) + (M > 0 ? (6 * M + M) * 8 : 0) + (uint32_t)sizeof(FtocpConstRec);
        mbar_expect_tx(&ks.bar, bytes);
        bulk_g2s(&ks.c, table + a.set_idx[b], sizeof(FtocpConstRec), &ks.bar);
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
            bulk_g2s(&w.SS[0], a.SS + (long long)b * 6 * M, 6 * M * 8, &ks.bar);
            bulk_g2s(&w.Qfun[0], a.Qfun + (long long)b * M, M * 8, &ks.bar);
        }
    }
    double x0[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) x0[i] = a.x0[(long long)b * 6 + i];
    if (lane < 2) w.uOld[lane] = a.uOld[(long long)b * 2 + lane];
    __syncwarp();
    mbar_wait(&ks.bar, 0);

    // ---- solve ----
    const FtocpConst& c = ks.c.c;
    SolveInfo info;
    Pdip<N, M, NCX, NCU>::solve(w, c, x0, info, (M > 0) ? w.d4i : nullptr, a.slack ? a.slack + (long long)b * N * NCX : nullptr,
                                a.warm ? a.warm + (long long)b * a.warm_stride : nullptr, a.warm ? a.warm_valid + b : nullptr);

    // ---- unpack (PC.py:364-384) ----
    for (int e = lane; e < (N + 1) * 6; e += 32) a.xPred[(long long)b * (N + 1) * 6 + e] = w.x[e];
    for (int e = lane; e < N * 2; e += 32) a.uPred[(long long)b * N * 2 + e] = w.u[e];
    if (M > 0) {
        const double* lam = w.d4i;   // solve() left lambda here
        if (a.lambd)
            for (int e = lane; e < M; e += 32) a.lambd[(long long)b * M + e] = lam[e];
        for (int e = lane; e < 14; e += 32) {
            double v = 0.0;
            if (e < 6) {           // slackTerminal = SS lam - x_N
                if (a.slackT) {
                    for (int l = 0; l < M; ++l) v += w.SS[e * M + l] * lam[l];
                    a.slackT[(long long)b * 6 + e] = v - w.x[N * 6 + e];
                }
            } else if (e < 12) {   // zt = Succ_SS lam
                if (a.zt && a.SuccSS) {
                    const double* S = a.SuccSS + ((long long)b * 6 + (e - 6)) * M;
                    for (int l = 0; l < M; ++l) v += S[l] * lam[l];
                    a.zt[(long long)b * 6 + (e - 6)] = v;
                }
            } else {               // zt_u = Succ_uSS lam
                if (a.ztu && a.SuccU) {
                    const double* S = a.SuccU + ((long long)b * 2 + (e - 12)) * M;
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
static cudaError_t sets_configure_t() {
    return cudaFuncSetAttribute(ftocp_sets_kernel<N, M, 2, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)sizeof(KernelSmemSets<N, M, 2, 4>));
}

cudaError_t ftocp_sets_configure(int N, int M) {
    cudaError_t e = cudaErrorInvalidValue;
#define SCASE(n, m) if (N == n && (m == 0 || m == M)) { e = sets_configure_t<n, m>(); if (e != cudaSuccess) return e; }
    LMPC_FOR_EACH_CASE(SCASE)
#undef SCASE
    return e;
}

cudaError_t ftocp_sets_launch(int N, int M, const FtocpConstRec* table, const FtocpArgs& a, cudaStream_t st) {
#define LCASE(n, m)                                                                                               \
    if (N == n && M == m) {                                                                                       \
        ftocp_sets_kernel<n, m, 2, 4><<<a.batch, 32, sizeof(KernelSmemSets<n, m, 2, 4>), st>>>(table, a);        \
        return cudaGetLastError();                                                                                \
    }
    LMPC_FOR_EACH_CASE(LCASE)
#undef LCASE
    return cudaErrorInvalidValue;
}
