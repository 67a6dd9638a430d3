// racinglmpc_b200/csrc/ftocp_launch.cuh — the QP kernel and what launches it: the bulk-copy helpers, the launch arguments, the
// resident-warp bounds and the instantiated (horizon, safe-set size) grid.  One kernel template, two variants:
//   ftocp_kernel<..., false> (lmpc_b200.cu) : parameters of the whole launch in the constant bank (handles without parameter sets)
//   ftocp_kernel<..., true>  (ftocp_sets.cu) : each instance's parameters from a table (lmpc_set_param_sets)
// and, for handles with per-controller shapes, ftocp_shaped_kernel (ftocp_shapes.cu), a kernel of its own for the same reason.
// Each translation unit instantiates only its own variant, and the body is the kernel itself, not a function inlined into two
// wrappers.  Both matter for the uniform kernels' code: with both variants instantiated in one unit, or with the body inlined into
// two __global__ wrappers, the compiler scheduled all 30 uniform instantiations differently (profiles/h100_param_sets.txt).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "ftocp_pdip.cuh"
#include "lap_budget.cuh"

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

// One row of the per-controller parameter table: cp.async.bulk moves whole 16 B units, so the rows are padded to a multiple of 16 B
struct alignas(16) FtocpConstRec {
    FtocpConst c;
};
static_assert(sizeof(FtocpConstRec) % 16 == 0, "bulk copies need 16 B multiples");

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
    const FtocpConstRec* sets;   // the parameter table set_idx indexes (read by ftocp_kernel<..., true> only)
    LapBudget retire;     // lap budgets of the closed loop: the warp of a retired instance solves nothing; every other caller leaves it null

    // The instances [lo, lo + nb) of these arguments as a batch of their own, for the <N, M, 2, 4> kernel: every per-instance
    // pointer moves by lo instances (null ones stay null; a shared model, abc_inst_stride == 0, stays in place); the late counter
    // and the parameter table are shared by all instances
    FtocpArgs range(int lo, int nb, int N, int M) const {
        auto at = [lo](auto* p, long long per) { return p ? p + lo * per : p; };
        FtocpArgs r = *this;
        r.batch = nb;
        r.x0 = at(x0, 6); r.uOld = at(uOld, 2); r.abc = at(abc, abc_inst_stride);
        r.SS = at(SS, 6 * M); r.Qfun = at(Qfun, M); r.SuccSS = at(SuccSS, 6 * M); r.SuccU = at(SuccU, 2 * M);
        r.xPred = at(xPred, (N + 1) * 6); r.uPred = at(uPred, N * 2); r.slack = at(slack, N * 2);
        r.lambd = at(lambd, M); r.slackT = at(slackT, 6); r.zt = at(zt, 6); r.ztu = at(ztu, 2);
        r.status = at(status, 1); r.iters = at(iters, 1); r.resid = at(resid, 3);
        r.warm = at(warm, warm_stride); r.warm_valid = at(warm_valid, 1);
        r.set_idx = at(set_idx, 1);
        r.retire.budget = at(retire.budget, 1); r.retire.lap_n = at(retire.lap_n, 1);
        return r;
    }
};

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

// shared memory of one warp: the solver's workspace, the mbarrier of the staging copies and, with per-controller parameters, the
// instance's parameter record
template <int N, int M, int NCX, int NCU, bool SETS>
struct KernelSmem {
    Work<N, M, NCX, NCU> w;
    alignas(8) uint64_t bar;
};
template <int N, int M, int NCX, int NCU>
struct KernelSmem<N, M, NCX, NCU, true> {
    Work<N, M, NCX, NCU> w;
    FtocpConstRec c;
    alignas(8) uint64_t bar;
};

// the kernel's first parameter: the launch's parameters in the constant bank, or nothing when every instance reads its own record
template <bool SETS> struct ParamArg { using type = FtocpConst; };
template <> struct ParamArg<true> { struct type {}; };

// One warp (= one 32-thread CTA) per QP: stage the instance's model and safe set into shared memory, solve, unpack.
// SETS: the parameters are row a.sets[a.set_idx[b]], which lane 0 bulk-copies into shared memory on the same mbarrier as the stage
// model (sizeof(FtocpConstRec) more shared memory per warp); Pdip::solve is the same code, only the address space of c differs.
template <int N, int M, int NCX, int NCU, bool SETS>
__global__ void __launch_bounds__(32, ftocp_min_blocks(N, M, SETS ? (int)sizeof(FtocpConstRec) : 0))
    ftocp_kernel(const __grid_constant__ typename ParamArg<SETS>::type p, const FtocpArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using KS = KernelSmem<N, M, NCX, NCU, SETS>;
    KS& ks = *reinterpret_cast<KS*>(smem_raw);
    auto& w = ks.w;
    const int b = blockIdx.x;
    if (b >= a.batch) return;
    if (a.retire.retired(b)) return;       // before the mbarrier exists and before any bulk copy is in flight
    const int lane = threadIdx.x;

    // ---- stage the instance's model into shared memory (TMA 1-D bulk copies) ----
    if (lane == 0) {
        mbar_init(&ks.bar, 1);
        constexpr bool STREAM = Work<N, M, NCX, NCU>::STREAM;   // long horizons read the stage model in place (ftocp_pdip.cuh)
        uint32_t bytes = (STREAM ? 0 : N * 54 * 8) + (M > 0 ? (6 * M + M) * 8 : 0) + (SETS ? (uint32_t)sizeof(FtocpConstRec) : 0);
        mbar_expect_tx(&ks.bar, bytes);
        if constexpr (SETS) bulk_g2s(&ks.c, a.sets + a.set_idx[b], sizeof(FtocpConstRec), &ks.bar);
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
    const FtocpConst* c;
    if constexpr (SETS) c = &ks.c.c;
    else c = &p;
    SolveInfo info;
    Pdip<N, M, NCX, NCU>::solve(w, *c, x0, info, (M > 0) ? w.d4i : nullptr, a.slack ? a.slack + (long long)b * N * NCX : nullptr,
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

// The supported (horizon, safe-set size) grid: one instantiation of the solver per pair.
// Horizons 4..48 with and without the reference's 48-point safe set (initControllerParameters.py:43-44), and other safe-set
// sizes (numSS_it x even points per lap) at the reference's and BASELINE's horizons.
#define LMPC_FOR_EACH_CASE(X) \
    X(4, 0) X(6, 0) X(8, 0) X(10, 0) X(12, 0) X(14, 0) X(16, 0) X(20, 0) X(24, 0) X(32, 0) X(48, 0) \
    X(4, 48) X(6, 48) X(8, 48) X(10, 48) X(12, 48) X(14, 48) X(16, 48) X(20, 48) X(24, 48) X(32, 48) X(48, 48) \
    X(12, 24) X(12, 32) X(12, 64) X(12, 96) X(14, 24) X(14, 32) X(14, 64) X(14, 96)
#define LMPC_GRID_TEXT "N in {4,6,8,10,12,14,16,20,24,32,48} with numSS_Points in {0,48}; N in {12,14} also with numSS_Points in {24,32,64,96}"

// ftocp_sets.cu: opt the SETS instantiations (N, M) and (N, 0) into their shared-memory size on the current device, and launch one
// with a.sets = table; both return a CUDA error code (cudaErrorInvalidValue for a pair outside the grid)
cudaError_t ftocp_sets_configure(int N, int M);
cudaError_t ftocp_sets_launch(int N, int M, const FtocpConstRec* table, FtocpArgs a, cudaStream_t st);

// ftocp_shapes.cu: the QP kernel of handles with per-controller shapes (lmpc_set_shapes), ftocp_shaped_kernel<N_b, M_b, 2, 4>.  One
// launch covers the controllers inst[0 .. n) of one shape; each reads its parameters from the table a.sets (row a.set_idx[b], or
// row 0 when a.set_idx is null) and addresses every buffer with the handle's strides N, M (M = 0: no safe set).
struct ShapedLaunch {
    const int* inst;
    int N, M;
};
// opt the shaped instantiations (N, M) and (N, 0) into their shared-memory size on the current device; launch n controllers of
// shape (N, M) with a.sets = table.  Both return a CUDA error code (cudaErrorInvalidValue for a pair outside the grid).
cudaError_t ftocp_shaped_configure(int N, int M);
cudaError_t ftocp_shaped_launch(int N, int M, const FtocpConstRec* table, ShapedLaunch s, int n, FtocpArgs a, cudaStream_t st);
