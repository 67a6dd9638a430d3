// tests/support/host_core.cpp — TEST INFRASTRUCTURE ONLY.
// Compiles racinglmpc_b200/csrc/ftocp_pdip.cuh as a 1-lane host emulation so that the solver's
// arithmetic can be checked against the oracle on a machine without a GPU.  Never loaded by the
// product package (racinglmpc_b200 fails loudly when its CUDA library is missing).
#include "../../racinglmpc_b200/csrc/ftocp_pdip.cuh"
#include <new>
#include <cstring>

using namespace lmpc;

// Every (N, M) pair of LMPC_FOR_EACH_CASE (racinglmpc_b200/csrc/ftocp_launch.cuh, which needs the CUDA toolkit and is not
// included here).  tests/test_qp_iterates.py parses that list and checks that this one solves every pair of it.
#define HOST_FOR_EACH_CASE(X) \
    X(4, 0) X(6, 0) X(8, 0) X(10, 0) X(12, 0) X(14, 0) X(16, 0) X(20, 0) X(24, 0) X(32, 0) X(48, 0) \
    X(4, 48) X(6, 48) X(8, 48) X(10, 48) X(12, 48) X(14, 48) X(16, 48) X(20, 48) X(24, 48) X(32, 48) X(48, 48) \
    X(12, 24) X(12, 32) X(12, 64) X(12, 96) X(14, 24) X(14, 32) X(14, 64) X(14, 96)

template <int N, int M>
static int run(const FtocpConst* c, const double* abc, const double* ss, const double* qfun, const double* x0,
               const double* uold, double* xpred, double* upred, double* lam, double* slack, double* info_out, double* warm, int* warm_valid) {
    using P = Pdip<N, M, 2, 4>;
    typename P::W* w = new typename P::W();
    std::memcpy(w->ABC, abc, sizeof(double) * N * 54);
    if (M > 0) {
        std::memcpy(w->SS, ss, sizeof(double) * 6 * M);
        std::memcpy(w->Qfun, qfun, sizeof(double) * M);
    }
    w->uOld[0] = uold[0];
    w->uOld[1] = uold[1];
    SolveInfo info;
    P::solve(*w, *c, x0, info, lam, slack, warm, warm ? warm_valid : nullptr);
    std::memcpy(xpred, w->x, sizeof(double) * (N + 1) * 6);
    std::memcpy(upred, w->u, sizeof(double) * N * 2);
    info_out[0] = info.status; info_out[1] = info.iters; info_out[2] = info.r_prim; info_out[3] = info.r_dual; info_out[4] = info.gap;
    info_out[5] = info.late;
    delete w;
    return info.status;
}

extern "C" int host_core_solve(int N, int M, const FtocpConst* c, const double* abc, const double* ss, const double* qfun,
                               const double* x0, const double* uold, double* xpred, double* upred, double* lam,
                               double* slack, double* info_out, double* warm, int* warm_valid) {
#define CASE(n, m) if (N == n && M == m) return run<n, m>(c, abc, ss, qfun, x0, uold, xpred, upred, lam, slack, info_out, warm, warm_valid);
    HOST_FOR_EACH_CASE(CASE)
#undef CASE
    return -1;
}
// The starting point Pdip::warm_point builds from a warm-start record wb (WS_SIZE doubles), before any iteration:
// out = x [(N+1)*6] | u [N*2] | s, nu1, nu3 [N*2 each] | nu2 [N*4] | lam, nu4 [M each] | y1.
template <int N, int M>
static int warm_point_run(const FtocpConst* c, const double* abc, const double* x0, const double* wb, double* out) {
    using P = Pdip<N, M, 2, 4>;
    typename P::W* w = new typename P::W();
    typename P::RG* g = new typename P::RG();
    std::memcpy(w->ABC, abc, sizeof(double) * N * 54);
    P::warm_point(*w, *g, *c, x0, wb);
    double* o = out;
    auto put = [&](const double* src, int n) { std::memcpy(o, src, sizeof(double) * n); o += n; };
    put(w->x, (N + 1) * 6); put(w->u, N * 2);
    put(g->s, P::R1); put(g->nu1, P::R1); put(g->nu3, P::R1); put(g->nu2, P::R2);
    if (M > 0) { put(g->lam, M); put(g->nu4, M); put(&g->y1, 1); }
    delete g;
    delete w;
    return P::WS_SIZE;
}

extern "C" int host_core_warm_point(int N, int M, const FtocpConst* c, const double* abc, const double* x0, const double* wb,
                                    double* out) {
#define CASE(n, m) if (N == n && M == m) return warm_point_run<n, m>(c, abc, x0, wb, out);
    HOST_FOR_EACH_CASE(CASE)
#undef CASE
    return -1;
}
#ifdef LMPC_HOST_COUNT
// Branch counts since the last reset: corrector passes, recentring passes, step reductions (the discrete decisions of an
// interior-point iteration that rounding can flip)
extern "C" void host_core_counts(long* out3, int reset) {
    for (int i = 0; i < 3; ++i) { out3[i] = lmpc::g_host_count[i]; if (reset) lmpc::g_host_count[i] = 0; }
}
#endif
extern "C" int host_core_const_size() { return (int)sizeof(FtocpConst); }
