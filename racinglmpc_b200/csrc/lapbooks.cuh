// racinglmpc_b200/csrc/lapbooks.cuh — the reference's per-controller lap bookkeeping, on the device.
//
// LMPC and PredictiveModel keep Python lists of laps and decide from them, once per lap, which stored laps the next lap
// uses:  LMPC.addTrajectory appends (SS, uSS, Qfun, LapTime) and `it += 1` (PC.py:418-445); addTerminalComponents takes
// np.argsort(LapTime)[:numSS_it] (PC.py:395,402) and treats lap it-1 specially (PC.py:506-512; addPoint extends it,
// PC.py:466-476); PredictiveModel.addTrajectory keeps laps sorted by length so that usedIt = [0..trToUse) are the shortest
// (PredictiveModel.py:31,35-46).  For a Monte-Carlo batch these decisions are made for thousands of controllers in the same
// step, so they live here: one thread per controller walks its (at most 8-entry) slot tables.  Only laps that can still be
// selected are stored (a lap that is not among the fastest when it arrives never becomes one: faster laps only push it
// further down), which makes the fixed-capacity pools equivalent to the reference's unbounded lists as long as the laps that
// must stay resident fit (health bit 64 otherwise).  tests/support/lapbook_exact.py restates the lists and the tests compare
// the tables with them after every hand-over and import.
//
// Slot tables per controller b:  safe set  ss_time[b][cap], ss_lap[b][cap] (lap number, -1 = free), it[b];
//                                model     md_time[b][mcap], md_seq[b][mcap] (arrival order, -1 = free), md_cnt[b].
// Orders are the reference's: stable argsort of LapTime = ascending (time, lap number); model laps ascending (rows, arrival).
#pragma once
#include "safeset.cuh"

namespace lmpc {

struct LapBooks {
    int *ss_time, *ss_lap, *it;
    int *md_time, *md_seq, *md_cnt;
    int *sel, *isprev, *prevslot, *used;   // what K2 / addPoint / K1 read (same arrays the host-driven path uploads)
    int *lap_hist, *lap_n;                 // lengths of the laps a controller drove itself [B][LAP_HIST], count [B]
    int ss_cap, md_cap, numSS_it, trToUse;
};
constexpr int LAP_HIST = 16;

__device__ __forceinline__ bool key_less(int t1, int n1, int t2, int n2) { return t1 < t2 || (t1 == t2 && n1 < n2); }

// The lap windows of every controller (lmpc_set_lap_windows): ss_window / model_window most recent laps, 0 = unbounded.  Without a
// window table (tab == null) every window is unbounded.
using LapWindowRec = lmpc_lap_window_params;
using LapWindows = Table<LapWindowRec>;
__device__ __forceinline__ LapWindowRec book_windows(const LapWindows& w, int b) { return w.tab ? w.of(b) : LapWindowRec{0, 0}; }

// The lane rules of every controller (lmpc_set_lane_rules) and the QP constants (Fx, bx) they judge against: the controller's
// parameter-set row, else the handle's.  Without a rule table (rule.tab == null) no lap is judged and the key of a lap is its lap
// time.
using LaneRuleRec = lmpc_lane_rule_params;
struct LaneRules {
    Table<LaneRuleRec> rule;
    Table<FtocpConstRec> qp;
};

// Does the lap x[0 .. T) (row r at x + r * stride, its state in the first 6 entries) leave the lane Fx x <= bx of c by more than
// tol?  A row does when an entry is not finite or d_i = Fx[i] . x - bx[i] > tol for one of the ncx == 2 lane rows, evaluated in
// order without contraction: the arithmetic of report_step (safeset.cuh), kept as a copy rather than a helper shared with the
// closed loop's step kernel.  One block-wide pass; every thread of the block must call it.
__device__ __forceinline__ bool lane_leaves_block(const FtocpConst& c, const double* x, int T, int stride, double tol) {
    bool bad = false;
    for (int t = threadIdx.x; t < T && !bad; t += blockDim.x) {
        const double* xr = x + (size_t)t * stride;
        double v[6];
        bool finite = true;
#pragma unroll
        for (int j = 0; j < 6; ++j) { v[j] = xr[j]; finite = finite && isfinite(v[j]); }
        if (!finite) { bad = true; break; }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            double s = __dmul_rn(c.Fx[i * 6], v[0]);
#pragma unroll
            for (int j = 1; j < 6; ++j) s = __dadd_rn(s, __dmul_rn(c.Fx[i * 6 + j], v[j]));
            bad = bad || __dsub_rn(s, c.bx[i]) > tol;
        }
    }
    return __syncthreads_or(bad) != 0;
}

// Is the lap x[0 .. T) lane-unsafe for controller b: does it leave its lane by more than its lane_tol?  False without a table or
// under mode 0.  Both tests are uniform over the block (a kernel argument, the controller's own row): no barrier is skipped by part
// of it.
__device__ __forceinline__ bool lane_unsafe_block(const LaneRules& lr, int b, const double* x, int T, int stride) {
    if (!lr.rule.tab) return false;
    const LaneRuleRec r = lr.rule.of(b);
    if (r.mode != 1) return false;
    return lane_leaves_block(lr.qp.of(b).c, x, T, stride, r.lane_tol);
}
// The safe-set key a lap of lap time T is filed with: T, plus LMPC_LANE_UNSAFE_KEY when it was judged lane-unsafe
__device__ __forceinline__ int lane_key(int T, bool unsafe) { return unsafe ? T + LMPC_LANE_UNSAFE_KEY : T; }
// The lap time of a safe-set key (the pooled export ranks and ships raw lap times); rules: a lane-rule table is installed.  Without
// one a key is its lap time, whatever its value.
__device__ __forceinline__ int lane_lap_time(int key, bool rules) { return rules && key >= LMPC_LANE_UNSAFE_KEY ? key - LMPC_LANE_UNSAFE_KEY : key; }

// The lane margins of every controller (lmpc_set_lane_margins): the table, the untightened QP rows (the controller's parameter-set
// row, else the handle's), the derived planning rows plan[B] (the source row with bx_i - m_b) that every QP of the handle reads,
// the margins m[B] and the warm-start validity (null without warm start).  Without a margin table (rule.tab == null)
// commit_laps_books_kernel reads none of it.
using LaneMarginRec = lmpc_lane_margin_params;
struct LaneMargins {
    Table<LaneMarginRec> rule;
    Table<FtocpConstRec> qp;
    FtocpConstRec* plan;
    double* m;
    int* warm_valid;
};
// Row b of the planning table plans with margin m: the lane rows of its source row, moved in by m (rounded once)
__device__ __forceinline__ void margin_plan_bx(const LaneMargins& lm, int b, double m) {
    const FtocpConst& src = lm.qp.of(b).c;
#pragma unroll
    for (int i = 0; i < 2; ++i) lm.plan[b].c.bx[i] = __dsub_rn(src.bx[i], m);
}
// The margin after a lap under a mode 2 row r: up by step_up after a lap that left the lane, down by step_down after one that kept
// to it, within [margin0, margin_max]
__device__ __forceinline__ double margin_adapt(const LaneMarginRec& r, double m, bool left) {
    return left ? fmin(__dadd_rn(m, r.step_up), r.margin_max) : fmax(__dsub_rn(m, r.step_down), r.margin0);
}

// Every controller's planning row from its source row and its margin: m_b = 0 (mode 0), margin0 (mode 1), margin0 under mode 2
// when reset2 (the install and the seedings), else the m_b it has (lmpc_set_param_sets, a snapshot restore).  idx[b] = b: the
// identity index the QP kernels read the table through.  One CTA of 128 threads per controller copies the 1 776-byte row.
__global__ void __launch_bounds__(128) lane_margin_rows_kernel(int batch, LaneMargins lm, int* idx, int reset2) {
    const int b = blockIdx.x;
    if (b >= batch) return;
    const uint4* src = reinterpret_cast<const uint4*>(&lm.qp.of(b));
    uint4* dst = reinterpret_cast<uint4*>(lm.plan + b);
    for (int e = threadIdx.x; e < (int)(sizeof(FtocpConstRec) / 16); e += blockDim.x) dst[e] = src[e];
    __syncthreads();
    if (threadIdx.x == 0) {
        const LaneMarginRec r = lm.rule.of(b);
        const double m = r.mode == 0 ? 0.0 : r.mode == 1 || reset2 ? r.margin0 : lm.m[b];
        lm.m[b] = m;
        margin_plan_bx(lm, b, m);
        idx[b] = b;
    }
}

// book_ss_add under a safe-set window of W >= 1 laps: after the event the window is lap numbers [it' - W, it'), it' = it + 1.  A
// lap stays stored while it is in the window and fewer than nit NEWER laps rank ahead of it: older laps leave the window before it
// does, newer ones stay as long as it does, so only they can keep it out of the selection for good.  An import's only newer lap
// is the own latest: it is not stored when it lies outside the window on arrival (W = 1) or nit == 1 and the own latest is faster.
// Among the stored laps that can no longer be selected the slowest, then the oldest, is evicted, as without a window.  With
// W <= ss_cap a lap outside the window is always there to evict, so -2 needs W > ss_cap.
__device__ inline int book_ss_add_window(const LapBooks& k, int b, int T, bool import, int nit, int W) {
    int* tm = k.ss_time + (size_t)b * k.ss_cap;
    int* ln = k.ss_lap + (size_t)b * k.ss_cap;
    const int it = k.it[b];
    const int lapno = import ? it - 1 : it;
    const int lo = it + 1 - W;                                   // oldest lap number of the window after the event
    if (import) {
        if (it < 1) return -1;
        int ahead = 0;                                           // the own latest (it-1 -> it) ahead of the new lap
        for (int s = 0; s < k.ss_cap; ++s) if (ln[s] == it - 1 && key_less(tm[s], it, T, lapno)) ahead = 1;
        if (lapno < lo || ahead >= nit) return -1;               // never selected -> not stored
        for (int s = 0; s < k.ss_cap; ++s) if (ln[s] == it - 1) ln[s] = it;
    }
    int slot = -1;
    for (int s = 0; s < k.ss_cap; ++s) if (ln[s] < 0) { slot = s; break; }
    if (slot < 0) {
        int vt = -1, vn = 0;
        for (int s = 0; s < k.ss_cap; ++s) {
            if (import && ln[s] == it) continue;                 // the own latest lap stays
            if (ln[s] >= lo) {                                   // in the window: evictable once nit newer laps rank ahead
                int newer = key_less(T, lapno, tm[s], ln[s]) ? 1 : 0;    // every candidate is older than the new lap
                for (int j = 0; j < k.ss_cap; ++j) if (ln[j] > ln[s] && key_less(tm[j], ln[j], tm[s], ln[s])) ++newer;
                if (newer < nit) continue;
            }
            if (slot < 0 || tm[s] > vt || (tm[s] == vt && ln[s] < vn)) { slot = s; vt = tm[s]; vn = ln[s]; }
        }
        if (slot < 0) {
            if (import) for (int s = 0; s < k.ss_cap; ++s) if (ln[s] == it) ln[s] = it - 1;
            return -2;
        }
    }
    tm[slot] = T;
    ln[slot] = lapno;
    k.it[b] = it + 1;
    return slot;
}

// book_md_add under a model window of W >= 1 laps: arrival numbers [md_cnt' - W, md_cnt').  The new lap has no newer lap, so it is
// always stored; a stored lap stays while it is in the window and fewer than trToUse newer laps are shorter.  Among the others
// the slowest (length, arrival) is evicted; with W <= md_cap there always is one.
__device__ inline int book_md_add_window(const LapBooks& k, int b, int T, int W) {
    int* tm = k.md_time + (size_t)b * k.md_cap;
    int* sq = k.md_seq + (size_t)b * k.md_cap;
    const int seq = k.md_cnt[b];
    k.md_cnt[b] = seq + 1;
    const int lo = seq + 1 - W;
    int slot = -1;
    for (int s = 0; s < k.md_cap; ++s) if (sq[s] < 0) { slot = s; break; }
    if (slot < 0) {
        int vt = -1, vs = -1, any = -1, at = -1, as = -1;
        for (int s = 0; s < k.md_cap; ++s) {
            if (any < 0 || key_less(at, as, tm[s], sq[s])) { any = s; at = tm[s]; as = sq[s]; }
            if (sq[s] >= lo) {
                int newer = (T < tm[s]) ? 1 : 0;                 // the new lap is newer than every stored one
                for (int j = 0; j < k.md_cap; ++j) if (sq[j] > sq[s] && key_less(tm[j], sq[j], tm[s], sq[s])) ++newer;
                if (newer < k.trToUse) continue;
            }
            if (slot < 0 || key_less(vt, vs, tm[s], sq[s])) { slot = s; vt = tm[s]; vs = sq[s]; }
        }
        if (slot < 0) slot = any;
    }
    tm[slot] = T;
    sq[slot] = seq;
    return slot;
}

// LMPC.addTrajectory bookkeeping for a lap of `T` rows.  import == false: the controller's own new lap (lap number it).
// import == true: a lap another controller drove, filed BEFORE the controller's own latest lap (which stays lap it-1, the one
// addPoint extends): it takes lap number it-1, the own latest moves to it; it is skipped (-1) when it would not be among the
// nit fastest (nit: the controller's numSS_it).  Returns the slot to copy the lap into, -1 = not stored, -2 = pool too small (the
// tables are left as they were).  W: the controller's safe-set window, 0 = unbounded; W > 0 files under book_ss_add_window.
__device__ inline int book_ss_add(const LapBooks& k, int b, int T, bool import, int nit, int W) {
    if (W > 0) return book_ss_add_window(k, b, T, import, nit, W);
    int* tm = k.ss_time + (size_t)b * k.ss_cap;
    int* ln = k.ss_lap + (size_t)b * k.ss_cap;
    const int it = k.it[b];
    const int lapno = import ? it - 1 : it;
    if (import) {
        if (it < 1) return -1;
        // numbers after the insertion: own latest it-1 -> it.  Rank of the new lap among the stored ones:
        int rank = 0;
        for (int s = 0; s < k.ss_cap; ++s)
            if (ln[s] >= 0) { const int n2 = (ln[s] == it - 1) ? it : ln[s]; if (key_less(tm[s], n2, T, lapno)) ++rank; }
        if (rank >= nit) return -1;                              // never selected (PC.py:395) -> not stored
        for (int s = 0; s < k.ss_cap; ++s) if (ln[s] == it - 1) ln[s] = it;
    }
    int slot = -1;
    for (int s = 0; s < k.ss_cap; ++s) if (ln[s] < 0) { slot = s; break; }
    if (slot < 0) {                                              // evict a stored lap that can no longer be selected
        int vt = -1, vn = 0;
        for (int s = 0; s < k.ss_cap; ++s) {
            if (import && ln[s] == it) continue;                 // the own latest lap stays
            int rank = key_less(T, lapno, tm[s], ln[s]) ? 1 : 0;
            for (int j = 0; j < k.ss_cap; ++j) if (j != s && key_less(tm[j], ln[j], tm[s], ln[s])) ++rank;
            if (rank < nit) continue;                            // one of the fastest: keep
            if (slot < 0 || tm[s] > vt || (tm[s] == vt && ln[s] < vn)) { slot = s; vt = tm[s]; vn = ln[s]; }
        }
        if (slot < 0) {                                          // nothing filed: the own latest lap keeps its number
            if (import) for (int s = 0; s < k.ss_cap; ++s) if (ln[s] == it) ln[s] = it - 1;
            return -2;
        }
    }
    tm[slot] = T;
    ln[slot] = lapno;
    k.it[b] = it + 1;
    return slot;
}

// PredictiveModel.addTrajectory bookkeeping for a lap of `T` rows.  Returns the slot, or -1 when the lap can never be among
// the trToUse shortest.  W: the controller's model window, 0 = unbounded; W > 0 files under book_md_add_window.
__device__ inline int book_md_add(const LapBooks& k, int b, int T, int W) {
    if (W > 0) return book_md_add_window(k, b, T, W);
    int* tm = k.md_time + (size_t)b * k.md_cap;
    int* sq = k.md_seq + (size_t)b * k.md_cap;
    const int seq = k.md_cnt[b];
    k.md_cnt[b] = seq + 1;
    int rank = 0, stored = 0;
    for (int s = 0; s < k.md_cap; ++s) if (sq[s] >= 0) { ++stored; if (tm[s] <= T) ++rank; }   // bisect_right: ties stay ahead
    if (!(rank < k.trToUse || seq + 1 <= k.trToUse)) return -1;
    int slot = -1;
    for (int s = 0; s < k.md_cap; ++s) if (sq[s] < 0) { slot = s; break; }
    if (slot < 0) {                                              // evict the slowest stored lap outside the new usedIt
        int vt = -1, vs = -1, any = -1, at = -1, as = -1;
        for (int s = 0; s < k.md_cap; ++s) {
            int r2 = (T < tm[s]) ? 1 : 0;                        // the new lap sorts before s only when strictly shorter
            for (int j = 0; j < k.md_cap; ++j) if (j != s && key_less(tm[j], sq[j], tm[s], sq[s])) ++r2;
            if (any < 0 || key_less(at, as, tm[s], sq[s])) { any = s; at = tm[s]; as = sq[s]; }
            if (r2 < k.trToUse) continue;
            if (slot < 0 || key_less(vt, vs, tm[s], sq[s])) { slot = s; vt = tm[s]; vs = sq[s]; }
        }
        if (slot < 0) slot = any;
    }
    tm[slot] = T;
    sq[slot] = seq;
    return slot;
}

// What the next lap reads: the nit fastest safe-set laps in argsort order (nit: the controller's numSS_it), which of them is lap
// it-1, the slot addPoint extends, and usedIt of the regression model.  Returns 0, or 8 when fewer than nit laps are stored (the
// reference raises IndexError at PC.py:402-403).  Entries nit .. k.numSS_it-1 of sel repeat the last selected slot and those of
// isprev are 0: K2 reads none of them, and a snapshot packs them as they are.  Only laps in the controller's windows w count
// (lap numbers >= it - ss_window, arrival numbers >= md_cnt - model_window; a window of 0 starts at 0, and a free slot, -1, is
// below every start).
__device__ inline int book_refresh(const LapBooks& k, int b, int nit, LapWindowRec w) {
    const int* tm = k.ss_time + (size_t)b * k.ss_cap;
    const int* ln = k.ss_lap + (size_t)b * k.ss_cap;
    const int it = k.it[b];
    const int lo = w.ss_window > 0 ? max(it - w.ss_window, 0) : 0;
    int flag = 0, prev = -1, last = 0;
    for (int s = 0; s < k.ss_cap; ++s) if (it > 0 && ln[s] == it - 1) prev = s;   // it = 0: no lap (a free slot has ln = -1)
    for (int c = 0; c < nit; ++c) {
        int best = -1;
        for (int s = 0; s < k.ss_cap; ++s) {
            if (ln[s] < lo) continue;
            int rank = 0;
            for (int j = 0; j < k.ss_cap; ++j) if (j != s && ln[j] >= lo && key_less(tm[j], ln[j], tm[s], ln[s])) ++rank;
            if (rank == c) best = s;
        }
        if (best < 0) { flag = 8; best = last; } else last = best;
        k.sel[(size_t)b * k.numSS_it + c] = best;
        k.isprev[(size_t)b * k.numSS_it + c] = (it > 0 && ln[best] == it - 1) ? 1 : 0;
    }
    for (int c = nit; c < k.numSS_it; ++c) { k.sel[(size_t)b * k.numSS_it + c] = last; k.isprev[(size_t)b * k.numSS_it + c] = 0; }
    k.prevslot[b] = prev;
    const int* mt = k.md_time + (size_t)b * k.md_cap;
    const int* ms = k.md_seq + (size_t)b * k.md_cap;
    const int lom = w.model_window > 0 ? max(k.md_cnt[b] - w.model_window, 0) : 0;
    last = 0;
    for (int c = 0; c < k.trToUse; ++c) {
        int best = -1;
        for (int s = 0; s < k.md_cap; ++s) {
            if (ms[s] < lom) continue;
            int rank = 0;
            for (int j = 0; j < k.md_cap; ++j) if (j != s && ms[j] >= lom && key_less(mt[j], ms[j], mt[s], ms[s])) ++rank;
            if (rank == c) best = s;
        }
        if (best < 0) best = last; else last = best;             // fewer laps than trToUse: the slowest one repeats
        k.used[(size_t)b * k.trToUse + c] = best;
    }
    return flag;
}

// The selection of tables written from outside (lmpc_books_set): book_refresh of every controller.  One thread per controller.
__global__ void books_refresh_kernel(int batch, LapBooks k, SsLaps laps, LapWindows win) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) book_refresh(k, b, ss_laps_of(laps, b, k.numSS_it), book_windows(win, b));
}

// Lap hand-over of every controller whose lap just ended (done[b] != 0), bookkeeping included: main.py:113-119
// (lmpc.addTrajectory + predictiveModel.addTrajectory of the lap Simulator.sim returned), SysModel.py:50 (s -= TrackLength),
// PC.py:445 (timeStep = 0).  One CTA per controller; no host involvement.  Each table below is read only while it is installed.
// Lap reports: the running report row is filed as the lap's.  Lane rules: the lap's rows 0 .. Trec-1 are judged and an unsafe
// lap is filed with its lap time + LMPC_LANE_UNSAFE_KEY as its safe-set key (its report carries LMPC_REPORT_LANE_UNSAFE).
// Lane margins: under a mode 2 row the same rows adapt the margin m_b (margin_adapt, threshold 0), and a margin that changed
// rewrites the controller's planning bx and invalidates its warm-start record.
__global__ void __launch_bounds__(256) commit_laps_books_kernel(int batch, LapPool ss, LapPool model, LapBooks k, const double* cl_x,
                                                                const double* cl_u, int* cl_len, int Tcl, double* x_cur, int* timeStep,
                                                                int* done, int* flags_or, Tracks trk, int lmpc, LapBudget retire,
                                                                SsLaps laps, LapReports rep, LapWindows win, LaneRules lane,
                                                                LaneMargins margin) {
    const int b = blockIdx.x;
    if (b >= batch || retire.retired(b) || !done[b]) return;
    __shared__ int s_ss, s_md;
    const int Trec = cl_len[b];
    const double TrackLength = trk.of(b).TrackLength;
    const bool unsafe = lane_unsafe_block(lane, b, cl_x + (size_t)b * Tcl * 6, Trec, 6);
    if (margin.rule.tab) {
        const LaneMarginRec r = margin.rule.of(b);
        if (r.mode == 2) {                                       // uniform over the block: no barrier is skipped by part of it
            const bool left = lane_leaves_block(margin.qp.of(b).c, cl_x + (size_t)b * Tcl * 6, Trec, 6, 0.0);
            if (threadIdx.x == 0) {
                const double m0 = margin.m[b], m1 = margin_adapt(r, m0, left);
                if (m1 != m0) {
                    margin.m[b] = m1;
                    margin_plan_bx(margin, b, m1);
                    if (margin.warm_valid) margin.warm_valid[b] = 0;
                }
            }
        }
    }
    if (threadIdx.x == 0) {
        const LapWindowRec w = book_windows(win, b);
        s_ss = lmpc ? book_ss_add(k, b, lane_key(Trec, unsafe), false, ss_laps_of(laps, b, k.numSS_it), w.ss_window) : -1;   // ordered by the lap time; rows beyond Tmax are not stored
        s_md = book_md_add(k, b, Trec, w.model_window);
        const int n = k.lap_n[b];
        if (n < LAP_HIST) k.lap_hist[(size_t)b * LAP_HIST + n] = Trec;
        k.lap_n[b] = n + 1;
    }
    __syncthreads();
    const double* cx = cl_x + (size_t)b * Tcl * 6;
    const double* cu = cl_u + (size_t)b * Tcl * 2;
    if (s_ss >= 0) copy_ss_lap_block(ss, ss.lap_index(b, s_ss), cx, cu, Trec, TrackLength);
    if (s_md >= 0) copy_lap_block(model, model.lap_index(b, s_md), cx, cu, Trec);
    __syncthreads();
    if (threadIdx.x == 0) {
        int f = book_refresh(k, b, ss_laps_of(laps, b, k.numSS_it), book_windows(win, b));
        if (s_ss == -2) f |= 64;                                 // safe-set pool too small for numSS_it + 2 laps
        if (f && flags_or) flags_or[b] |= f;
        if (rep.rows) {
            if (unsafe) rep.run[b].row.flags |= LMPC_REPORT_LANE_UNSAFE;
            report_file(rep, b);
        }
        restart_record(b, cl_len, x_cur, timeStep, done, TrackLength);
    }
}

// main.py:99-110 with device bookkeeping: the record every controller just drove becomes `copies` laps of both stores.
// With lap reports the report table starts afresh, like lap_n.  With lane rules the record is judged once and every copy is filed
// with the same key.
__global__ void __launch_bounds__(256) seed_books_kernel(int batch, LapPool ss, LapPool model, LapBooks k, int copies, const double* cl_x,
                                                         const double* cl_u, int* cl_len, int Tcl, int N, double* xLin, double* uLin,
                                                         double* zt, double* OldInput, int* timeStep, int* hasPred, int* done,
                                                         Tracks trk, int lmpc, Shapes shp, SsLaps laps, LapReports rep, LapWindows win,
                                                         LaneRules lane) {
    const int b = blockIdx.x;
    if (b >= batch) return;
    __shared__ int s_ss, s_md;
    const int Trec = cl_len[b];
    const double TrackLength = trk.of(b).TrackLength;
    const double* cx = cl_x + (size_t)b * Tcl * 6;
    const double* cu = cl_u + (size_t)b * Tcl * 2;
    if (threadIdx.x == 0) {                                      // fresh books
        for (int s = 0; s < k.ss_cap; ++s) { k.ss_lap[(size_t)b * k.ss_cap + s] = -1; k.ss_time[(size_t)b * k.ss_cap + s] = 0x7fffffff; }
        for (int s = 0; s < k.md_cap; ++s) { k.md_seq[(size_t)b * k.md_cap + s] = -1; k.md_time[(size_t)b * k.md_cap + s] = 0x7fffffff; }
        k.it[b] = 0; k.md_cnt[b] = 0; k.lap_n[b] = 0;
    }
    const bool unsafe = lane_unsafe_block(lane, b, cx, Trec, 6);
    __syncthreads();
    for (int c = 0; c < copies; ++c) {
        if (threadIdx.x == 0) {
            const LapWindowRec w = book_windows(win, b);
            s_ss = lmpc ? book_ss_add(k, b, lane_key(Trec, unsafe), false, ss_laps_of(laps, b, k.numSS_it), w.ss_window) : -1;
            s_md = book_md_add(k, b, Trec, w.model_window);
        }
        __syncthreads();
        if (s_ss >= 0) copy_ss_lap_block(ss, ss.lap_index(b, s_ss), cx, cu, Trec, TrackLength);
        if (s_md >= 0) copy_lap_block(model, model.lap_index(b, s_md), cx, cu, Trec);
        __syncthreads();
    }
    seed_state_block(b, N, shp, cx, cu, xLin, uLin, zt, OldInput);
    if (threadIdx.x == 0) {
        book_refresh(k, b, ss_laps_of(laps, b, k.numSS_it), book_windows(win, b)); timeStep[b] = 0; hasPred[b] = 0; cl_len[b] = 0; done[b] = 0;
        if (rep.rows) report_restart(rep, b);
    }
}

// The state of a freshly enabled report table: n = 0 and an empty running row for every controller.
__global__ void lap_reports_reset_kernel(int batch, LapReports rep) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) report_restart(rep, b);
}

// ---- pooled safe-set exchange (SURVEY §8e) -------------------------------------------------------------------------------
// meta rows of an exchanged lap: (rows incl. the addPoint overrun, lap time, global controller id, pool group)
// Pool groups (lmpc_set_pool_groups): controller b exchanges laps only within group grp[b] of G; grp == null puts every
// controller in group 0 (G = 1).  Every pool array is group-major: G blocks of kbest rows on the send side, and on the receive
// side G rankings of at most POOL_MAXSRC rows each.
constexpr int POOL_MAXK = 8;
constexpr int POOL_MAXSRC = 64;            // gathered candidates ranked per group
constexpr int POOL_MAXG = 64;              // LMPC_MAX_POOL_GROUPS
// int scratch of the exchange, sized once for POOL_MAXG groups: best instances [G][kbest], rankings [G][POOL_MAXSRC], ranked
// rows per group [G], laps filed [1], ship mask of a masked export [G]
constexpr int POOL_ORDER = POOL_MAXG * POOL_MAXK;
constexpr int POOL_COUNT = POOL_ORDER + POOL_MAXG * POOL_MAXSRC;
constexpr int POOL_TOOK = POOL_COUNT + POOL_MAXG;
constexpr int POOL_SHIP = POOL_TOOK + 1;
constexpr int POOL_SCRATCH = POOL_SHIP + POOL_MAXG;

__device__ __forceinline__ int pool_group(const int* grp, int b) { return grp ? grp[b] : 0; }

// The k fastest "latest own laps" of this rank in group blockIdx.x, ascending (lap time, controller id): the only laps of this
// rank that can be among the group's k fastest.  A latest lap takes part only once the rows it ships (at most Tpad) reach
// `min_over` rows past its finish line (rows - lap time; addPoint appends them during the next lap): an importer's safe-set
// window near the finish reaches into those rows.  One CTA per group; k rounds of block arg-min over the group's controllers.
// ship (null: every group) masks groups out of this export: a group with ship[g] == 0 chooses no controller, so
// pool_export_kernel ships its kbest rows with global id -1 and importers file nothing of it.  rules (null: none) is the lane-rule
// table: with one, a latest lap is ranked and tested by its lap time, its safe-set key without LMPC_LANE_UNSAFE_KEY.
__global__ void __launch_bounds__(1024) pool_local_best_kernel(int batch, LapPool ss, LapBooks k, int kbest, int Tpad, int min_over,
                                                               const int* grp, const int* ship, int* best_inst,
                                                               const LaneRuleRec* rules) {
    __shared__ unsigned long long red[32];
    __shared__ int taken[POOL_MAXK];
    const int g = blockIdx.x;
    if (ship && !ship[g]) {                                       // uniform over the CTA: no barrier is skipped by part of it
        if (threadIdx.x < kbest) best_inst[g * kbest + threadIdx.x] = -1;
        return;
    }
    for (int r = 0; r < kbest; ++r) {
        unsigned long long mine = ~0ull;
        for (int b = threadIdx.x; b < batch; b += blockDim.x) {
            const int sl = k.prevslot[b];
            if (sl < 0 || pool_group(grp, b) != g) continue;
            const int t = lane_lap_time(k.ss_time[(size_t)b * k.ss_cap + sl], rules != nullptr);
            if (min_over > 0 && min(ss.len[ss.lap_index(b, sl)], Tpad) - t < min_over) continue;
            bool skip = false;
            for (int j = 0; j < r; ++j) skip |= (taken[j] == b);
            if (skip) continue;
            const unsigned long long key = ((unsigned long long)(unsigned)t << 32) | (unsigned)b;
            mine = key < mine ? key : mine;
        }
        for (int o = 16; o > 0; o >>= 1) { const unsigned long long v = __shfl_xor_sync(0xffffffffu, mine, o); mine = v < mine ? v : mine; }
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mine;
        __syncthreads();
        if (threadIdx.x < 32) {
            mine = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : ~0ull;
            for (int o = 16; o > 0; o >>= 1) { const unsigned long long v = __shfl_xor_sync(0xffffffffu, mine, o); mine = v < mine ? v : mine; }
            if (threadIdx.x == 0) { taken[r] = (mine == ~0ull) ? -1 : (int)(mine & 0xffffffffu); best_inst[g * kbest + r] = taken[r]; }
        }
        __syncthreads();
    }
}

// Pack the latest own lap of the chosen controllers into exchange rows rows[G][kbest][Tpad][XR_COLS], meta[G][kbest][4].
// One CTA per row r = g * kbest + j.  With a lane-rule table (rules, null: none) meta[.,1] is the lap time, the safe-set key
// without LMPC_LANE_UNSAFE_KEY.
__global__ void __launch_bounds__(256) pool_export_kernel(LapPool ss, LapBooks k, const int* best_inst, int kbest, int Tpad,
                                                          long long gid_base, double* rows, int* meta, const LaneRuleRec* rules) {
    const int r = blockIdx.x;
    const int b = best_inst[r];
    const int sl = b < 0 ? -1 : k.prevslot[b];
    const size_t lap = ss.lap_index(b < 0 ? 0 : b, sl < 0 ? 0 : sl);
    const int T = sl < 0 ? 0 : min(ss.len[lap], Tpad);
    pack_lap_row_block(ss, lap, T, Tpad, rows + (size_t)r * Tpad * XR_COLS);
    if (threadIdx.x == 0) {
        meta[r * 4 + 0] = T;
        meta[r * 4 + 1] = sl < 0 ? 0x7fffffff : lane_lap_time(k.ss_time[(size_t)b * k.ss_cap + sl], rules != nullptr);
        meta[r * 4 + 2] = sl < 0 ? -1 : (int)(gid_base + b);
        meta[r * 4 + 3] = r / kbest;
    }
}

// Rank the gathered laps of group blockIdx.x (meta[.,3] == g; a few per rank) by (lap time, global id): order[g][0..cnt[g]).
// Rows of another group are skipped; a row whose group lies outside [0, G) -- it came from another rank -- is ranked by no
// block.  A group holds at most POOL_MAXSRC ranked rows: slower ones are dropped (only the `share` + 1 fastest are ever read).
__global__ void __launch_bounds__(64) pool_rank_kernel(int n_src, const int* meta, int* order, int* cnt) {
    const int grp = blockIdx.x;
    __shared__ int s_n;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n_src; i += blockDim.x) {
        if (meta[i * 4 + 3] != grp) continue;
        const int t = meta[i * 4 + 1], g = meta[i * 4 + 2], len = meta[i * 4 + 0];
        int rank = 0;
        for (int j = 0; j < n_src; ++j) {
            if (meta[j * 4 + 3] != grp) continue;
            const int tj = meta[j * 4 + 1], gj = meta[j * 4 + 2], lj = meta[j * 4 + 0];
            const bool vj = gj >= 0 && lj >= 2, vi = g >= 0 && len >= 2;
            if (j != i && ((vj && !vi) || (vj == vi && (key_less(tj, gj, t, g) || (tj == t && gj == g && j < i))))) ++rank;
        }
        if (rank < POOL_MAXSRC) order[grp * POOL_MAXSRC + rank] = i;
        atomicAdd(&s_n, 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) cnt[grp] = min(s_n, POOL_MAXSRC);
}

// Every controller takes the `share` fastest laps of its own pool group that it does not own (LMPC.addTrajectory +
// PredictiveModel.addTrajectory of a lap another controller drove, main.py:117-119), filed before its own latest lap.  A lap
// is ordered by its lap time lt in both tables, as an own lap by Trec; only the rows that fit are stored.  The regression model
// takes the lap also when the safe set drops it: main.py adds every lap to both lists, and with trToUse > numSS_it a lap outside
// the numSS_it fastest can be among the trToUse shortest.  A controller with no lap of its own (it = 0) takes nothing.  The
// importer ranks a lap against its own numSS_it and its own windows, so a group may mix lap counts and windows.  With lane rules
// the importer judges the shipped rows 0 .. min(lt, rows, Tpad)-1 against its own rule and QP constants and files an unsafe lap
// with the safe-set key lt + LMPC_LANE_UNSAFE_KEY (the model takes lt).  One CTA per controller.
__global__ void __launch_bounds__(256) pool_import_kernel(int batch, LapPool ss, LapPool model, LapBooks k, int share, int Tpad,
                                                          const double* rows, const int* meta, const int* grp, const int* order,
                                                          const int* cnt, long long gid_base, int* took, int* flags_or, SsLaps laps,
                                                          LapWindows win, LaneRules lane) {
    const int b = blockIdx.x;
    if (b >= batch) return;
    __shared__ int s_ss, s_md, s_src;
    const int g = pool_group(grp, b);
    const int n = cnt[g];
    int given = 0;
    for (int o = 0; o < n && given < share; ++o) {
        const int src = order[g * POOL_MAXSRC + o];
        const int len = meta[src * 4 + 0], lt = meta[src * 4 + 1], gid = meta[src * 4 + 2];
        if (gid < 0 || len < 2) break;                            // nothing valid further down the ranking
        if ((long long)gid == gid_base + b) continue;             // its own lap
        ++given;
        const bool unsafe = lane_unsafe_block(lane, b, rows + (size_t)src * Tpad * XR_COLS, min(min(lt, len), Tpad), XR_COLS);
        if (threadIdx.x == 0) {
            s_src = src;
            const LapWindowRec w = book_windows(win, b);
            s_ss = book_ss_add(k, b, lane_key(lt, unsafe), true, ss_laps_of(laps, b, k.numSS_it), w.ss_window);
            s_md = -1;
            if (s_ss != -2 && k.it[b] > 0) s_md = book_md_add(k, b, lt, w.model_window);
        }
        __syncthreads();
        const int c_ss = s_ss, c_md = s_md;                       // private copies: thread 0 rewrites the shared ones next round
        const double* R = rows + (size_t)s_src * Tpad * XR_COLS;
        if (c_ss >= 0) file_ss_row_block(ss, ss.lap_index(b, c_ss), R, min(len, min(Tpad, ss.Tmax)), took);
        // the model stores the lap as driven: rows up to the finish line, of the Tpad rows shipped
        if (c_md >= 0) file_model_row_block(model, model.lap_index(b, c_md), R, min(min(lt, len), min(Tpad, model.Tmax)));
        __syncthreads();
        if (threadIdx.x == 0 && c_ss == -2 && flags_or) flags_or[b] |= 64;
    }
    if (threadIdx.x == 0 && given > 0) book_refresh(k, b, ss_laps_of(laps, b, k.numSS_it), book_windows(win, b));
}

// Progress of a Monte-Carlo batch in four numbers per pool group, so that the host only polls a few bytes every few steps:
// out[g][0] = min over the controllers of group g of laps driven, out[g][1] = max, out[g][2] = min closed-loop steps into the
// current lap over the group's controllers that are at lap out[g][0], out[g][3] = the group's controllers with a non-zero health
// flag.  grp == null puts every controller in group 0 (G = 1): the batch's four numbers.  A group without a controller reports
// (INT32_MAX, 0, INT32_MAX, 0), which a MIN over ranks leaves to the ranks that have some.  Each thread accumulates in registers
// while consecutive controllers of its stride stay in one group and folds into shared memory when the group changes (once per
// thread without groups).
// Retired controllers (lap budgets) are left out of out[g][0] and out[g][2] and still count in out[g][1] and out[g][3]: a group is
// not held back by a controller that will not drive again, and a group whose controllers have all retired reports the
// empty-group row (INT32_MAX, lap_max, INT32_MAX, flagged), which reads as ready for every round and as done.
__global__ void __launch_bounds__(1024) rollout_stats_kernel(int batch, LapBooks k, const int* cl_len, const int* health,
                                                             const int* grp, int G, int* out, LapBudget retire) {
    __shared__ int s_min[POOL_MAXG], s_max[POOL_MAXG], s_since[POOL_MAXG], s_flag[POOL_MAXG];
    for (int g = threadIdx.x; g < G; g += blockDim.x) { s_min[g] = 0x7fffffff; s_max[g] = 0; s_since[g] = 0x7fffffff; s_flag[g] = 0; }
    __syncthreads();
    int cur = -1, mn = 0x7fffffff, mx = 0, fl = 0;
    for (int b = threadIdx.x; b < batch; b += blockDim.x) {
        const int g = pool_group(grp, b);
        if (g != cur) {
            if (cur >= 0) { atomicMin(&s_min[cur], mn); atomicMax(&s_max[cur], mx); atomicAdd(&s_flag[cur], fl); }
            cur = g; mn = 0x7fffffff; mx = 0; fl = 0;
        }
        const int n = k.lap_n[b]; mn = retire.retired(b) ? mn : min(mn, n); mx = max(mx, n); fl += (health && health[b]) ? 1 : 0;
    }
    if (cur >= 0) { atomicMin(&s_min[cur], mn); atomicMax(&s_max[cur], mx); atomicAdd(&s_flag[cur], fl); }
    __syncthreads();
    int since = 0x7fffffff;
    cur = -1;
    for (int b = threadIdx.x; b < batch; b += blockDim.x) {
        const int g = pool_group(grp, b);
        if (g != cur) {
            if (cur >= 0) atomicMin(&s_since[cur], since);
            cur = g; since = 0x7fffffff;
        }
        if (k.lap_n[b] == s_min[g] && !retire.retired(b)) since = min(since, cl_len[b]);
    }
    if (cur >= 0) atomicMin(&s_since[cur], since);
    __syncthreads();
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        out[g * 4 + 0] = s_min[g]; out[g * 4 + 1] = s_max[g]; out[g * 4 + 2] = s_since[g]; out[g * 4 + 3] = s_flag[g];
    }
}

// ---- presentation support (SURVEY §8f rank 4: what plot.py reads) ----------------------------------------------------------
// Map.getGlobalPosition (Track.py:135-189): curvilinear (s, ey) -> inertial (X, Y) on the segment table
// [x_end, y_end, psi_end, s_start, length, curvature] (Map.PointAndTangent), row i-1 wrapping to the last row like Python's
// negative index.  ok[i] = 0 where no segment contains s (the reference raises there).
__global__ void track_global_position_kernel(const double* table, int nseg, double TrackLength, int n, const double* s_in,
                                             const double* ey_in, double* xy, int* ok) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    const double PI = 3.141592653589793;
    double s = s_in[idx];
    const double ey = ey_in[idx];
    int found = -1;
    if (s <= 64.0 * TrackLength) {
        while (s > TrackLength) s = s - TrackLength;
        for (int i = 0; i < nseg; ++i) {
            const double s0 = table[i * 6 + 3], ln = table[i * 6 + 4];
            if (s >= s0 && s < s0 + ln) { found = i; break; }
        }
    }
    if (found < 0) { xy[idx * 2] = 0.0; xy[idx * 2 + 1] = 0.0; if (ok) ok[idx] = 0; return; }
    const int i = found, im = (i == 0) ? nseg - 1 : i - 1;
    const double* ti = table + i * 6;
    const double* tm = table + im * 6;
    double x, y;
    if (ti[5] == 0.0) {
        const double rel = (s - ti[3]) / ti[4];
        x = (1 - rel) * tm[0] + rel * ti[0] + ey * cos(ti[2] + PI / 2);
        y = (1 - rel) * tm[1] + rel * ti[1] + ey * sin(ti[2] + PI / 2);
    } else {
        const double r = 1 / ti[5], ang = tm[2];
        const double d = (r >= 0) ? 1.0 : -1.0;
        const double cx = tm[0] + fabs(r) * cos(ang + d * PI / 2);
        const double cy = tm[1] + fabs(r) * sin(ang + d * PI / 2);
        const double span = (s - ti[3]) / (PI * fabs(r)) * PI;
        double an = d * PI / 2 + ang;
        if (an < -PI) an = 2 * PI + an; else if (an > PI) an = an - 2 * PI;      // wrap (Track.py:367-375)
        const double angle = -(PI - fabs(an)) * ((an >= 0) ? 1.0 : -1.0);
        x = cx + (fabs(r) - d * ey) * cos(angle + d * span);
        y = cy + (fabs(r) - d * ey) * sin(angle + d * span);
    }
    xy[idx * 2] = x; xy[idx * 2 + 1] = y;
    if (ok) ok[idx] = 1;
}

// Trace of chosen controllers during a device-resident rollout: what LMPC.unpackSolution stores per step for plot.py
// (xStoredPredTraj, SSStoredPredTraj: PC.py:377-379) plus the closed-loop point and the lap it belongs to.
struct TraceBufs {
    int n, cap, N, M;
    const int* inst;      // [n] traced controllers
    int* steps;           // [n] rows written
    double* x;            // [n][cap][6]   curvilinear state at the step
    double* g;            // [n][cap][6]   global state (SysModel.py x_glob: vx vy wz psi X Y)
    double* u;            // [n][cap][2]   applied input
    double* xPred;        // [n][cap][N+1][6]
    double* ss;           // [n][cap][6][M] selected safe-set points (SS_PointSelectedTot)
    int* lap;             // [n][cap]      laps the controller had driven before this step
};
__global__ void trace_step_kernel(TraceBufs t, const double* x, const double* xg, const double* uPred, long long u_stride,
                                  const double* xPred, const double* SS_sel, const int* lap_n, LapBudget retire) {
    const int tr = blockIdx.x;
    if (tr >= t.n) return;
    const int b = t.inst[tr];
    if (retire.retired(b)) return;            // a retired controller writes no trace row
    const int row = t.steps[tr];
    if (row >= t.cap) return;
    const size_t o = (size_t)tr * t.cap + row;
    for (int e = threadIdx.x; e < 6; e += blockDim.x) { t.x[o * 6 + e] = x[(size_t)b * 6 + e]; t.g[o * 6 + e] = xg[(size_t)b * 6 + e]; }
    for (int e = threadIdx.x; e < 2; e += blockDim.x) t.u[o * 2 + e] = uPred[(size_t)b * u_stride + e];
    const int np = (t.N + 1) * 6;
    for (int e = threadIdx.x; e < np; e += blockDim.x) t.xPred[o * np + e] = xPred[(size_t)b * np + e];
    if (t.M > 0 && SS_sel)                    // a step without a safe set (modes 0 and 2) selected no points: the row's ss stays unwritten
        for (int e = threadIdx.x; e < 6 * t.M; e += blockDim.x) t.ss[o * 6 * t.M + e] = SS_sel[(size_t)b * 6 * t.M + e];
    __syncthreads();
    if (threadIdx.x == 0) { t.lap[o] = lap_n ? lap_n[b] : 0; t.steps[tr] = row + 1; }
}

}  // namespace lmpc
