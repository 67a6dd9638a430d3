// racinglmpc_b200/csrc/lapbooks.cuh — the reference's per-controller lap bookkeeping, on the device.
//
// LMPC and PredictiveModel keep Python lists of laps and decide from them, once per lap, which stored laps the next lap
// uses:  LMPC.addTrajectory appends (SS, uSS, Qfun, LapTime) and `it += 1` (PC.py:418-445); addTerminalComponents takes
// np.argsort(LapTime)[:numSS_it] (PC.py:395,402) and treats lap it-1 specially (PC.py:506-512; addPoint extends it,
// PC.py:466-476); PredictiveModel.addTrajectory keeps laps sorted by length so that usedIt = [0..trToUse) are the shortest
// (PredictiveModel.py:31,35-46).  For a Monte-Carlo batch these decisions are made for thousands of controllers in the same
// step, so they live here: one thread per controller walks its (at most 8-entry) slot tables.  Only laps that can still be
// selected are stored (a lap that is not among the fastest when it arrives never becomes one: faster laps only push it
// further down), which makes the fixed-capacity pools equivalent to the reference's unbounded lists.
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

// LMPC.addTrajectory bookkeeping for a lap of `T` rows.  import == false: the controller's own new lap (lap number it).
// import == true: a lap another controller drove, filed BEFORE the controller's own latest lap (which stays lap it-1, the one
// addPoint extends): it takes lap number it-1, the own latest moves to it; it is skipped (-1) when it would not be among the
// numSS_it fastest.  Returns the slot to copy the lap into, -1 = not stored, -2 = pool too small.
__device__ inline int book_ss_add(const LapBooks& k, int b, int T, bool import) {
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
        if (rank >= k.numSS_it) return -1;                       // never selected (PC.py:395) -> not stored
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
            if (rank < k.numSS_it) continue;                     // one of the fastest: keep
            if (slot < 0 || tm[s] > vt || (tm[s] == vt && ln[s] < vn)) { slot = s; vt = tm[s]; vn = ln[s]; }
        }
        if (slot < 0) return -2;
    }
    tm[slot] = T;
    ln[slot] = lapno;
    k.it[b] = it + 1;
    return slot;
}

// PredictiveModel.addTrajectory bookkeeping for a lap of `T` rows.  Returns the slot, or -1 when the lap can never be among
// the trToUse shortest.
__device__ inline int book_md_add(const LapBooks& k, int b, int T) {
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

// What the next lap reads: the numSS_it fastest safe-set laps in argsort order, which of them is lap it-1, the slot addPoint
// extends, and usedIt of the regression model.  Returns 0, or 8 when fewer than numSS_it laps are stored (the reference
// raises IndexError at PC.py:402-403).
__device__ inline int book_refresh(const LapBooks& k, int b) {
    const int* tm = k.ss_time + (size_t)b * k.ss_cap;
    const int* ln = k.ss_lap + (size_t)b * k.ss_cap;
    const int it = k.it[b];
    int flag = 0, prev = -1, last = 0;
    for (int s = 0; s < k.ss_cap; ++s) if (ln[s] == it - 1) prev = s;
    for (int c = 0; c < k.numSS_it; ++c) {
        int best = -1;
        for (int s = 0; s < k.ss_cap; ++s) {
            if (ln[s] < 0) continue;
            int rank = 0;
            for (int j = 0; j < k.ss_cap; ++j) if (j != s && ln[j] >= 0 && key_less(tm[j], ln[j], tm[s], ln[s])) ++rank;
            if (rank == c) best = s;
        }
        if (best < 0) { flag = 8; best = last; } else last = best;
        k.sel[(size_t)b * k.numSS_it + c] = best;
        k.isprev[(size_t)b * k.numSS_it + c] = (ln[best] == it - 1) ? 1 : 0;
    }
    k.prevslot[b] = prev;
    const int* mt = k.md_time + (size_t)b * k.md_cap;
    const int* ms = k.md_seq + (size_t)b * k.md_cap;
    last = 0;
    for (int c = 0; c < k.trToUse; ++c) {
        int best = -1;
        for (int s = 0; s < k.md_cap; ++s) {
            if (ms[s] < 0) continue;
            int rank = 0;
            for (int j = 0; j < k.md_cap; ++j) if (j != s && ms[j] >= 0 && key_less(mt[j], ms[j], mt[s], ms[s])) ++rank;
            if (rank == c) best = s;
        }
        if (best < 0) best = last; else last = best;             // fewer laps than trToUse: the slowest one repeats
        k.used[(size_t)b * k.trToUse + c] = best;
    }
    return flag;
}

// Copy `T` rows of (x | u) from a closed-loop record into a pool slot; block-wide.
__device__ inline void copy_lap_block(const LapPool& pool, size_t lap, const double* cx, const double* cu, int T) {
    for (int e = threadIdx.x; e < T * 6; e += blockDim.x) pool.x[lap * pool.Tmax * 6 + e] = cx[e];
    for (int e = threadIdx.x; e < T * 2; e += blockDim.x) pool.u[lap * pool.Tmax * 2 + e] = cu[e];
    if (threadIdx.x == 0) pool.len[lap] = T;
}

// Lap hand-over of every controller whose lap just ended (done[b] != 0), bookkeeping included: main.py:113-119
// (lmpc.addTrajectory + predictiveModel.addTrajectory of the lap Simulator.sim returned), SysModel.py:50 (s -= TrackLength),
// PC.py:445 (timeStep = 0).  One CTA per controller; no host involvement.
__global__ void __launch_bounds__(256) commit_laps_books_kernel(int batch, LapPool ss, LapPool model, LapBooks k, const double* cl_x,
                                                                const double* cl_u, int* cl_len, int Tcl, double* x_cur, int* timeStep,
                                                                int* done, int* flags_or, Tracks trk, int lmpc) {
    const int b = blockIdx.x;
    if (b >= batch || !done[b]) return;
    __shared__ int s_ss, s_md;
    const int Trec = cl_len[b];
    const double TrackLength = trk.of(b).TrackLength;
    if (threadIdx.x == 0) {
        s_ss = lmpc ? book_ss_add(k, b, min(Trec, ss.Tmax), false) : -1;
        s_md = book_md_add(k, b, min(Trec, model.Tmax));
        const int n = k.lap_n[b];
        if (n < LAP_HIST) k.lap_hist[(size_t)b * LAP_HIST + n] = Trec;
        k.lap_n[b] = n + 1;
    }
    __syncthreads();
    const double* cx = cl_x + (size_t)b * Tcl * 6;
    const double* cu = cl_u + (size_t)b * Tcl * 2;
    if (s_ss >= 0) {
        const size_t lap = ss.lap_index(b, s_ss);
        copy_lap_block(ss, lap, cx, cu, min(Trec, ss.Tmax));
        __syncthreads();
        lap_cost_block(ss, lap, TrackLength);
    }
    if (s_md >= 0) copy_lap_block(model, model.lap_index(b, s_md), cx, cu, min(Trec, model.Tmax));
    __syncthreads();
    if (threadIdx.x == 0) {
        int f = book_refresh(k, b);
        if (s_ss == -2) f |= 64;                                 // safe-set pool too small for numSS_it + 2 laps
        if (f && flags_or) flags_or[b] |= f;
        cl_len[b] = 0;
        x_cur[(size_t)b * 6 + 4] -= TrackLength;
        timeStep[b] = 0;
        done[b] = 0;
    }
}

// main.py:99-110 with device bookkeeping: the record every controller just drove becomes `copies` laps of both stores.
__global__ void __launch_bounds__(256) seed_books_kernel(int batch, LapPool ss, LapPool model, LapBooks k, int copies, const double* cl_x,
                                                         const double* cl_u, int* cl_len, int Tcl, int N, double* xLin, double* uLin,
                                                         double* zt, double* OldInput, int* timeStep, int* hasPred, int* done,
                                                         Tracks trk, int lmpc) {
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
    __syncthreads();
    for (int c = 0; c < copies; ++c) {
        if (threadIdx.x == 0) {
            s_ss = lmpc ? book_ss_add(k, b, min(Trec, ss.Tmax), false) : -1;
            s_md = book_md_add(k, b, min(Trec, model.Tmax));
        }
        __syncthreads();
        if (s_ss >= 0) {
            const size_t lap = ss.lap_index(b, s_ss);
            copy_lap_block(ss, lap, cx, cu, min(Trec, ss.Tmax));
            __syncthreads();
            lap_cost_block(ss, lap, TrackLength);
        }
        if (s_md >= 0) copy_lap_block(model, model.lap_index(b, s_md), cx, cu, min(Trec, model.Tmax));
        __syncthreads();
    }
    for (int e = threadIdx.x; e < (N + 1) * 6; e += blockDim.x) xLin[(size_t)b * (N + 1) * 6 + e] = cx[6 + e];     // PC.py:432
    for (int e = threadIdx.x; e < N * 2; e += blockDim.x) uLin[(size_t)b * N * 2 + e] = cu[2 + e];                 // PC.py:433
    __syncthreads();
    if (threadIdx.x < 6) zt[(size_t)b * 6 + threadIdx.x] = (threadIdx.x == 4) ? 10.0 : 0.0;                         // PC.py:330
    if (threadIdx.x < 2) OldInput[(size_t)b * 2 + threadIdx.x] = 0.0;
    if (threadIdx.x == 0) { book_refresh(k, b); timeStep[b] = 0; hasPred[b] = 0; cl_len[b] = 0; done[b] = 0; }
}

// ---- pooled safe-set exchange (SURVEY §8e) -------------------------------------------------------------------------------
// meta rows of an exchanged lap: (rows incl. the addPoint overrun, lap time, global controller id, -)
constexpr int POOL_MAXK = 8;

// The k fastest "latest own laps" of this rank, ascending (lap time, controller id): the only laps of this rank that can be
// among the global k fastest.  One CTA; k rounds of block arg-min over the batch.
__global__ void __launch_bounds__(1024) pool_local_best_kernel(int batch, LapBooks k, int kbest, int* best_inst) {
    __shared__ unsigned long long red[32];
    __shared__ int taken[POOL_MAXK];
    for (int r = 0; r < kbest; ++r) {
        unsigned long long mine = ~0ull;
        for (int b = threadIdx.x; b < batch; b += blockDim.x) {
            const int sl = k.prevslot[b];
            if (sl < 0) continue;
            bool skip = false;
            for (int j = 0; j < r; ++j) skip |= (taken[j] == b);
            if (skip) continue;
            const unsigned long long key = ((unsigned long long)(unsigned)k.ss_time[(size_t)b * k.ss_cap + sl] << 32) | (unsigned)b;
            mine = key < mine ? key : mine;
        }
        for (int o = 16; o > 0; o >>= 1) { const unsigned long long v = __shfl_xor_sync(0xffffffffu, mine, o); mine = v < mine ? v : mine; }
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mine;
        __syncthreads();
        if (threadIdx.x < 32) {
            mine = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : ~0ull;
            for (int o = 16; o > 0; o >>= 1) { const unsigned long long v = __shfl_xor_sync(0xffffffffu, mine, o); mine = v < mine ? v : mine; }
            if (threadIdx.x == 0) { taken[r] = (mine == ~0ull) ? -1 : (int)(mine & 0xffffffffu); best_inst[r] = taken[r]; }
        }
        __syncthreads();
    }
}

// Pack the latest own lap of the chosen controllers: rows[kbest][Tpad][9] = (x 6 | u 2 | Qfun 1), meta[kbest][4].
__global__ void __launch_bounds__(256) pool_export_kernel(LapPool ss, LapBooks k, const int* best_inst, int Tpad, long long gid_base,
                                                          double* rows, int* meta) {
    const int r = blockIdx.x;
    const int b = best_inst[r];
    const int sl = b < 0 ? -1 : k.prevslot[b];
    const size_t lap = ss.lap_index(b < 0 ? 0 : b, sl < 0 ? 0 : sl);
    const int T = sl < 0 ? 0 : min(ss.len[lap], Tpad);
    const double* X = ss.x + lap * ss.Tmax * 6;
    const double* U = ss.u + lap * ss.Tmax * 2;
    const double* Q = ss.q + lap * ss.Tmax;
    for (int e = threadIdx.x; e < Tpad * 9; e += blockDim.x) {
        const int t = e / 9, j = e - t * 9;
        double v = 0.0;
        if (t < T) v = (j < 6) ? X[t * 6 + j] : (j < 8 ? U[t * 2 + (j - 6)] : Q[t]);
        rows[(size_t)r * Tpad * 9 + e] = v;
    }
    if (threadIdx.x == 0) {
        meta[r * 4 + 0] = T;
        meta[r * 4 + 1] = sl < 0 ? 0x7fffffff : k.ss_time[(size_t)b * k.ss_cap + sl];
        meta[r * 4 + 2] = sl < 0 ? -1 : (int)(gid_base + b);
        meta[r * 4 + 3] = 0;
    }
}

// Rank the gathered laps (n_src <= 64, a few per rank) by (lap time, global id): order[0..n_src).
__global__ void __launch_bounds__(64) pool_rank_kernel(int n_src, const int* meta, int* order) {
    const int i = threadIdx.x;
    if (i >= n_src) return;
    const int t = meta[i * 4 + 1], g = meta[i * 4 + 2], len = meta[i * 4 + 0];
    int rank = 0;
    for (int j = 0; j < n_src; ++j) {
        const int tj = meta[j * 4 + 1], gj = meta[j * 4 + 2], lj = meta[j * 4 + 0];
        const bool vj = gj >= 0 && lj >= 2, vi = g >= 0 && len >= 2;
        if (j != i && ((vj && !vi) || (vj == vi && (key_less(tj, gj, t, g) || (tj == t && gj == g && j < i))))) ++rank;
    }
    order[rank] = i;
}

// Every controller takes the `share` globally fastest laps it does not own (LMPC.addTrajectory + PredictiveModel.addTrajectory
// of a lap another controller drove, main.py:117-119), filed before its own latest lap.  One CTA per controller.
__global__ void __launch_bounds__(256) pool_import_kernel(int batch, LapPool ss, LapPool model, LapBooks k, int n_src, int share, int Tpad,
                                                          const double* rows, const int* meta, const int* order, long long gid_base,
                                                          int* took, int* flags_or) {
    const int b = blockIdx.x;
    if (b >= batch) return;
    __shared__ int s_ss, s_md, s_src;
    int given = 0;
    for (int o = 0; o < n_src && given < share; ++o) {
        const int src = order[o];
        const int len = meta[src * 4 + 0], lt = meta[src * 4 + 1], gid = meta[src * 4 + 2];
        if (gid < 0 || len < 2) break;                            // nothing valid further down the ranking
        if ((long long)gid == gid_base + b) continue;             // its own lap
        ++given;
        if (threadIdx.x == 0) {
            s_src = src;
            s_ss = book_ss_add(k, b, lt, true);
            s_md = -1;
            if (s_ss >= 0) s_md = book_md_add(k, b, lt);
        }
        __syncthreads();
        const int c_ss = s_ss, c_md = s_md;                       // private copies: thread 0 rewrites the shared ones next round
        const double* R = rows + (size_t)s_src * Tpad * 9;
        if (c_ss >= 0) {
            const int T = min(len, min(Tpad, ss.Tmax));
            const size_t lap = ss.lap_index(b, c_ss);
            for (int e = threadIdx.x; e < T * 9; e += blockDim.x) {
                const int t = e / 9, j = e - t * 9;
                const double v = R[e];
                if (j < 6) ss.x[(lap * ss.Tmax + t) * 6 + j] = v;
                else if (j < 8) ss.u[(lap * ss.Tmax + t) * 2 + (j - 6)] = v;
                else ss.q[lap * ss.Tmax + t] = v;
            }
            if (threadIdx.x == 0) { ss.len[lap] = T; if (took) atomicAdd(took, 1); }
        }
        if (c_md >= 0) {                                          // the model stores the lap as driven: rows up to the finish line
            const int Tm = min(lt, min(len, model.Tmax));
            const size_t lap = model.lap_index(b, c_md);
            for (int e = threadIdx.x; e < Tm * 8; e += blockDim.x) {
                const int t = e >> 3, j = e & 7;
                const double v = R[t * 9 + j];
                if (j < 6) model.x[(lap * model.Tmax + t) * 6 + j] = v;
                else model.u[(lap * model.Tmax + t) * 2 + (j - 6)] = v;
            }
            if (threadIdx.x == 0) model.len[lap] = Tm;
        }
        __syncthreads();
        if (threadIdx.x == 0 && c_ss == -2 && flags_or) flags_or[b] |= 64;
    }
    if (threadIdx.x == 0 && given > 0) book_refresh(k, b);
}

// Progress of a Monte-Carlo batch in four numbers, so that the host only polls a few bytes every few steps:
// out[0] = min over controllers of laps driven, out[1] = max, out[2] = min closed-loop steps into the current lap over the
// controllers that are at lap out[0], out[3] = controllers with a non-zero health flag.
__global__ void __launch_bounds__(1024) rollout_stats_kernel(int batch, LapBooks k, const int* cl_len, const int* health, int* out) {
    __shared__ int s_min, s_max, s_since, s_flag;
    if (threadIdx.x == 0) { s_min = 0x7fffffff; s_max = 0; s_since = 0x7fffffff; s_flag = 0; }
    __syncthreads();
    int mn = 0x7fffffff, mx = 0, fl = 0;
    for (int b = threadIdx.x; b < batch; b += blockDim.x) { const int n = k.lap_n[b]; mn = min(mn, n); mx = max(mx, n); fl += (health && health[b]) ? 1 : 0; }
    atomicMin(&s_min, mn); atomicMax(&s_max, mx); atomicAdd(&s_flag, fl);
    __syncthreads();
    int since = 0x7fffffff;
    for (int b = threadIdx.x; b < batch; b += blockDim.x) if (k.lap_n[b] == s_min) since = min(since, cl_len[b]);
    atomicMin(&s_since, since);
    __syncthreads();
    if (threadIdx.x == 0) { out[0] = s_min; out[1] = s_max; out[2] = s_since; out[3] = s_flag; }
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
                                  const double* xPred, const double* SS_sel, const int* lap_n) {
    const int tr = blockIdx.x;
    if (tr >= t.n) return;
    const int b = t.inst[tr];
    const int row = t.steps[tr];
    if (row >= t.cap) return;
    const size_t o = (size_t)tr * t.cap + row;
    for (int e = threadIdx.x; e < 6; e += blockDim.x) { t.x[o * 6 + e] = x[(size_t)b * 6 + e]; t.g[o * 6 + e] = xg[(size_t)b * 6 + e]; }
    for (int e = threadIdx.x; e < 2; e += blockDim.x) t.u[o * 2 + e] = uPred[(size_t)b * u_stride + e];
    const int np = (t.N + 1) * 6;
    for (int e = threadIdx.x; e < np; e += blockDim.x) t.xPred[o * np + e] = xPred[(size_t)b * np + e];
    if (t.M > 0)
        for (int e = threadIdx.x; e < 6 * t.M; e += blockDim.x) t.ss[o * 6 * t.M + e] = SS_sel[(size_t)b * 6 * t.M + e];
    __syncthreads();
    if (threadIdx.x == 0) { t.lap[o] = lap_n ? lap_n[b] : 0; t.steps[tr] = row + 1; }
}

}  // namespace lmpc
