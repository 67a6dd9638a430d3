// racinglmpc_b200/csrc/snapshot.cuh — controller snapshots: one byte record per controller (lmpc_snapshot_*, DESIGN.md
// "Controller snapshots").
//
// Every per-controller buffer of the store and the rollout is [B][...], so one controller's part of a buffer is one contiguous
// range: a section of the record is (handle buffer, bytes per controller).  One copy kernel serves both directions; a table of
// sections travels as a kernel argument and a grid over (chunk of a section, record) moves the widest words both sides allow
// (16 B for every large section) with coalesced loads and stores.  Records are outside input, so before an unpack one check
// kernel validates every record against the destination: header, track row, and every field a kernel later uses as an index or
// a bound.
#pragma once
#include "lapbooks.cuh"

namespace lmpc {

// Section slots of the record, in the order of lmpc_snapshot_header.sect_off (the Python decoder names them in the same order)
enum SnapSection {
    SN_SS_X, SN_SS_U, SN_SS_Q, SN_SS_LEN, SN_MD_X, SN_MD_U, SN_MD_LEN,
    SN_SS_TIME, SN_SS_LAP, SN_IT, SN_MD_TIME, SN_MD_SEQ, SN_MD_CNT, SN_LAP_HIST, SN_LAP_N, SN_SEL, SN_ISPREV, SN_PREVSLOT, SN_USED,
    SN_XLIN, SN_ULIN, SN_ZT, SN_OLDINPUT, SN_XPREDPREV, SN_TIMESTEP, SN_HASPRED,
    SN_WARM, SN_WARM_VALID,
    SN_RX, SN_RG, SN_CLX, SN_CLU, SN_CLLEN, SN_DONE, SN_HEALTH_FLAGS, SN_HEALTH_UNSOLVED, SN_ABC_LTI,
    SN_LAP_REPORTS, SN_LAP_RUN,          // lmpc_rollout_enable_lap_reports: absent (0 bytes) without reports
    SN_LANE_MARGIN,                      // lmpc_set_lane_margins: absent (0 bytes) without a table
    SN_COUNT,
    // pack-only entries of the copy table: the header (up to the track row) and the controller's track row
    SN_HEADER = SN_COUNT, SN_TRACK, SN_TABLE
};
static_assert(SN_COUNT <= LMPC_SNAPSHOT_SECTIONS, "the header has a slot for every section");

struct SnapSect {
    char* base;           // handle buffer: controller b at base + b * stride (stride 0: the same bytes for every controller)
    const int* idx;       // non-null: controller b reads row idx[b] instead of row b (the track table)
    long long stride;     // bytes between controllers in the handle buffer
    int bytes;            // bytes per controller (0: absent)
    int rec_off;          // offset in the record, 16-byte aligned
    int word;             // 16, 8 or 4: the widest access that divides bytes, stride and rec_off
    int pack_only;        // written by pack, never restored (header, track row)
};

constexpr int SNAP_MAXCHUNK = 224;
struct SnapTable {
    SnapSect s[SN_TABLE];
    int chunk_bytes;                          // a multiple of 16
    int nchunk;
    unsigned short chunk_sect[SNAP_MAXCHUNK]; // chunk c moves bytes [chunk_no * chunk_bytes, + chunk_bytes) of section chunk_sect
    unsigned short chunk_no[SNAP_MAXCHUNK];
};

template <typename W>
__device__ __forceinline__ void snap_copy_words(const char* src, char* dst, int n) {
    const W* s = reinterpret_cast<const W*>(src);
    W* d = reinterpret_cast<W*>(dst);
    for (int e = threadIdx.x; e < n / (int)sizeof(W); e += blockDim.x) d[e] = s[e];
}

// Pack (unpack == 0): record i <- controller inst[i].  Unpack: controller inst[i] <- record rec_of[i].  Grid (n, nchunk).
__global__ void __launch_bounds__(256) snapshot_copy_kernel(const __grid_constant__ SnapTable t, int unpack, const int* inst,
                                                            const int* rec_of, char* rec, long long rec_bytes) {
    const int i = blockIdx.x, c = blockIdx.y;
    const SnapSect& s = t.s[t.chunk_sect[c]];
    if (unpack && s.pack_only) return;
    const long long lo = (long long)t.chunk_no[c] * t.chunk_bytes;
    const int n = (int)min((long long)s.bytes - lo, (long long)t.chunk_bytes);
    const int b = inst[i];
    char* hp = s.base + (long long)(s.idx ? s.idx[b] : b) * s.stride + lo;
    char* rp = rec + (long long)(unpack ? rec_of[i] : i) * rec_bytes + s.rec_off + lo;
    const char* src = unpack ? rp : hp;
    char* dst = unpack ? hp : rp;
    if (s.word == 16) snap_copy_words<uint4>(src, dst, n);
    else if (s.word == 8) snap_copy_words<unsigned long long>(src, dst, n);
    else snap_copy_words<unsigned int>(src, dst, n);
    // a record is deterministic: pack zeroes the padding that rounds the section up to 16 bytes (at most three words)
    const int pad = ((s.bytes + 15) & ~15) - s.bytes;
    if (!unpack && lo + n == s.bytes && (int)threadIdx.x < pad / 4) reinterpret_cast<unsigned int*>(rp + n)[threadIdx.x] = 0u;
}

// Field codes of the check kernel: header word w < 16 is code w, the section table 16, then the fields below (names in
// lmpc_b200.cu, snap_field_name)
enum SnapField {
    SF_WARM_MODE = 14, SF_SECTIONS = 16, SF_TRACK, SF_SS_LEN, SF_MD_LEN, SF_IT, SF_SS_LAP, SF_MD_CNT, SF_MD_SEQ, SF_LAP_N, SF_SEL,
    SF_ISPREV, SF_PREVSLOT, SF_USED, SF_TIMESTEP, SF_HASPRED, SF_WARM_VALID, SF_CLLEN, SF_DONE, SF_LAP_REPORTS, SF_LAP_REPORT_N,
    SF_LANE_KEY, SF_LANE_MARGIN_LAYOUT, SF_LANE_MARGIN, SF_NFIELD
};
constexpr int SNAP_HDR_WORDS = 16 + 2 * LMPC_SNAPSHOT_SECTIONS;   // int words of the header before the track row

struct SnapCheckArgs {
    const int* hdr;       // [SNAP_HDR_WORDS] the header this handle would write (warm_mode word not compared)
    int rec_off[SN_COUNT];
    Tracks trk;
    int ss_cap, md_cap, numSS_it, trToUse, Tmax, Tcl, warm_mode;
    Table<LaneRuleRec> lane;   // lane rules (lmpc_set_lane_rules): only a controller whose rule is on may hold a lane-unsafe key
    Table<LaneMarginRec> margin;   // lane margins (lmpc_set_lane_margins): a margin is finite, >= 0 and, under mode 2, in [margin0, margin_max]
};

__device__ __forceinline__ const int* snap_ints(const char* R, const SnapCheckArgs& a, int sect) {
    return reinterpret_cast<const int*>(R + a.rec_off[sect]);
}

// One thread per restore i (record rec_of[i] into controller inst[i]): out[0] = min over failures of i * 64 + field code,
// out[1] / out[2] = min / max warm_mode over the records that carry one (!= -1).
__global__ void __launch_bounds__(128) snapshot_check_kernel(const SnapCheckArgs a, int n, const int* inst, const int* rec_of,
                                                             const char* rec, long long rec_bytes, int* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const char* R = rec + (long long)rec_of[i] * rec_bytes;
    const int* H = reinterpret_cast<const int*>(R);
    int f = SF_NFIELD;
    for (int j = 0; j < SNAP_HDR_WORDS && f == SF_NFIELD; ++j) {
        const int w = j < 2 ? j : j < 15 ? j + 1 : j == 15 ? 2 : j;     // magic, version, the layout ints, then the sizes
        if (w != SF_WARM_MODE && H[w] != a.hdr[w]) f = w < SF_SECTIONS ? w : SF_SECTIONS;
    }
    // a record with or without reports, or with another report capacity, differs in its size too: name the reports instead
    for (int s = SN_LAP_REPORTS; f >= 2 && f != SF_NFIELD && s <= SN_LAP_RUN; ++s)
        if (H[16 + LMPC_SNAPSHOT_SECTIONS + s] != a.hdr[16 + LMPC_SNAPSHOT_SECTIONS + s]) f = SF_LAP_REPORTS;
    // so does a record with or without a lane margin
    if (f >= 2 && f != SF_NFIELD && f != SF_LAP_REPORTS &&
        H[16 + LMPC_SNAPSHOT_SECTIONS + SN_LANE_MARGIN] != a.hdr[16 + LMPC_SNAPSHOT_SECTIONS + SN_LANE_MARGIN])
        f = SF_LANE_MARGIN_LAYOUT;
    if (f == SF_NFIELD) {      // the layout is this handle's: the sections lie where this handle puts them
        // the circuit, bit for bit: nseg, its nseg rows and TrackLength (padding and unused rows are not part of it)
        const TrackRec& tr = *reinterpret_cast<const TrackRec*>(R + SNAP_HDR_WORDS * 4);
        const TrackRec& mine = a.trk.of(inst[i]);
        if (tr.nseg != mine.nseg || __double_as_longlong(tr.TrackLength) != __double_as_longlong(mine.TrackLength)) f = SF_TRACK;
        for (int k = 0; f == SF_NFIELD && k < mine.nseg * 3; ++k)
            if (__double_as_longlong(tr.seg[k]) != __double_as_longlong(mine.seg[k])) f = SF_TRACK;
    }
    const int mode = H[SF_WARM_MODE];
    if (f == SF_NFIELD && (mode < -1 || mode > 1 || (a.warm_mode >= 0 && mode >= 0 && mode != a.warm_mode))) f = SF_WARM_MODE;
#define BAD(cond, code) if (f == SF_NFIELD && (cond)) f = code
    if (f == SF_NFIELD) {
        const int it = snap_ints(R, a, SN_IT)[0], md_cnt = snap_ints(R, a, SN_MD_CNT)[0];
        BAD(it < 0, SF_IT);
        BAD(md_cnt < 0, SF_MD_CNT);
        for (int s = 0; s < a.ss_cap; ++s) {
            const int len = snap_ints(R, a, SN_SS_LEN)[s], ln = snap_ints(R, a, SN_SS_LAP)[s];
            BAD(len < 0 || len > a.Tmax, SF_SS_LEN);
            BAD(ln < -1 || ln >= it, SF_SS_LAP);
            BAD(ln >= 0 && snap_ints(R, a, SN_SS_TIME)[s] >= LMPC_LANE_UNSAFE_KEY && !(a.lane.tab && a.lane.of(inst[i]).mode == 1),
                SF_LANE_KEY);
        }
        for (int s = 0; s < a.md_cap; ++s) {
            const int len = snap_ints(R, a, SN_MD_LEN)[s], sq = snap_ints(R, a, SN_MD_SEQ)[s];
            BAD(len < 0 || len > a.Tmax, SF_MD_LEN);
            BAD(sq < -1 || sq >= md_cnt, SF_MD_SEQ);
        }
        BAD(snap_ints(R, a, SN_LAP_N)[0] < 0, SF_LAP_N);
        for (int c = 0; c < a.numSS_it; ++c) {
            const int sl = snap_ints(R, a, SN_SEL)[c], ip = snap_ints(R, a, SN_ISPREV)[c];
            BAD(sl < 0 || sl >= a.ss_cap, SF_SEL);
            BAD(ip != 0 && ip != 1, SF_ISPREV);
        }
        const int pv = snap_ints(R, a, SN_PREVSLOT)[0];
        BAD(pv < -1 || pv >= a.ss_cap, SF_PREVSLOT);
        for (int c = 0; c < a.trToUse; ++c) {
            const int u = snap_ints(R, a, SN_USED)[c];
            BAD(u < 0 || u >= a.md_cap, SF_USED);
        }
        BAD(snap_ints(R, a, SN_TIMESTEP)[0] < 0, SF_TIMESTEP);
        const int hp = snap_ints(R, a, SN_HASPRED)[0];
        BAD(hp != 0 && hp != 1, SF_HASPRED);
        if (a.rec_off[SN_WARM_VALID] > 0) {
            const int wv = snap_ints(R, a, SN_WARM_VALID)[0];
            BAD(wv < 0 || (mode < 0 && wv != 0), SF_WARM_VALID);
        }
        if (a.Tcl > 0) {
            const int cl = snap_ints(R, a, SN_CLLEN)[0], dn = snap_ints(R, a, SN_DONE)[0];
            BAD(cl < 0 || cl > a.Tcl, SF_CLLEN);
            BAD(dn != 0 && dn != 1, SF_DONE);
        }
        if (a.rec_off[SN_LAP_RUN] > 0) BAD(reinterpret_cast<const LapRun*>(R + a.rec_off[SN_LAP_RUN])->n < 0, SF_LAP_REPORT_N);
        if (a.rec_off[SN_LANE_MARGIN] > 0) {
            const double m = *reinterpret_cast<const double*>(R + a.rec_off[SN_LANE_MARGIN]);
            const LaneMarginRec& r = a.margin.of(inst[i]);
            BAD(!(isfinite(m) && m >= 0.0) || (r.mode == 2 && (m < r.margin0 || m > r.margin_max)), SF_LANE_MARGIN);
        }
    }
#undef BAD
    if (f != SF_NFIELD) atomicMin(&out[0], i * 64 + f);
    else if (mode >= 0) { atomicMin(&out[1], mode); atomicMax(&out[2], mode); }
}

}  // namespace lmpc
