// racinglmpc_b200/csrc/lap_schedule.cuh — lap schedules of the device-resident closed loop (lmpc_rollout_set_lap_schedule).
//
// A schedule replaces controller b's row of a plant-side table (vehicles, process noise, measurement noise) by the row of the lap
// it drives: rows[b][min(lap_n[b], L - 1)], lap_n being the laps handed over since the seeding (the lap books).  Like the lap
// budget it is derived from the lap count and never stored per step, so a restored snapshot resumes at its entry.  A null schedule
// (the PID lap, a handle without one for this table) reads the table's own index.
#pragma once

namespace lmpc {

struct LapSchedule {
    const int* rows;      // [B][L] row of the table per lap, or nullptr: the table's own index
    int L;
    const int* lap_n;     // [B] laps handed over so far (the lap books)
    template <typename T>
    __device__ __forceinline__ const T& of(const Table<T>& t, int b) const {
        if (!rows) return t.of(b);
        return t.tab[rows[(size_t)b * L + min(lap_n[b], L - 1)]];
    }
    // the row of lap lap_n[b] - back (back 0 or 1: the observer's model prior looks at the step before a hand-over)
    template <typename T>
    __device__ __forceinline__ const T& of_before(const Table<T>& t, int b, int back) const {
        if (!rows) return t.of(b);
        return t.tab[rows[(size_t)b * L + min(max(lap_n[b] - back, 0), L - 1)]];
    }
};

}  // namespace lmpc
