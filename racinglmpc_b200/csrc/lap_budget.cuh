// racinglmpc_b200/csrc/lap_budget.cuh — lap budgets of the device-resident closed loop (lmpc_rollout_set_lap_budget).
//
// Controller b is retired once it has handed over budget[b] laps: its state stays as that hand-over left it and no kernel of the
// closed-loop step works for it.  Retired is derived from the lap count, never stored, so raising the budget revives a controller
// where it stopped, seeding (lap_n = 0) revives every controller and a restored snapshot needs nothing extra.  Every kernel that
// honours the budget asks this one helper; a null budget (the host-driven entry points, the PID lap, a handle without budgets)
// retires nobody.
#pragma once

namespace lmpc {

struct LapBudget {
    const int* budget;    // [B] laps controller b drives, or nullptr: no budget
    const int* lap_n;     // [B] laps handed over so far (the lap books)
    __device__ __forceinline__ bool retired(int b) const { return budget && lap_n[b] >= budget[b]; }
};

}  // namespace lmpc
