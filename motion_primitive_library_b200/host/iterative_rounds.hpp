// iterative_rounds.hpp — the per-query bookkeeping of MapPlanner::iterativePlan (map_planner.cpp:413-430), which
// MultiQueryPlanner::iterativePlan applies to every query of a batch after each round.  Its own header so that the
// CPU test (tests/test_iterative_rounds_cpu.py) can drive it with scripted round results.
#pragma once

namespace MPL {

struct IterativeQuery {
  double prev_cost = 0;  // prev_traj_cost starts at 0, so a first plan of cost 0 ends the loop
  int iterations = 0;    // plan() calls made (MapPlanner::iterations())
  bool ok = true;        // what iterativePlan returns
  bool running = true;   // plans again in the next round
};

/// A query before its first round: max_num <= 0 makes no plan() call and returns true.
inline IterativeQuery iterative_begin(int max_num) {
  IterativeQuery s;
  s.running = max_num > 0;
  return s;
}

/// After one plan() of the query: a failed plan ends the loop returning false, a cost equal (==) to the previous one
/// ends it returning true, and so does reaching max_num plan() calls.
inline void iterative_round(IterativeQuery &s, bool planned, double cost, int max_num) {
  s.iterations++;
  if (!planned) {
    s.ok = false;
    s.running = false;
    return;
  }
  if (s.prev_cost == cost) {
    s.running = false;
    return;
  }
  s.prev_cost = cost;
  s.running = s.iterations < max_num;
}

}  // namespace MPL
