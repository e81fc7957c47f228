// MultiQueryPlanner::iterativePlan's per-query bookkeeping (host/iterative_rounds.hpp), driven by scripted round
// results for tests/test_iterative_rounds_cpu.py.
#include "../motion_primitive_library_b200/host/iterative_rounds.hpp"

// Runs one query through rounds of (planned[r], cost[r]) until it stops (at most n rounds); writes the iterations,
// the return value and the rounds it took.
extern "C" void ir_run(const int *planned, const double *cost, int n, int max_num, int *iterations, int *ok,
                       int *rounds) {
  MPL::IterativeQuery s = MPL::iterative_begin(max_num);
  int r = 0;
  while (s.running && r < n) {
    MPL::iterative_round(s, planned[r] != 0, cost[r], max_num);
    r++;
  }
  *iterations = s.iterations;
  *ok = s.ok ? 1 : 0;
  *rounds = r;
}
