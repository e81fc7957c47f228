// traj_rows.hpp — the row layouts in which the C entry points return trajectory samples and waypoints, for any
// command or waypoint type with pos / vel / acc / jrk (Dim each), yaw and t (and yaw_dot for a command).
// C++11 and free of the host library's types, so that code built against other trajectory classes writes the
// same rows.
#pragma once
#include <cstddef>

namespace mplh {
/// row i of rows[] := {pos, vel, acc, jrk (Dim each), yaw, yaw_dot, t} of command c (4 Dim + 3 doubles per row)
template <int Dim, class Command>
void put_command_row(double *rows, std::size_t i, const Command &c) {
  double *o = rows + i * (4 * Dim + 3);
  for (int d = 0; d < Dim; d++) { o[d] = c.pos(d); o[Dim + d] = c.vel(d); o[2 * Dim + d] = c.acc(d); o[3 * Dim + d] = c.jrk(d); }
  o[4 * Dim] = c.yaw; o[4 * Dim + 1] = c.yaw_dot; o[4 * Dim + 2] = c.t;
}

/// row i of rows[] := {pos, vel, acc, jrk (Dim each), yaw, t} of waypoint w (4 Dim + 2 doubles per row)
template <int Dim, class Point>
void put_waypoint_row(double *rows, std::size_t i, const Point &w) {
  double *o = rows + i * (4 * Dim + 2);
  for (int d = 0; d < Dim; d++) { o[d] = w.pos(d); o[Dim + d] = w.vel(d); o[2 * Dim + d] = w.acc(d); o[3 * Dim + d] = w.jrk(d); }
  o[4 * Dim] = w.yaw; o[4 * Dim + 1] = w.t;
}
}  // namespace mplh
