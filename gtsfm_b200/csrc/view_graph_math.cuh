// fp64 cycle error of a rotation triplet, usable from host and device (the host build is the unit-test harness in
// tests/cpp/test_view_graph_math.cpp; the device build is view_graph.cu).  oracle/view_graph_ref.py states the same maths
// in NumPy.
//
// What it restates (GTSfM):
//   cycle_error_deg   compute_cyclic_rotation_error: the angle of i2Ri0.between(i2Ri1).compose(i1Ri0)
//                     utils/geometry_comparisons.py:226-241 (the angle: compute_relative_rotation_angle, :137-159)
#pragma once
#include "twoview_eval.cuh"

namespace vgraph {

// Triplet i0 < i1 < i2 with R01 = i1Ri0, R12 = i2Ri1, R02 = i2Ri0 (row-major): the angle of C = (R02^T R12) R01 in degrees.
// rotation_angle_deg(Ra, Rb) measures Ra^T Rb, so Ra = (R02^T R12)^T = R12^T R02 and Rb = R01: C is formed in the
// reference's order, and its angle by the atan2 form, accurate near 0 and near 180 degrees.
TE_HD double cycle_error_deg(const double* R01, const double* R12, const double* R02) {
  double A[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A[i * 3 + j] = R12[i] * R02[j] + R12[3 + i] * R02[3 + j] + R12[6 + i] * R02[6 + j];
  return tveval::rotation_angle_deg(A, R01);
}

}  // namespace vgraph
