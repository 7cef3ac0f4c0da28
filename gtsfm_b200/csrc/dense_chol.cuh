// Dense fp64 solve of the reduced systems of the LM solvers (global_ba.cu, translation_recovery.cu): a blocked
// right-looking Cholesky of 64 x 64 tiles, then the two triangular solves.
#pragma once
#include "common.cuh"

constexpr int CHOL_NB = 64;  // tile; the system's order np is a multiple of it

// S: device, row-major np x np, lower triangle (overwritten by L); b: the right-hand side, overwritten; y: scratch [np];
// x: the solution [np].  flag: device int, set to 1 when a pivot is not positive and finite; every kernel returns at once
// while it is set, so a failed factorisation leaves x unwritten.  Launches only (no synchronisation) on `st`.
int dense_chol_solve(b2_context* ctx, double* S, int np, double* b, double* y, double* x, int* flag, cudaStream_t st);
