// tests/host_emul/ref_qp_matrices.cpp — TEST INFRASTRUCTURE (CPU suite only): copies of the reference's condensed-model
// matrices A_qp and B_qp after a solve.
//
// Built by tests/test_prediction.py against oracle/_ref/libref_mpc.so (the reference's SolverMPC.cpp compiled unchanged
// against oracle/eigen_shim) and the same shim header, so the matrix objects are read through the shim's own class rather
// than through an assumed memory layout.  SolverMPC.cpp:26-27 defines both with external linkage (fpt = float,
// common_types.h); refshim_solve (oracle/ref_shim_probe.cpp) fills them for the record it solves.
#include <eigen3/Eigen/Dense>

extern Eigen::Matrix<float, Eigen::Dynamic, 13> A_qp;
extern Eigen::Matrix<float, Eigen::Dynamic, Eigen::Dynamic> B_qp;

extern "C" {

/* rows / columns of B_qp after the last solve (A_qp has the same rows and 13 columns) */
int refqp_rows(void) { return B_qp.rows(); }
int refqp_cols(void) { return B_qp.cols(); }

/* Aqp [rows][13], Bqp [rows][cols], row-major */
void refqp_copy(float* Aqp, float* Bqp)
{
  for (int i = 0; i < A_qp.rows(); i++)
    for (int j = 0; j < 13; j++) Aqp[i * 13 + j] = A_qp(i, j);
  for (int i = 0; i < B_qp.rows(); i++)
    for (int j = 0; j < B_qp.cols(); j++) Bqp[i * B_qp.cols() + j] = B_qp(i, j);
}

}  // extern "C"
