// Test shim: the pose graph's device arithmetic (openvslam_b200/csrc/sim3_math.cuh) compiled for the host, so that
// tests/test_graph_oracle.py can compare it with the oracle (oracle/graph_oracle.c) without a GPU.
// Built by that test with g++ -ffp-contract=off (the oracle is built the same way).
#include "../../openvslam_b200/csrc/sim3_math.cuh"

extern "C" {
void gc_sim3_log(const double* S, double* xi) { ovs::sim3_log(S, xi); }
void gc_sim3_phi7(const double* A, double* F) { ovs::sim3_phi7(A, F); }
void gc_graph_edge(const double* S_ji, const double* S_i, const double* S_j, double* e, double* J) { ovs::graph_edge(S_ji, S_i, S_j, e, J); }
}
