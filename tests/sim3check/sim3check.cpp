// Test shim: the transform optimiser's device arithmetic (openvslam_b200/csrc/sim3_math.cuh) compiled for the host, so that
// tests/test_transform_oracle.py can compare it with the oracle (oracle/sim3_oracle.c) without a GPU.
// Built by that test with g++ -ffp-contract=off (the oracle is built the same way).
#include "../../openvslam_b200/csrc/sim3_math.cuh"

extern "C" {
void sc_sim3_exp(const double* u, double* S) { ovs::sim3_exp(u, S); }
void sc_sim3_oplus(const double* S, const double* u, int fix_scale, double* out) { ovs::sim3_oplus(S, u, fix_scale != 0, out); }
void sc_edge_forward(const ovs::CameraD* cam, const double* S, const double* pc2, const double* obs, double* e, double* J) {
    ovs::sim3_edge_forward(*cam, S, pc2, obs, e, J);
}
void sc_edge_backward(const ovs::CameraD* cam, const double* S, const double* pc1, const double* obs, double* e, double* J) {
    ovs::sim3_edge_backward(*cam, S, pc1, obs, e, J);
}
int sc_solve7(const double* Hs, double lambda, const double* b, double* x) { return ovs::solve7(Hs, lambda, b, x) ? 1 : 0; }
}
