// Test shim: the essential solver's device arithmetic (openvslam_b200/csrc/essential_math.cuh) compiled for the host, so that
// tests/test_essential_solver_oracle.py can compare it with the oracle (oracle/essential_solver_oracle.c) without a GPU.
// Built by that test with g++ -ffp-contract=off (the oracle is built the same way).
#include "../../openvslam_b200/csrc/essential_math.cuh"

extern "C" {
void esc_sample8(uint64_t seed, int k, int n, int* idx) { ovs::ransac_sample<8>(seed, k, n, idx); }
// the eight-point E_21 on n matches (idx may be null) with the sequential fixed-order sums
void esc_compute_E(int n, const double* b1, const double* b2, const int* idx, double* E) {
    const ovs::EssPairs P{b1, b2, nullptr};
    ovs::essential_from_pairs(P, idx, ovs::PnpSeqSum{n}, E);
}
// the same with the bearings indexed through a pair list (pairs[2 m], pairs[2 m + 1]), as the composed matcher reads them
void esc_compute_E_pairs(int n, const double* b1, const double* b2, const int* pairs, double* E) {
    const ovs::EssPairs P{b1, b2, pairs};
    ovs::essential_from_pairs(P, nullptr, ovs::PnpSeqSum{n}, E);
}
int esc_check_inliers(const double* E, int n, const double* b1, const double* b2, unsigned char* flags, double* score) {
    const ovs::EssPairs P{b1, b2, nullptr};
    return ovs::essential_score_seq(E, P, n, flags, score);
}
void esc_jacobi9(const double* A_in, double* evals, double* V) {
    double A[81];
    for (int k = 0; k < 81; ++k) A[k] = A_in[k];
    ovs::jacobi_sym<9>(A, V);
    for (int k = 0; k < 9; ++k) evals[k] = A[10 * k];
}
}
