// The symmetric 3x3 eigen-solver shared by the geometric features (geometry.cu) and the superpoint features
// (sp_graph.cu): a cyclic Jacobi method in fp64.
#pragma once

namespace spg {

// one Jacobi rotation zeroing A[p][q] (A symmetric, V accumulates the eigenvectors as columns)
__device__ __forceinline__ void geo_jacobi_rot(double A[3][3], double V[3][3], int p, int q) {
    const double apq = A[p][q];
    if (apq == 0.0) return;
    const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
    const double t = fabs(theta) > 1e150 ? 0.5 / theta
                                         : (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
    const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
#pragma unroll
    for (int r = 0; r < 3; ++r) {  // A <- A J
        const double arp = A[r][p], arq = A[r][q];
        A[r][p] = cs * arp - sn * arq;
        A[r][q] = sn * arp + cs * arq;
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {  // A <- J^T A
        const double apr = A[p][r], aqr = A[q][r];
        A[p][r] = cs * apr - sn * aqr;
        A[q][r] = sn * apr + cs * aqr;
    }
    A[p][q] = A[q][p] = 0.0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double vrp = V[r][p], vrq = V[r][q];
        V[r][p] = cs * vrp - sn * vrq;
        V[r][q] = sn * vrp + cs * vrq;
    }
}

// cyclic Jacobi on A (overwritten; its diagonal ends up holding the eigenvalues), V = I on entry: quadratic
// convergence, 3x3 reaches fp64 round-off well within 8 sweeps
__device__ __forceinline__ void geo_jacobi(double A[3][3], double V[3][3]) {
    for (int sweep = 0; sweep < 8; ++sweep) {
        const double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
        const double diag = fabs(A[0][0]) + fabs(A[1][1]) + fabs(A[2][2]);
        if (off <= 1e-18 * diag || off == 0.0) break;
        geo_jacobi_rot(A, V, 0, 1);
        geo_jacobi_rot(A, V, 0, 2);
        geo_jacobi_rot(A, V, 1, 2);
    }
}

// puts the larger eigenvalue (and its vector) first
__device__ __forceinline__ void geo_order(double e[3], double v[3][3], int a, int b) {
    const bool sw = e[b] > e[a];
    const double ea = e[a], eb = e[b];
    e[a] = sw ? eb : ea;
    e[b] = sw ? ea : eb;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double va = v[a][r], vb = v[b][r];
        v[a][r] = sw ? vb : va;
        v[b][r] = sw ? va : vb;
    }
}

}  // namespace spg
