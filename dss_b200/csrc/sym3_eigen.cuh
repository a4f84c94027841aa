// sym3_eigen.cuh -- the float64 eigen-solve of a symmetric 3x3 matrix shared by local_frames.cu and normals.cu: a
// fixed number of cyclic Jacobi sweeps, then the eigenpairs in ascending order.  Every row takes the same instruction
// path up to the rotation guards, so the result does not depend on how fast a solver converges.
#pragma once

namespace dss {

constexpr int SYM3_SWEEPS = 6;          // cyclic Jacobi sweeps: 3x3 converges quadratically, 4 reach float64 on any input
constexpr double SYM3_DEGENERATE = 0x1p-40;   // two eigenvalues closer than this times the largest count as equal

// one Jacobi rotation of the symmetric A (upper triangle used) in the (p, q) plane; V accumulates the eigenvectors
// (columns)
template <int p, int q>
__device__ __forceinline__ void jacobi_rotate(double (&A)[3][3], double (&V)[3][3]) {
    const double apq = A[p][q];
    if (apq == 0.0) return;
    constexpr int r = 3 - p - q;
    const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
    // t = sgn(theta) / (|theta| + sqrt(theta^2 + 1)), the smaller root; theta^2 overflowing gives t = 0 (no rotation)
    const double t = copysign(1.0, theta) / (fabs(theta) + sqrt(fma(theta, theta, 1.0)));
    const double c = rsqrt(fma(t, t, 1.0)), s = t * c;
    const double arp = A[r < p ? r : p][r < p ? p : r], arq = A[r < q ? r : q][r < q ? q : r];
    A[p][p] -= t * apq;
    A[q][q] += t * apq;
    A[p][q] = 0.0;
    A[r < p ? r : p][r < p ? p : r] = c * arp - s * arq;
    A[r < q ? r : q][r < q ? q : r] = s * arp + c * arq;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double vp = V[k][p], vq = V[k][q];
        V[k][p] = c * vp - s * vq;
        V[k][q] = s * vp + c * vq;
    }
}

__device__ __forceinline__ void normalize3d(double &x, double &y, double &z) {
    const double il = rsqrt(x * x + y * y + z * z);
    x *= il, y *= il, z *= il;
}

// Eigenpairs of the symmetric A (upper triangle used; overwritten): l0 <= l1 <= l2 and the unit eigenvectors f0, f1,
// f2, by SYM3_SWEEPS cyclic sweeps and a fixed three-comparator network (ties keep the column order).
__device__ __forceinline__ void sym3_eigen(double (&A)[3][3], double &l0, double &l1, double &l2, double (&f0)[3],
                                           double (&f1)[3], double (&f2)[3]) {
    double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
#pragma unroll 1
    for (int sweep = 0; sweep < SYM3_SWEEPS; ++sweep) {
        jacobi_rotate<0, 1>(A, V);
        jacobi_rotate<0, 2>(A, V);
        jacobi_rotate<1, 2>(A, V);
    }
    l0 = A[0][0], l1 = A[1][1], l2 = A[2][2];
#pragma unroll
    for (int e = 0; e < 3; ++e) f0[e] = V[e][0], f1[e] = V[e][1], f2[e] = V[e][2];
    auto cswap = [](double &la, double (&fa)[3], double &lb, double (&fb)[3]) {
        if (lb < la) {
            const double t = la;
            la = lb, lb = t;
#pragma unroll
            for (int e = 0; e < 3; ++e) {
                const double x = fa[e];
                fa[e] = fb[e], fb[e] = x;
            }
        }
    };
    cswap(l0, f0, l1, f1);
    cswap(l1, f1, l2, f2);
    cswap(l0, f0, l1, f1);
}

// The degenerate rules: where the two smallest eigenvalues agree (collinear points), f1 = normalize(f2 x e_k), e_k the
// axis of the smallest |f2_k| (the first such axis); where all three agree (a cluster of duplicates, lambda = 0), first
// f2 = e_x, so that f1 = e_z.
__device__ __forceinline__ void sym3_fix_degenerate(double l0, double l1, double l2, double (&f1)[3], double (&f2)[3]) {
    if (l2 - l0 <= SYM3_DEGENERATE * fabs(l2)) {
        // isotropic (all lambda equal, e.g. 0 for duplicates): any frame; take the axes
        f2[0] = 1.0, f2[1] = 0.0, f2[2] = 0.0;
    }
    if (l1 - l0 <= SYM3_DEGENERATE * fabs(l2)) {
        // the two smallest agree: f1 = normalize(f2 x e_k), e_k the axis of the smallest |f2_k|
        const double ax = fabs(f2[0]), ay = fabs(f2[1]), az = fabs(f2[2]);
        const int k = (ax <= ay && ax <= az) ? 0 : (ay <= az ? 1 : 2);
        // f2 x e_k
        f1[0] = k == 0 ? 0.0 : (k == 1 ? -f2[2] : f2[1]);
        f1[1] = k == 0 ? f2[2] : (k == 1 ? 0.0 : -f2[0]);
        f1[2] = k == 0 ? -f2[1] : (k == 1 ? f2[0] : 0.0);
        normalize3d(f1[0], f1[1], f1[2]);
    }
}

}  // namespace dss
