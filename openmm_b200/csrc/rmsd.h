// rmsd.h -- the arithmetic of RMSDForce that the device kernels (rmsd.cu) and the host probes (b200md_rmsd_probe,
// b200md_rmsd_eigen_probe) share: the quaternion matrix of the correlation matrix, its largest eigenpair, the rotation and the
// RMSD (Coutsias, Seok and Dill, "Using quaternions to calculate RMSD", J. Comput. Chem. 25:1849, 2004; the reference's
// ReferenceRMSDForce).  Plain double arithmetic, no CUDA types, so that a CPU build runs exactly the device's code.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define RMSD_HD __host__ __device__ __forceinline__
#else
#define RMSD_HD inline
#endif

// The symmetric 4x4 matrix F of the correlation matrix R[i][j] = sum_k (x_k - c)_i r_k,j (row-major, F[4 a + b]).
RMSD_HD void rmsd_quaternion_matrix(const double R[9], double F[16]) {
    const double r00 = R[0], r01 = R[1], r02 = R[2], r10 = R[3], r11 = R[4], r12 = R[5], r20 = R[6], r21 = R[7], r22 = R[8];
    F[0] = r00 + r11 + r22;  F[1] = r12 - r21;         F[2] = r20 - r02;          F[3] = r01 - r10;
    F[4] = r12 - r21;        F[5] = r00 - r11 - r22;   F[6] = r01 + r10;          F[7] = r02 + r20;
    F[8] = r20 - r02;        F[9] = r01 + r10;         F[10] = -r00 + r11 - r22;  F[11] = r12 + r21;
    F[12] = r01 - r10;       F[13] = r02 + r20;        F[14] = r12 + r21;         F[15] = -r00 - r11 + r22;
}

// Largest eigenvalue of the symmetric 4x4 matrix A (row-major) and a unit eigenvector of it, by cyclic Jacobi rotations
// (Golub and Van Loan, section 8.5) run until the off-diagonal part is zero to double precision or no rotation changes the
// matrix.  Each rotation zeroes A[p][q] with the stable choice of tan(theta) of smaller magnitude; V accumulates them.
// The sweep order is fixed, so the result is a pure function of A.  Returns the number of sweeps.
RMSD_HD int rmsd_jacobi4(const double Ain[16], double* lambda, double q[4]) {
    double A[16], V[16];
    for (int k = 0; k < 16; k++) { A[k] = Ain[k]; V[k] = (k % 5 == 0) ? 1.0 : 0.0; }
    int sweep = 0;
    for (; sweep < 64; sweep++) {
        double off = 0.0, diag = 0.0;
#pragma unroll
        for (int p = 0; p < 4; p++) {
            diag += A[5*p]*A[5*p];
            for (int r = p + 1; r < 4; r++) off += A[4*p + r]*A[4*p + r];
        }
        if (off == 0.0 || off <= 1e-36*diag) break;
        bool changed = false;
#pragma unroll
        for (int p = 0; p < 3; p++)
#pragma unroll
            for (int r = p + 1; r < 4; r++) {
                const double apq = A[4*p + r];
                if (apq == 0.0) continue;
                const double theta = (A[5*r] - A[5*p])/(2.0*apq);
                const double t = (theta >= 0.0 ? 1.0 : -1.0)/(fabs(theta) + sqrt(theta*theta + 1.0));
                const double c = 1.0/sqrt(t*t + 1.0), s = t*c;
                if (s == 0.0) continue;
                changed = true;
                for (int k = 0; k < 4; k++) {          // A <- A J (columns p and r)
                    const double akp = A[4*k + p], akr = A[4*k + r];
                    A[4*k + p] = c*akp - s*akr; A[4*k + r] = s*akp + c*akr;
                }
                for (int k = 0; k < 4; k++) {          // A <- J^T A (rows p and r)
                    const double apk = A[4*p + k], ark = A[4*r + k];
                    A[4*p + k] = c*apk - s*ark; A[4*r + k] = s*apk + c*ark;
                }
                A[4*p + r] = A[4*r + p] = 0.0;
                for (int k = 0; k < 4; k++) {          // V <- V J
                    const double vkp = V[4*k + p], vkr = V[4*k + r];
                    V[4*k + p] = c*vkp - s*vkr; V[4*k + r] = s*vkp + c*vkr;
                }
            }
        if (!changed) break;
    }
    // the largest diagonal element, then its column of V, by selects rather than a run-time index (the matrices stay in
    // registers on the device)
    double best = A[0];
    for (int k = 0; k < 4; k++) q[k] = V[4*k];
#pragma unroll
    for (int m = 1; m < 4; m++)
        if (A[5*m] > best) {
            best = A[5*m];
            for (int k = 0; k < 4; k++) q[k] = V[4*k + m];
        }
    *lambda = best;
    return sweep;
}

// The rotation matrix U of the unit quaternion q, as ReferenceRMSDForce forms it; the reference positions rotate as
// r'_j = sum_i U[i][j] r_i.
RMSD_HD void rmsd_rotation(const double q[4], double U[9]) {
    const double q00 = q[0]*q[0], q01 = q[0]*q[1], q02 = q[0]*q[2], q03 = q[0]*q[3];
    const double q11 = q[1]*q[1], q12 = q[1]*q[2], q13 = q[1]*q[3];
    const double q22 = q[2]*q[2], q23 = q[2]*q[3], q33 = q[3]*q[3];
    U[0] = q00 + q11 - q22 - q33; U[1] = 2*(q12 - q03);         U[2] = 2*(q13 + q02);
    U[3] = 2*(q12 + q03);         U[4] = q00 - q11 + q22 - q33; U[5] = 2*(q23 - q01);
    U[6] = 2*(q13 - q02);         U[7] = 2*(q23 + q01);         U[8] = q00 - q11 - q22 + q33;
}

// The RMSD of n particles from their sums: sumSq = sum |x - c|^2, refSq = sum |r|^2 (r centred), R the correlation matrix.
// Writes the rotation U and the force factor 1/(n rmsd).  As ReferenceRMSDForce, an MSD below 1e-20 is a perfect alignment:
// the RMSD and every force are 0 (factor 0), rather than the 0/0 of the gradient there.
RMSD_HD double rmsd_solve(int n, double sumSq, double refSq, const double R[9], double U[9], double* forceFactor) {
    double F[16], lambda, q[4];
    rmsd_quaternion_matrix(R, F);
    rmsd_jacobi4(F, &lambda, q);
    rmsd_rotation(q, U);
    const double msd = (sumSq + refSq - 2.0*lambda)/n;
    if (!(msd >= 1e-20)) { *forceFactor = 0.0; return 0.0; }
    const double rmsd = sqrt(msd);
    *forceFactor = 1.0/(rmsd*n);
    return rmsd;
}

// The force on a particle at x (centred: d = x - c) with centred reference position r: -(d - U^T r)/(n rmsd).
RMSD_HD void rmsd_force(const double d[3], const double r[3], const double U[9], double forceFactor, double f[3]) {
    for (int j = 0; j < 3; j++) {
        const double rot = U[j]*r[0] + U[3 + j]*r[1] + U[6 + j]*r[2];
        f[j] = -(d[j] - rot)*forceFactor;
    }
}
