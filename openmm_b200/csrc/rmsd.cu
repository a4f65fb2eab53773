// rmsd.cu -- RMSDForce: the RMSD of a particle subset from reference positions after the optimal rotation, and its forces
// (restating ReferenceRMSDForce::calculateIxn; the arithmetic lives in rmsd.h, shared with the host probes).  Three kernels on
// the bonded stream, behind the centroid kernels:
//   k_rmsd_sums:   one CTA per object: the centre c of its particles' continuous coordinates, sum |x - c|^2 and the correlation
//                  matrix R = sum (x - c) r^T with the reference positions r, which the host centred once.  All sums in double,
//                  per thread over a fixed stride, then a fixed shared-memory tree: the result does not depend on timing.
//   k_rmsd_solve:  one warp per object: the quaternion matrix of R, its largest eigenpair by cyclic Jacobi, the RMSD, the
//                  rotation and the force factor 1/(N rmsd).  Solving here rather than on
//                  the host keeps the evaluation free of host syncs, so it stays inside the captured step graph.
//   k_rmsd_forces: one thread per entry of the objects' concatenated particle lists: F = -(x - c - U^T r)/(N rmsd) through the
//                  2^32 fixed-point integer atomics.  Its thread 0 adds the RMSDs of the objects to EN_RMSD in object order, so
//                  the energy, like the forces, does not depend on timing.
// The coordinates are the continuous ones (posq plus cellOffset lattice vectors, what b200md_get_positions reports), so an RMSD
// does not jump when the list build wraps a molecule.
#include "engine.h"
#include "rmsd.h"
#include "../../include/b200md.h"
#include <algorithm>

#define RMSD_THREADS 256

__device__ __forceinline__ void rmsd_coords(const NbDev& nb, int a, double* v) {
    const float4 x = nb.posq[a];
    const int kx = nb.cellOffset[a], ky = nb.cellOffset[a + nb.npad], kz = nb.cellOffset[a + 2*nb.npad];
    v[0] = x.x + (kx*nb.box.dax + ky*(double) nb.box.bx + kz*(double) nb.box.cx);
    v[1] = x.y + (ky*nb.box.dby + kz*(double) nb.box.cy);
    v[2] = x.z + kz*nb.box.dcz;
}

__device__ __forceinline__ bool rmsd_in_groups(const RmsdDev& rd, int o) { return (rd.groupMask >> (rd.group[o] & 31)) & 1u; }

// sum of NV values per thread over the CTA, in a fixed tree; every thread gets the totals
template <int NV>
__device__ __forceinline__ void rmsd_block_sum(double (*red)[RMSD_THREADS], double* v) {
    for (int k = 0; k < NV; k++) red[k][threadIdx.x] = v[k];
    __syncthreads();
    for (int w = RMSD_THREADS/2; w > 0; w >>= 1) {
        if ((int) threadIdx.x < w)
            for (int k = 0; k < NV; k++) red[k][threadIdx.x] += red[k][threadIdx.x + w];
        __syncthreads();
    }
    for (int k = 0; k < NV; k++) v[k] = red[k][0];
    __syncthreads();
}

__global__ void __launch_bounds__(RMSD_THREADS) k_rmsd_sums(NbDev nb, RmsdDev rd) {
    const int o = blockIdx.x;
    if (!rmsd_in_groups(rd, o)) return;
    __shared__ double red[10][RMSD_THREADS];
    const int begin = rd.objStart[o], end = rd.objStart[o+1];
    double c[3] = {0.0, 0.0, 0.0};
    for (int k = begin + threadIdx.x; k < end; k += RMSD_THREADS) {
        double x[3];
        rmsd_coords(nb, rd.atoms[k], x);
        c[0] += x[0]; c[1] += x[1]; c[2] += x[2];
    }
    rmsd_block_sum<3>(red, c);
    const double inv = 1.0/(end - begin);
    c[0] *= inv; c[1] *= inv; c[2] *= inv;
    double s[10] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};       // R row-major, then sum |x - c|^2
    for (int k = begin + threadIdx.x; k < end; k += RMSD_THREADS) {
        double x[3];
        rmsd_coords(nb, rd.atoms[k], x);
        const double d[3] = {x[0] - c[0], x[1] - c[1], x[2] - c[2]};
        const double* r = rd.ref + 3*(size_t) k;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) s[3*i + j] += d[i]*r[j];
        s[9] += d[0]*d[0] + d[1]*d[1] + d[2]*d[2];
    }
    rmsd_block_sum<10>(red, s);
    if (threadIdx.x == 0) {
        double* out = rd.sums + 16*(size_t) o;
        out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = s[9];
        for (int k = 0; k < 9; k++) out[4 + k] = s[k];
    }
}

__global__ void __launch_bounds__(128) k_rmsd_solve(RmsdDev rd) {
    const int o = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
    if (o >= rd.nobj || (threadIdx.x & 31) != 0 || !rmsd_in_groups(rd, o)) return;
    const double* in = rd.sums + 16*(size_t) o;
    double U[9], factor;
    const double rmsd = rmsd_solve(rd.objStart[o+1] - rd.objStart[o], in[3], rd.refSq[o], in + 4, U, &factor);
    double* out = rd.solved + 16*(size_t) o;
    for (int k = 0; k < 9; k++) out[k] = U[k];
    out[9] = factor; out[10] = rmsd;
}

__global__ void __launch_bounds__(128) k_rmsd_forces(NbDev nb, RmsdDev rd, int wantEnergy) {
    const int t = blockIdx.x*blockDim.x + threadIdx.x;
    if (wantEnergy && t == 0) {
        double e = 0.0;
        for (int o = 0; o < rd.nobj; o++)
            if (rmsd_in_groups(rd, o)) e += rd.solved[16*(size_t) o + 10];
        if (e != 0.0) nb.energy[EN_RMSD] += e;
    }
    if (t >= rd.nentries) return;
    const int o = rd.entryObj[t];
    if (!rmsd_in_groups(rd, o)) return;
    const double* sv = rd.solved + 16*(size_t) o;
    const double* cs = rd.sums + 16*(size_t) o;
    const int a = rd.atoms[t];
    double x[3], r[3], f[3];
    rmsd_coords(nb, a, x);
    const double d[3] = {x[0] - cs[0], x[1] - cs[1], x[2] - cs[2]};
    for (int k = 0; k < 3; k++) r[k] = rd.ref[3*(size_t) t + k];
    rmsd_force(d, r, sv, sv[9], f);
    for (int k = 0; k < 3; k++)
        atomicAdd((unsigned long long*) &nb.force[a + k*nb.npad], (unsigned long long) __double2ll_rn(f[k]*B200MD_FORCE_SCALE));
}

void launch_rmsd(const NbDev& nb, const RmsdDev& rd, bool energy, cudaStream_t s) {
    launch_high(k_rmsd_sums, rd.nobj, RMSD_THREADS, 0, s, nb, rd);
    launch_high(k_rmsd_solve, (rd.nobj + 3)/4, 128, 0, s, rd);
    launch_high(k_rmsd_forces, std::max(1, (rd.nentries + 127)/128), 128, 0, s, nb, rd, energy ? 1 : 0);
}

// ---- host probes: the arithmetic of rmsd.h on the CPU, no context and no device ----
extern "C" int b200md_rmsd_probe(int n, const double* pos, const double* ref, double* rmsd, double* forces) {
    if (n < 1) return -1;
    double c[3] = {0.0, 0.0, 0.0}, cr[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < n; k++)
        for (int d = 0; d < 3; d++) { c[d] += pos[3*k + d]; cr[d] += ref[3*k + d]; }
    for (int d = 0; d < 3; d++) { c[d] /= n; cr[d] /= n; }
    double R[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, sumSq = 0.0, refSq = 0.0;
    for (int k = 0; k < n; k++) {
        const double x[3] = {pos[3*k] - c[0], pos[3*k+1] - c[1], pos[3*k+2] - c[2]};
        const double r[3] = {ref[3*k] - cr[0], ref[3*k+1] - cr[1], ref[3*k+2] - cr[2]};
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) R[3*i + j] += x[i]*r[j];
        sumSq += x[0]*x[0] + x[1]*x[1] + x[2]*x[2];
        refSq += r[0]*r[0] + r[1]*r[1] + r[2]*r[2];
    }
    double U[9], factor;
    *rmsd = rmsd_solve(n, sumSq, refSq, R, U, &factor);
    for (int k = 0; k < n; k++) {
        const double x[3] = {pos[3*k] - c[0], pos[3*k+1] - c[1], pos[3*k+2] - c[2]};
        const double r[3] = {ref[3*k] - cr[0], ref[3*k+1] - cr[1], ref[3*k+2] - cr[2]};
        rmsd_force(x, r, U, factor, forces + 3*k);
    }
    return 0;
}

extern "C" int b200md_rmsd_eigen_probe(const double* a, double* lambda, double* q) {
    return rmsd_jacobi4(a, lambda, q);
}
