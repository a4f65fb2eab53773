/* oracle/md_oracle.c -- TEST INFRASTRUCTURE, not product code.
 *
 * A plain-C, double-precision CPU restatement of the reference's algorithm for the hot path
 * (NonbondedForce direct space + PME reciprocal space + exclusion correction + 1-4 exceptions, harmonic bonds /
 * angles / periodic torsions, SETTLE, Verlet / Langevin / LangevinMiddle updates).  Each function cites the
 * reference file:line it follows (pandegroup/openmm 7.6-dev, platforms/reference).
 *
 * Pinning: tests/test_oracle.py checks this file against (1) the Gromacs golden forces/energy the reference's own
 * test holds (tests/TestEwald.h:222-271, fixture tests/golden/ewald_triclinic_gromacs.json), (2) outputs of the
 * reference itself (oracle/_ref/libOpenMM.so, Reference platform) on seeded systems, committed as fixtures under
 * tests/golden/ with the script that generated them (tests/golden/make_golden.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may call into this file.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ONE_4PI_EPS0 138.93545764438198          /* SimTKOpenMMRealType.h:89 */
#define BOLTZ 0.00831446261815324        /* SimTKOpenMMRealType.h:76-80 */
#define PME_ORDER 5                      /* ReferenceLJCoulombIxn.cpp:243 */

/* box: 9 doubles, rows a, b, c in reduced lower-triangular form.  ReferenceForce::getDeltaRPeriodic
 * (ReferenceForce.cpp:90-101): subtract c, then b, then a, each by floor(x/L + 0.5). */
static void min_image(double d[3], const double* box) {
    double s = floor(d[2]/box[8] + 0.5);
    d[0] -= s*box[6]; d[1] -= s*box[7]; d[2] -= s*box[8];
    s = floor(d[1]/box[4] + 0.5);
    d[0] -= s*box[3]; d[1] -= s*box[4];
    s = floor(d[0]/box[0] + 0.5);
    d[0] -= s*box[0];
}

int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ------------------------------------------------------------------------------------------------------------
 * Direct space.  method: 0 NoCutoff, 1 CutoffNonPeriodic, 2 CutoffPeriodic, 4 PME.
 * ReferenceLJCoulombIxn::calculateEwaldIxn direct part (ReferenceLJCoulombIxn.cpp:373-460) and calculateOneIxn
 * (:573-626); pair selection as computeNeighborListVoxelHash (r <= cutoff, exclusions removed,
 * ReferenceNeighborList.cpp:221-259) -- here a plain O(N^2) double loop.
 * excl: CSR (exclStart[n+1], exclList) listing for every atom all its excluded partners.
 * forces are ACCUMULATED; returns the energy. */
double orc_direct(int n, const double* pos, const double* q, const double* sigma, const double* eps,
                  const double* box, int method, double cutoff, double alpha, double rfDielectric,
                  int useSwitch, double switchDist, const int* exclStart, const int* exclList, double* forces) {
    const int periodic = (method == 2 || method == 4);
    const int useCutoff = (method != 0);
    const double krf = useCutoff ? pow(cutoff, -3.0)*(rfDielectric-1.0)/(2.0*rfDielectric+1.0) : 0.0;   /* :79-80 */
    const double crf = useCutoff ? (1.0/cutoff)*(3.0*rfDielectric)/(2.0*rfDielectric+1.0) : 0.0;
    const double SQRT_PI = sqrt(M_PI);
    double energy = 0.0;
    int nthreads = orc_num_threads();
    double* fbuf = (double*) calloc((size_t) nthreads*3*n, sizeof(double));
#pragma omp parallel reduction(+:energy)
    {
#ifdef _OPENMP
        double* f = fbuf + (size_t) omp_get_thread_num()*3*n;
#else
        double* f = fbuf;
#endif
#pragma omp for schedule(dynamic, 16)
        for (int i = 0; i < n; i++) {
            for (int j = i+1; j < n; j++) {
                double d[3] = {pos[3*i]-pos[3*j], pos[3*i+1]-pos[3*j+1], pos[3*i+2]-pos[3*j+2]};   /* x_i - x_j */
                if (periodic) min_image(d, box);
                const double r2 = d[0]*d[0] + d[1]*d[1] + d[2]*d[2];
                if (useCutoff && r2 > cutoff*cutoff) continue;
                int excluded = 0;
                for (int e = exclStart[i]; e < exclStart[i+1]; e++) if (exclList[e] == j) { excluded = 1; break; }
                if (excluded) continue;
                const double r = sqrt(r2), invR = 1.0/r;
                double sw = 1, dsw = 0;
                if (useSwitch && r > switchDist) {
                    double t = (r-switchDist)/(cutoff-switchDist);
                    sw = 1+t*t*t*(-10+t*(15-t*6));
                    dsw = t*t*(-30+t*(60-t*30))/(cutoff-switchDist);
                }
                const double sig = 0.5*(sigma[i]+sigma[j]);
                const double ep = 4.0*sqrt(eps[i]*eps[j]);        /* (2 sqrt ei)(2 sqrt ej), ReferenceKernels.cpp:1093-1097 */
                double s2 = sig*invR; s2 *= s2;
                const double s6 = s2*s2*s2;
                const double qq = ONE_4PI_EPS0*q[i]*q[j];
                double dEdR, ec;
                if (method == 4) {
                    const double ar = alpha*r;
                    dEdR = qq*invR*invR*invR*(erfc(ar) + 2*ar*exp(-ar*ar)/SQRT_PI);
                    ec = qq*invR*erfc(ar);
                }
                else if (useCutoff) {
                    dEdR = qq*(invR - 2.0*krf*r2)*invR*invR;
                    ec = qq*(invR + krf*r2 - crf);
                }
                else {
                    dEdR = qq*invR*invR*invR;
                    ec = qq*invR;
                }
                dEdR += sw*ep*(12.0*s6 - 6.0)*s6*invR*invR;
                double elj = ep*(s6-1.0)*s6;
                if (useSwitch) { dEdR -= elj*dsw*invR; elj *= sw; }
                for (int k = 0; k < 3; k++) { f[3*i+k] += dEdR*d[k]; f[3*j+k] -= dEdR*d[k]; }
                energy += ec + elj;
            }
        }
    }
    for (int t = 0; t < nthreads; t++)
        for (int k = 0; k < 3*n; k++) forces[k] += fbuf[(size_t) t*3*n + k];
    free(fbuf);
    return energy;
}

/* Ewald self energy (ReferenceLJCoulombIxn.cpp:220-233) */
double orc_self_energy(int n, const double* q, double alpha) {
    double e = 0;
    for (int i = 0; i < n; i++) e -= ONE_4PI_EPS0*q[i]*q[i]*alpha/sqrt(M_PI);
    return e;
}

/* Exclusion correction under Ewald/PME (ReferenceLJCoulombIxn.cpp:462-523): every exception pair, no minimum image
 * unless exceptionsUsePeriodic.  Returns the energy contribution (already negative-signed). */
double orc_exclusion_correction(int nexc, const int* ei, const int* ej, const double* pos, const double* q,
                                const double* box, int periodicExceptions, double alpha, double* forces) {
    const double SQRT_PI = sqrt(M_PI);
    double energy = 0;
    for (int e = 0; e < nexc; e++) {
        const int i = ei[e], j = ej[e];
        double d[3] = {pos[3*i]-pos[3*j], pos[3*i+1]-pos[3*j+1], pos[3*i+2]-pos[3*j+2]};
        if (periodicExceptions) min_image(d, box);
        const double r = sqrt(d[0]*d[0] + d[1]*d[1] + d[2]*d[2]), invR = 1.0/r;
        const double ar = alpha*r;
        const double qq = ONE_4PI_EPS0*q[i]*q[j];
        if (erf(ar) > 1e-6) {
            const double dEdR = qq*invR*invR*invR*(erf(ar) - 2*ar*exp(-ar*ar)/SQRT_PI);
            for (int k = 0; k < 3; k++) { forces[3*i+k] -= dEdR*d[k]; forces[3*j+k] += dEdR*d[k]; }
            energy -= qq*invR*erf(ar);
        }
        else
            energy -= alpha*2.0/SQRT_PI*qq;
    }
    return energy;
}

/* 1-4 exceptions (ReferenceLJCoulomb14::calculateBondIxn, ReferenceLJCoulomb14.cpp:75-110): plain Coulomb + LJ with
 * the exception's own (chargeProd, sigma, epsilon); evaluated only if chargeProd != 0 or epsilon != 0
 * (ReferenceKernels.cpp:885-895). */
double orc_exceptions14(int nexc, const int* ei, const int* ej, const double* qq, const double* sigma, const double* eps,
                        const double* pos, double* forces) {
    double energy = 0;
    for (int e = 0; e < nexc; e++) {
        if (qq[e] == 0.0 && eps[e] == 0.0) continue;
        const int i = ei[e], j = ej[e];
        double d[3] = {pos[3*i]-pos[3*j], pos[3*i+1]-pos[3*j+1], pos[3*i+2]-pos[3*j+2]};
        const double r2 = d[0]*d[0] + d[1]*d[1] + d[2]*d[2], invR = 1.0/sqrt(r2);
        double s2 = sigma[e]*invR; s2 *= s2;
        const double s6 = s2*s2*s2;
        const double c = ONE_4PI_EPS0*qq[e];
        const double dEdR = (4.0*eps[e]*(12.0*s6 - 6.0)*s6 + c*invR)*invR*invR;
        for (int k = 0; k < 3; k++) { forces[3*i+k] += dEdR*d[k]; forces[3*j+k] -= dEdR*d[k]; }
        energy += 4.0*eps[e]*(s6-1.0)*s6 + c*invR;
    }
    return energy;
}

/* ------------------------------------------------------------------------------------------------------------
 * PME reciprocal space: pme_exec (ReferencePME.cpp:756-805) = index/fraction (:206-266), B-splines (:274-327),
 * spread (:330-405), forward FFT, convolution (:409-514), backward FFT, interpolation (:617-713).
 * The 3-D transform is a separable direct DFT (O(n^2) per line, same unnormalised convention as fftpack.cpp:
 * forward exp(-2 pi i jk/n)), adequate for the grid sizes the tests use. */
static void bspline_moduli(int n, double* mod) {       /* pme_calculate_bsplines_moduli, ReferencePME.cpp:98-193 */
    const int order = PME_ORDER;
    double data[PME_ORDER];
    double* bs = (double*) calloc((size_t) (n > order+1 ? n : order+1), sizeof(double));
    memset(data, 0, sizeof(data));
    data[0] = 1;
    for (int k = 3; k < order; k++) {
        double div = 1.0/(k-1.0);
        data[k-1] = 0;
        for (int l = 1; l < k-1; l++) data[k-l-1] = div*(l*data[k-l-2] + (k-l)*data[k-l-1]);
        data[0] = div*data[0];
    }
    double div = 1.0/(order-1);
    data[order-1] = 0;
    for (int l = 1; l < order-1; l++) data[order-l-1] = div*(l*data[order-l-2] + (order-l)*data[order-l-1]);
    data[0] = div*data[0];
    for (int i = 1; i <= order; i++) bs[i] = data[i-1];
    const int nb = (n > order+1 ? n : order+1);
    for (int i = 0; i < n; i++) {
        double sc = 0, ss = 0;
        for (int j = 0; j < n && j < nb; j++) {
            double arg = (2.0*M_PI*i*j)/n;
            sc += bs[j]*cos(arg); ss += bs[j]*sin(arg);
        }
        mod[i] = sc*sc + ss*ss;
    }
    for (int i = 0; i < n; i++)
        if (mod[i] < 1.0e-7) mod[i] = (mod[(i-1+n)%n] + mod[(i+1)%n])/2;
    free(bs);
}

static void bsplines(double dr, double* data, double* ddata) {   /* pme_update_bsplines, ReferencePME.cpp:274-327 */
    const int order = PME_ORDER;
    data[order-1] = 0; data[1] = dr; data[0] = 1-dr;
    for (int k = 3; k < order; k++) {
        double div = 1.0/(k-1.0);
        data[k-1] = div*dr*data[k-2];
        for (int l = 1; l < k-1; l++) data[k-l-1] = div*((dr+l)*data[k-l-2] + (k-l-dr)*data[k-l-1]);
        data[0] = div*(1-dr)*data[0];
    }
    ddata[0] = -data[0];
    for (int k = 1; k < order; k++) ddata[k] = data[k-1] - data[k];
    double div = 1.0/(order-1);
    data[order-1] = div*dr*data[order-2];
    for (int l = 1; l < order-1; l++) data[order-l-1] = div*((dr+l)*data[order-l-2] + (order-l-dr)*data[order-l-1]);
    data[0] = div*(1-dr)*data[0];
}

/* in-place 1-D DFT over a strided line; sign -1 forward, +1 backward; unnormalised */
static void dft_line(double* re, double* im, int n, long stride, int sign, const double* cs, const double* sn, double* tr, double* ti) {
    for (int k = 0; k < n; k++) {
        double ar = 0, ai = 0;
        for (int j = 0; j < n; j++) {
            const int m = (int) (((long) j*k) % n);
            const double c = cs[m], s = sign*sn[m];
            const double xr = re[j*stride], xi = im[j*stride];
            ar += xr*c - xi*s; ai += xr*s + xi*c;
        }
        tr[k] = ar; ti[k] = ai;
    }
    for (int k = 0; k < n; k++) { re[k*stride] = tr[k]; im[k*stride] = ti[k]; }
}

static void dft3d(double* re, double* im, int nx, int ny, int nz, int sign) {
    const int dims[3] = {nx, ny, nz};
    const long strides[3] = {(long) ny*nz, nz, 1};
    for (int d = 0; d < 3; d++) {
        const int n = dims[d];
        double* cs = (double*) malloc(sizeof(double)*n); double* sn = (double*) malloc(sizeof(double)*n);
        for (int m = 0; m < n; m++) { cs[m] = cos(2*M_PI*m/n); sn[m] = sin(2*M_PI*m/n); }
        const long nlines = (long) nx*ny*nz/n;
#pragma omp parallel
        {
            double* tr = (double*) malloc(sizeof(double)*n); double* ti = (double*) malloc(sizeof(double)*n);
#pragma omp for
            for (long l = 0; l < nlines; l++) {
                long base;      /* enumerate the start of every line along dimension d */
                if (d == 0) base = l;
                else if (d == 1) base = (l/nz)*(long) ny*nz + (l % nz);
                else base = l*nz;
                dft_line(re+base, im+base, n, strides[d], sign, cs, sn, tr, ti);
            }
            free(tr); free(ti);
        }
        free(cs); free(sn);
    }
}

/* the 3-D transform alone (forward), for checking against fftpack_exec_3d / numpy */
void orc_fft3d_forward(int nx, int ny, int nz, double* re, double* im) { dft3d(re, im, nx, ny, nz, -1); }

double orc_pme_reciprocal(int n, const double* pos, const double* q, const double* box, double alpha,
                          int nx, int ny, int nz, double* forces) {
    const int order = PME_ORDER;
    const int ng[3] = {nx, ny, nz};
    const double det = box[0]*box[4]*box[8], sc = 1.0/det;
    double R[9];           /* invert_box_vectors, ReferencePME.cpp:196-204 */
    R[0] = box[4]*box[8]*sc; R[1] = 0; R[2] = 0;
    R[3] = -box[3]*box[8]*sc; R[4] = box[0]*box[8]*sc; R[5] = 0;
    R[6] = (box[3]*box[7] - box[4]*box[6])*sc; R[7] = -box[0]*box[7]*sc; R[8] = box[0]*box[4]*sc;
    const long G = (long) nx*ny*nz;
    double* gr = (double*) calloc(G, sizeof(double)); double* gi = (double*) calloc(G, sizeof(double));
    int* idx = (int*) malloc(sizeof(int)*3*n);
    double* th = (double*) malloc(sizeof(double)*3*order*n); double* dth = (double*) malloc(sizeof(double)*3*order*n);
    for (int i = 0; i < n; i++)
        for (int d = 0; d < 3; d++) {
            double t = pos[3*i]*R[d] + pos[3*i+1]*R[3+d] + pos[3*i+2]*R[6+d];
            t = (t - floor(t))*ng[d];
            int ti = (int) t;
            idx[3*i+d] = ti % ng[d];
            bsplines(t - ti, th + (3*i+d)*order, dth + (3*i+d)*order);
        }
    for (int i = 0; i < n; i++)
        for (int ix = 0; ix < order; ix++) { const int xi = (idx[3*i]+ix) % nx;
            for (int iy = 0; iy < order; iy++) { const int yi = (idx[3*i+1]+iy) % ny;
                for (int iz = 0; iz < order; iz++) { const int zi = (idx[3*i+2]+iz) % nz;
                    gr[((long) xi*ny + yi)*nz + zi] += q[i]*th[(3*i)*order+ix]*th[(3*i+1)*order+iy]*th[(3*i+2)*order+iz]; } } }
    dft3d(gr, gi, nx, ny, nz, -1);
    double* mx_ = (double*) malloc(sizeof(double)*nx); double* my_ = (double*) malloc(sizeof(double)*ny); double* mz_ = (double*) malloc(sizeof(double)*nz);
    bspline_moduli(nx, mx_); bspline_moduli(ny, my_); bspline_moduli(nz, mz_);
    const double factor = M_PI*M_PI/(alpha*alpha), boxfactor = M_PI*det;
    double esum = 0;
    for (int kx = 0; kx < nx; kx++) { const double mx = (kx < (nx+1)/2) ? kx : kx-nx; const double mhx = mx*R[0]; const double bx = boxfactor*mx_[kx];
        for (int ky = 0; ky < ny; ky++) { const double my = (ky < (ny+1)/2) ? ky : ky-ny; const double mhy = mx*R[3] + my*R[4]; const double by = my_[ky];
            for (int kz = 0; kz < nz; kz++) {
                if (kx == 0 && ky == 0 && kz == 0) continue;
                const double mz = (kz < (nz+1)/2) ? kz : kz-nz; const double mhz = mx*R[6] + my*R[7] + mz*R[8];
                const long p = ((long) kx*ny + ky)*nz + kz;
                const double m2 = mhx*mhx + mhy*mhy + mhz*mhz;
                const double eterm = ONE_4PI_EPS0*exp(-factor*m2)/(m2*bx*by*mz_[kz]);
                esum += eterm*(gr[p]*gr[p] + gi[p]*gi[p]);
                gr[p] *= eterm; gi[p] *= eterm;
            } } }
    dft3d(gr, gi, nx, ny, nz, +1);
    for (int i = 0; i < n; i++) {
        double fx = 0, fy = 0, fz = 0;
        for (int ix = 0; ix < order; ix++) { const int xi = (idx[3*i]+ix) % nx;
            for (int iy = 0; iy < order; iy++) { const int yi = (idx[3*i+1]+iy) % ny;
                for (int iz = 0; iz < order; iz++) { const int zi = (idx[3*i+2]+iz) % nz;
                    const double g = gr[((long) xi*ny + yi)*nz + zi];
                    const double tx = th[(3*i)*order+ix], ty = th[(3*i+1)*order+iy], tz = th[(3*i+2)*order+iz];
                    fx += dth[(3*i)*order+ix]*ty*tz*g; fy += tx*dth[(3*i+1)*order+iy]*tz*g; fz += tx*ty*dth[(3*i+2)*order+iz]*g; } } }
        forces[3*i]   -= q[i]*(fx*nx*R[0]);
        forces[3*i+1] -= q[i]*(fx*nx*R[3] + fy*ny*R[4]);
        forces[3*i+2] -= q[i]*(fx*nx*R[6] + fy*ny*R[7] + fz*nz*R[8]);
    }
    free(gr); free(gi); free(idx); free(th); free(dth); free(mx_); free(my_); free(mz_);
    return 0.5*esum;
}

/* ------------------------------------------------------------------------------------------------------------
 * Bonded terms (ReferenceHarmonicBondIxn.cpp, ReferenceAngleBondIxn.cpp, ReferenceProperDihedralBond.cpp).  The _pbc
 * forms take the box of a force whose usesPeriodicBoundaryConditions() is set: every displacement the term is built
 * from goes through the minimum image (ReferenceHarmonicBondIxn.cpp:86-89, ReferenceAngleBondIxn.cpp:121-128,
 * ReferenceProperDihedralBond.cpp:91-100); box == NULL is the plain form. */
static void delta(const double* pos, int from, int to, const double* box, double* d) {
    for (int c = 0; c < 3; c++) d[c] = pos[3*to+c] - pos[3*from+c];
    if (box) min_image(d, box);
}

double orc_bonds_pbc(int nb, const int* bi, const int* bj, const double* r0, const double* k, const double* pos, const double* box, double* forces) {
    double e = 0;
    for (int b = 0; b < nb; b++) {
        const int i = bi[b], j = bj[b];
        double d[3];
        delta(pos, j, i, box, d);
        const double r = sqrt(d[0]*d[0] + d[1]*d[1] + d[2]*d[2]);
        const double dr = r - r0[b];
        e += 0.5*k[b]*dr*dr;
        const double s = -k[b]*dr/r;
        for (int c = 0; c < 3; c++) { forces[3*i+c] += s*d[c]; forces[3*j+c] -= s*d[c]; }
    }
    return e;
}
double orc_bonds(int nb, const int* bi, const int* bj, const double* r0, const double* k, const double* pos, double* forces) {
    return orc_bonds_pbc(nb, bi, bj, r0, k, pos, NULL, forces);
}

static void cross3(const double* a, const double* b, double* c) { c[0] = a[1]*b[2]-a[2]*b[1]; c[1] = a[2]*b[0]-a[0]*b[2]; c[2] = a[0]*b[1]-a[1]*b[0]; }
static double dot3(const double* a, const double* b) { return a[0]*b[0]+a[1]*b[1]+a[2]*b[2]; }

double orc_angles_pbc(int na, const int* ai, const int* aj, const int* ak, const double* th0, const double* kk, const double* pos, const double* box,
                      double* forces) {
    double e = 0;
    for (int a = 0; a < na; a++) {
        const int i = ai[a], j = aj[a], k = ak[a];
        double v0[3], v1[3], cp[3], c1[3], c3[3];
        delta(pos, i, j, box, v0);
        delta(pos, k, j, box, v1);
        cross3(v0, v1, cp);
        double rp = sqrt(dot3(cp, cp)); if (rp < 1e-6) rp = 1e-6;
        const double r21 = dot3(v0, v0), r23 = dot3(v1, v1);
        double cs = dot3(v0, v1)/sqrt(r21*r23); if (cs > 1) cs = 1; if (cs < -1) cs = -1;
        const double th = acos(cs), dth = th - th0[a];
        e += 0.5*kk[a]*dth*dth;
        const double dE = kk[a]*dth;
        cross3(v0, cp, c1); cross3(cp, v1, c3);
        for (int c = 0; c < 3; c++) {
            const double f1 = c1[c]*dE/(r21*rp), f3 = c3[c]*dE/(r23*rp);
            forces[3*i+c] += f1; forces[3*k+c] += f3; forces[3*j+c] -= f1+f3;
        }
    }
    return e;
}
double orc_angles(int na, const int* ai, const int* aj, const int* ak, const double* th0, const double* kk, const double* pos, double* forces) {
    return orc_angles_pbc(na, ai, aj, ak, th0, kk, pos, NULL, forces);
}

double orc_torsions_pbc(int nt, const int* ti, const int* tj, const int* tk, const int* tl, const int* per, const double* phase, const double* kk,
                        const double* pos, const double* box, double* forces) {
    double e = 0;
    for (int t = 0; t < nt; t++) {
        const int a = ti[t], b = tj[t], c = tk[t], d = tl[t];
        double v0[3], v1[3], v2[3], cp0[3], cp1[3], cc[3];
        delta(pos, b, a, box, v0);
        delta(pos, b, c, box, v1);
        delta(pos, d, c, box, v2);
        cross3(v0, v1, cp0); cross3(v1, v2, cp1);
        const double n0 = dot3(cp0, cp0), n1 = dot3(cp1, cp1);
        double cs = dot3(cp0, cp1)/sqrt(n0*n1); if (cs > 1) cs = 1; if (cs < -1) cs = -1;
        double th;
        if (cs > 0.99 || cs < -0.99) {
            cross3(cp0, cp1, cc);
            double sc = sqrt(dot3(cc, cc)/(n0*n1)); if (sc > 1) sc = 1;
            th = asin(sc); if (cs < 0) th = M_PI - th;
        }
        else th = acos(cs);
        if (dot3(v0, cp1) < 0) th = -th;
        const double arg = per[t]*th - phase[t];
        e += kk[t]*(1.0 + cos(arg));
        const double dE = -kk[t]*per[t]*sin(arg);
        const double nbc2 = dot3(v1, v1), nbc = sqrt(nbc2);
        const double ffx = -dE*nbc/n0, ffw = dE*nbc/n1, ffy = dot3(v0, v1)/nbc2, ffz = dot3(v2, v1)/nbc2;
        for (int x = 0; x < 3; x++) {
            const double f1 = ffx*cp0[x], f4 = ffw*cp1[x], s = ffy*f1 - ffz*f4;
            forces[3*a+x] += f1; forces[3*b+x] += s - f1; forces[3*c+x] += -s - f4; forces[3*d+x] += f4;
        }
    }
    return e;
}
double orc_torsions(int nt, const int* ti, const int* tj, const int* tk, const int* tl, const int* per, const double* phase, const double* kk,
                    const double* pos, double* forces) {
    return orc_torsions_pbc(nt, ti, tj, tk, tl, per, phase, kk, pos, NULL, forces);
}

/* ------------------------------------------------------------------------------------------------------------
 * SETTLE (ReferenceSETTLEAlgorithm::apply, ReferenceSETTLEAlgorithm.cpp:54-195).  x0: positions before the step
 * (constraints satisfied), x1: unconstrained new positions (in/out).  cluster w: atoms (a0,a1,a2), d1 = |a0a1| =
 * |a0a2|, d2 = |a1a2|. */
void orc_settle(int nw, const int* a0, const int* a1, const int* a2, const double* d1, const double* d2,
                const double* mass, const double* x0, double* x1) {
    for (int w = 0; w < nw; w++) {
        const int A = a0[w], B = a1[w], C = a2[w];
        double xp0[3], xp1[3], xp2[3];
        for (int k = 0; k < 3; k++) { xp0[k] = x1[3*A+k]-x0[3*A+k]; xp1[k] = x1[3*B+k]-x0[3*B+k]; xp2[k] = x1[3*C+k]-x0[3*C+k]; }
        const double m0 = mass[A], m1 = mass[B], m2 = mass[C];
        const double xb0 = x0[3*B]-x0[3*A], yb0 = x0[3*B+1]-x0[3*A+1], zb0 = x0[3*B+2]-x0[3*A+2];
        const double xc0 = x0[3*C]-x0[3*A], yc0 = x0[3*C+1]-x0[3*A+1], zc0 = x0[3*C+2]-x0[3*A+2];
        const double invTotalMass = 1/(m0+m1+m2);
        const double xcom = (xp0[0]*m0 + (xb0+xp1[0])*m1 + (xc0+xp2[0])*m2)*invTotalMass;
        const double ycom = (xp0[1]*m0 + (yb0+xp1[1])*m1 + (yc0+xp2[1])*m2)*invTotalMass;
        const double zcom = (xp0[2]*m0 + (zb0+xp1[2])*m1 + (zc0+xp2[2])*m2)*invTotalMass;
        const double xa1 = xp0[0]-xcom, ya1 = xp0[1]-ycom, za1 = xp0[2]-zcom;
        const double xb1 = xb0+xp1[0]-xcom, yb1 = yb0+xp1[1]-ycom, zb1 = zb0+xp1[2]-zcom;
        const double xc1 = xc0+xp2[0]-xcom, yc1 = yc0+xp2[1]-ycom, zc1 = zc0+xp2[2]-zcom;
        const double xaksZd = yb0*zc0-zb0*yc0, yaksZd = zb0*xc0-xb0*zc0, zaksZd = xb0*yc0-yb0*xc0;
        const double xaksXd = ya1*zaksZd-za1*yaksZd, yaksXd = za1*xaksZd-xa1*zaksZd, zaksXd = xa1*yaksZd-ya1*xaksZd;
        const double xaksYd = yaksZd*zaksXd-zaksZd*yaksXd, yaksYd = zaksZd*xaksXd-xaksZd*zaksXd, zaksYd = xaksZd*yaksXd-yaksZd*xaksXd;
        const double axlng = sqrt(xaksXd*xaksXd+yaksXd*yaksXd+zaksXd*zaksXd), aylng = sqrt(xaksYd*xaksYd+yaksYd*yaksYd+zaksYd*zaksYd),
                     azlng = sqrt(xaksZd*xaksZd+yaksZd*yaksZd+zaksZd*zaksZd);
        const double t11 = xaksXd/axlng, t21 = yaksXd/axlng, t31 = zaksXd/axlng, t12 = xaksYd/aylng, t22 = yaksYd/aylng, t32 = zaksYd/aylng,
                     t13 = xaksZd/azlng, t23 = yaksZd/azlng, t33 = zaksZd/azlng;
        const double xb0d = t11*xb0+t21*yb0+t31*zb0, yb0d = t12*xb0+t22*yb0+t32*zb0, xc0d = t11*xc0+t21*yc0+t31*zc0, yc0d = t12*xc0+t22*yc0+t32*zc0;
        const double za1d = t13*xa1+t23*ya1+t33*za1;
        const double xb1d = t11*xb1+t21*yb1+t31*zb1, yb1d = t12*xb1+t22*yb1+t32*zb1, zb1d = t13*xb1+t23*yb1+t33*zb1;
        const double xc1d = t11*xc1+t21*yc1+t31*zc1, yc1d = t12*xc1+t22*yc1+t32*zc1, zc1d = t13*xc1+t23*yc1+t33*zc1;
        const double rc = 0.5*d2[w];
        double rb = sqrt(d1[w]*d1[w]-rc*rc);
        const double ra = rb*(m1+m2)*invTotalMass;
        rb -= ra;
        const double sinphi = za1d/ra, cosphi = sqrt(1-sinphi*sinphi);
        const double sinpsi = (zb1d-zc1d)/(2*rc*cosphi), cospsi = sqrt(1-sinpsi*sinpsi);
        const double ya2d = ra*cosphi;
        double xb2d = -rc*cospsi;
        const double yb2d = -rb*cosphi-rc*sinpsi*sinphi, yc2d = -rb*cosphi+rc*sinpsi*sinphi;
        const double xb2d2 = xb2d*xb2d;
        const double hh2 = 4.0*xb2d2+(yb2d-yc2d)*(yb2d-yc2d)+(zb1d-zc1d)*(zb1d-zc1d);
        const double deltx = 2.0*xb2d+sqrt(4.0*xb2d2-hh2+d2[w]*d2[w]);
        xb2d -= deltx*0.5;
        const double alpha = xb2d*(xb0d-xc0d)+yb0d*yb2d+yc0d*yc2d, beta = xb2d*(yc0d-yb0d)+xb0d*yb2d+xc0d*yc2d;
        const double gamma = xb0d*yb1d-xb1d*yb0d+xc0d*yc1d-xc1d*yc0d;
        const double al2be2 = alpha*alpha+beta*beta;
        const double sintheta = (alpha*gamma-beta*sqrt(al2be2-gamma*gamma))/al2be2, costheta = sqrt(1-sintheta*sintheta);
        const double xa3d = -ya2d*sintheta, ya3d = ya2d*costheta, za3d = za1d;
        const double xb3d = xb2d*costheta-yb2d*sintheta, yb3d = xb2d*sintheta+yb2d*costheta, zb3d = zb1d;
        const double xc3d = -xb2d*costheta-yc2d*sintheta, yc3d = -xb2d*sintheta+yc2d*costheta, zc3d = zc1d;
        const double xa3 = t11*xa3d+t12*ya3d+t13*za3d, ya3 = t21*xa3d+t22*ya3d+t23*za3d, za3 = t31*xa3d+t32*ya3d+t33*za3d;
        const double xb3 = t11*xb3d+t12*yb3d+t13*zb3d, yb3 = t21*xb3d+t22*yb3d+t23*zb3d, zb3 = t31*xb3d+t32*yb3d+t33*zb3d;
        const double xc3 = t11*xc3d+t12*yc3d+t13*zc3d, yc3 = t21*xc3d+t22*yc3d+t23*zc3d, zc3 = t31*xc3d+t32*yc3d+t33*zc3d;
        x1[3*A] = x0[3*A]+xcom+xa3; x1[3*A+1] = x0[3*A+1]+ycom+ya3; x1[3*A+2] = x0[3*A+2]+zcom+za3;
        x1[3*B] = x0[3*B]+xcom+xb3-xb0; x1[3*B+1] = x0[3*B+1]+ycom+yb3-yb0; x1[3*B+2] = x0[3*B+2]+zcom+zb3-zb0;
        x1[3*C] = x0[3*C]+xcom+xc3-xc0; x1[3*C+1] = x0[3*C+1]+ycom+yc3-yc0; x1[3*C+2] = x0[3*C+2]+zcom+zc3-zc0;
    }
}

/* One deterministic integrator step for rigid-water systems (noise term omitted: compare at temperature 0).
 * kind 0 Verlet (ReferenceVerletDynamics.cpp), 1 Langevin (ReferenceStochasticDynamics.cpp:89-194).
 * forces: at the current positions.  SETTLE clusters as in orc_settle (nw may be 0). */
/* Velocity form of SETTLE (ReferenceSETTLEAlgorithm::applyToVelocities, ReferenceSETTLEAlgorithm.cpp:197-244): for every
 * rigid triangle find the three impulses t_c along the unit bond vectors e_c (c = AB, BC, CA) that remove the relative
 * velocity along each bond, for three arbitrary masses.  The reference writes the solution of the 3x3 system in closed form
 * (:229-235); here the system is assembled from its definition -- impulse t_c changes atom p_c by +e_c t_c/m and atom q_c by
 * -e_c t_c/m (:236-238) -- and solved by elimination.  x: positions with the constraints satisfied; v in/out. */
void orc_settle_velocities(int nw, const int* a0, const int* a1, const int* a2, const double* mass, const double* x, double* v) {
    static const int P[3] = {0, 1, 2}, Q[3] = {1, 2, 0};          /* bond c runs from atom P[c] to atom Q[c] of the triangle */
    for (int w = 0; w < nw; w++) {
        const int at[3] = {a0[w], a1[w], a2[w]};
        double e[3][3], A[3][4];
        for (int c = 0; c < 3; c++) {
            double len = 0;
            for (int k = 0; k < 3; k++) { e[c][k] = x[3*at[Q[c]]+k] - x[3*at[P[c]]+k]; len += e[c][k]*e[c][k]; }
            len = sqrt(len);
            for (int k = 0; k < 3; k++) e[c][k] /= len;
        }
        for (int c = 0; c < 3; c++) {
            double vrel = 0;
            for (int k = 0; k < 3; k++) vrel += (v[3*at[Q[c]]+k] - v[3*at[P[c]]+k])*e[c][k];
            A[c][3] = -vrel;
            for (int d = 0; d < 3; d++) {
                /* change of (v_Q[c] - v_P[c]).e_c per unit impulse on bond d */
                double onQ = 0, onP = 0;
                if (P[d] == Q[c]) onQ += 1.0/mass[at[Q[c]]];
                if (Q[d] == Q[c]) onQ -= 1.0/mass[at[Q[c]]];
                if (P[d] == P[c]) onP += 1.0/mass[at[P[c]]];
                if (Q[d] == P[c]) onP -= 1.0/mass[at[P[c]]];
                A[c][d] = (onQ - onP)*dot3(e[d], e[c]);
            }
        }
        for (int p = 0; p < 3; p++) {                              /* 3x3 elimination with partial pivoting */
            int piv = p;
            for (int r = p+1; r < 3; r++) if (fabs(A[r][p]) > fabs(A[piv][p])) piv = r;
            for (int q = 0; q < 4; q++) { const double t = A[p][q]; A[p][q] = A[piv][q]; A[piv][q] = t; }
            for (int r = p+1; r < 3; r++) { const double f = A[r][p]/A[p][p]; for (int q = p; q < 4; q++) A[r][q] -= f*A[p][q]; }
        }
        double t[3];
        for (int p = 2; p >= 0; p--) { double acc = A[p][3]; for (int q = p+1; q < 3; q++) acc -= A[p][q]*t[q]; t[p] = acc/A[p][p]; }
        for (int c = 0; c < 3; c++)
            for (int k = 0; k < 3; k++) { v[3*at[P[c]]+k] += e[c][k]*t[c]/mass[at[P[c]]]; v[3*at[Q[c]]+k] -= e[c][k]*t[c]/mass[at[Q[c]]]; }
    }
}

int orc_ccma(int ncon, const int* ai, const int* aj, const double* dist, const double* invm, const double* x, double* xp,
             const int* row_start, const int* col, const double* val, int constrain_velocities, double tol, int maxit);

/* ---- the engine's random numbers ----
 * Philox4x32-10 (Salmon et al., SC'11) and the Box-Muller transform exactly as the engine defines its noise
 * (openmm_b200/csrc/engine.h: philox, gauss3): counter (atom, step_lo, step_hi, 0x5eed5eed), key (seed, 0xb200b200).  This
 * restates the engine's OWN definition: the Reference platform draws its normals from a different generator, so it cannot
 * be the oracle for these bits.  The integer-to-uniform conversion is the engine's, exact in any precision; the transform
 * is done in double (the engine's fp32 transform agrees to a few 1e-7 relative). */
void orc_philox4x32_10(const unsigned int ctr[4], const unsigned int key[2], unsigned int out[4]) {
    unsigned int c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3], k0 = key[0], k1 = key[1];
    for (int r = 0; r < 10; r++) {
        const unsigned long long p0 = 0xD2511F53ull*c0, p1 = 0xCD9E8D57ull*c2;
        const unsigned int hi0 = (unsigned int) (p0 >> 32), lo0 = (unsigned int) p0;
        const unsigned int hi1 = (unsigned int) (p1 >> 32), lo1 = (unsigned int) p1;
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

void orc_gauss3(unsigned int seed, int atom, unsigned long long step, double g[3]) {
    const unsigned int ctr[4] = {(unsigned int) atom, (unsigned int) step, (unsigned int) (step >> 32), 0x5eed5eedu};
    const unsigned int key[2] = {seed, 0xb200b200u};
    unsigned int r[4];
    orc_philox4x32_10(ctr, key, r);
    const double u1 = ((r[0] >> 8) + 1u)/16777216.0, u2 = (r[1] >> 8)/16777216.0;         /* (0,1], [0,1) */
    const double u3 = ((r[2] >> 8) + 1u)/16777216.0, u4 = (r[3] >> 8)/16777216.0;
    const double m1 = sqrt(-2.0*log(u1)), m2 = sqrt(-2.0*log(u3));
    g[0] = m1*cos(2.0*M_PI*u2); g[1] = m1*sin(2.0*M_PI*u2); g[2] = m2*cos(2.0*M_PI*u4);
}

/* orc_gauss3 for the atoms atoms[0..n) at one step: g[3*i..] */
void orc_gauss3_atoms(unsigned int seed, int n, const int* atoms, unsigned long long step, double* g) {
    for (int i = 0; i < n; i++) orc_gauss3(seed, atoms[i], step, g + 3*i);
}

/* One Verlet / Langevin / LangevinMiddle step with its random force.  kind 0: leapfrog Verlet (ReferenceVerletDynamics.cpp),
 * 1: Langevin (ReferenceStochasticDynamics.cpp:89-194), 2: LangevinMiddle (ReferenceLangevinMiddleDynamics.cpp:54-127: kick,
 * velocity constraints, half drift, friction + noise, half drift, position constraints, velocity correction by the constraint
 * displacement).  The noise of atom i is gauss[3*i..3*i+2] (NULL: none, the zero-temperature step), scaled as the reference
 * scales it: sqrt(kT (1 - vscale^2)/m) g (Langevin), sqrt(1 - vscale^2) sqrt(kT/m) g (LangevinMiddle); massless atoms neither
 * move nor change velocity.  Constraints: the nw SETTLE clusters as in orc_settle, and every other constraint (ncon of them,
 * SHAKE clusters included) by orc_ccma in double with an identity coupling matrix to `tol` -- the Reference platform treats
 * every non-water constraint as one CCMA system.  Returns the most CCMA iterations one solve used, -1 if a solve did not
 * converge. */
int orc_langevin_step(int kind, int n, double dt, double friction, double kT, const double* mass, const double* forces,
                      const double* gauss, double* x, double* v, int nw, const int* a0, const int* a1, const int* a2,
                      const double* d1, const double* d2, int ncon, const int* ai, const int* aj, const double* dist, double tol) {
    const int maxit = 100000;
    double* xn = (double*) malloc(sizeof(double)*3*n);
    double* invm = NULL;
    int* rs = NULL; int* col = NULL; double* val = NULL;
    int iters = 0;
    if (ncon > 0) {
        invm = (double*) malloc(sizeof(double)*n);
        for (int i = 0; i < n; i++) invm[i] = mass[i] > 0 ? 1.0/mass[i] : 0.0;
        rs = (int*) malloc(sizeof(int)*(ncon+1)); col = (int*) malloc(sizeof(int)*ncon); val = (double*) malloc(sizeof(double)*ncon);
        for (int k = 0; k <= ncon; k++) rs[k] = k;
        for (int k = 0; k < ncon; k++) { col[k] = k; val[k] = 1.0; }
    }
#define CCMA_SOLVE(target, vel) do { \
        const int it = orc_ccma(ncon, ai, aj, dist, invm, x, target, rs, col, val, vel, tol, maxit); \
        if (it >= maxit) iters = -1; else if (iters >= 0 && it > iters) iters = it; } while (0)
    const double vscale = exp(-dt*friction), fscale = (friction == 0 ? dt : (1-vscale)/friction);
    if (kind == 2) {
        double* xu = (double*) malloc(sizeof(double)*3*n);
        for (int i = 0; i < n; i++) if (mass[i] > 0) for (int k = 0; k < 3; k++) v[3*i+k] += dt*forces[3*i+k]/mass[i];
        if (nw > 0) orc_settle_velocities(nw, a0, a1, a2, mass, x, v);
        if (ncon > 0) CCMA_SOLVE(v, 1);
        for (int i = 0; i < n; i++) for (int k = 0; k < 3; k++) {
            if (mass[i] > 0) {
                xn[3*i+k] = x[3*i+k] + 0.5*dt*v[3*i+k];
                v[3*i+k] *= vscale;
                if (gauss) v[3*i+k] += sqrt(1-vscale*vscale)*sqrt(kT/mass[i])*gauss[3*i+k];
                xn[3*i+k] += 0.5*dt*v[3*i+k];
            }
            else xn[3*i+k] = x[3*i+k];
            xu[3*i+k] = xn[3*i+k];
        }
        if (nw > 0) orc_settle(nw, a0, a1, a2, d1, d2, mass, x, xn);
        if (ncon > 0) CCMA_SOLVE(xn, 0);
        for (int i = 0; i < n; i++) if (mass[i] > 0) for (int k = 0; k < 3; k++) { v[3*i+k] += (xn[3*i+k]-xu[3*i+k])/dt; x[3*i+k] = xn[3*i+k]; }
        free(xu);
    }
    else {
        for (int i = 0; i < n; i++) {
            const double im = mass[i] > 0 ? 1.0/mass[i] : 0.0;
            for (int k = 0; k < 3; k++) {
                double vn = (kind == 1) ? vscale*v[3*i+k] + fscale*im*forces[3*i+k] : v[3*i+k] + dt*im*forces[3*i+k];
                if (kind == 1 && gauss) vn += sqrt(kT*(1-vscale*vscale)*im)*gauss[3*i+k];
                if (im == 0) vn = v[3*i+k];
                v[3*i+k] = vn;
                xn[3*i+k] = x[3*i+k] + (im == 0 ? 0.0 : vn*dt);
            }
        }
        if (nw > 0) orc_settle(nw, a0, a1, a2, d1, d2, mass, x, xn);
        if (ncon > 0) CCMA_SOLVE(xn, 0);
        for (int i = 0; i < n; i++) {
            if (mass[i] > 0) for (int k = 0; k < 3; k++) { v[3*i+k] = (xn[3*i+k]-x[3*i+k])/dt; x[3*i+k] = xn[3*i+k]; }
        }
    }
#undef CCMA_SOLVE
    free(xn); free(invm); free(rs); free(col); free(val);
    return iters;
}

/* One deterministic step (no random force: temperature 0), SETTLE the only constraints: orc_langevin_step without noise. */
void orc_step(int kind, int n, double dt, double friction, const double* mass, const double* forces, double* x, double* v,
              int nw, const int* a0, const int* a1, const int* a2, const double* d1, const double* d2) {
    orc_langevin_step(kind, n, dt, friction, 0.0, mass, forces, NULL, x, v, nw, a0, a1, a2, d1, d2, 0, NULL, NULL, NULL, 0.0);
}

/* ---- CCMA: ReferenceCCMAAlgorithm::applyConstraints (ReferenceCCMAAlgorithm.cpp:235-316), positions or velocities ----
 * ncon constraints (ai, aj, dist), inverse masses invm, reference geometry x (constraints satisfied), target xp (new positions,
 * or velocities when constrain_velocities != 0).  The (approximate) inverse of the coupling matrix comes in CSR form
 * (row_start, col, val): the reference computes its own from a sparse QR (:137-190); the algorithm iterates to the
 * tolerance with any reasonable approximation.  Returns the number of iterations used (maxit if it did not converge). */
int orc_ccma(int ncon, const int* ai, const int* aj, const double* dist, const double* invm, const double* x, double* xp,
             const int* row_start, const int* col, const double* val, int constrain_velocities, double tol, int maxit) {
    double* r = (double*) malloc(sizeof(double)*4*(size_t) ncon);            /* r_ij and d_ij^2 (:255-262) */
    double* delta = (double*) malloc(sizeof(double)*(size_t) ncon);
    double* tmp = (double*) malloc(sizeof(double)*(size_t) ncon);
    for (int k = 0; k < ncon; k++) {
        for (int d = 0; d < 3; d++) r[4*k+d] = x[3*ai[k]+d] - x[3*aj[k]+d];
        r[4*k+3] = r[4*k]*r[4*k] + r[4*k+1]*r[4*k+1] + r[4*k+2]*r[4*k+2];
    }
    const double lower = 1 - 2*tol + tol*tol, upper = 1 + 2*tol + tol*tol;          /* :263-264 */
    int it = 0;
    while (it < maxit) {
        int converged = 0;
        for (int k = 0; k < ncon; k++) {
            double rp[3];
            for (int d = 0; d < 3; d++) rp[d] = xp[3*ai[k]+d] - xp[3*aj[k]+d];
            const double rrpr = rp[0]*r[4*k] + rp[1]*r[4*k+1] + rp[2]*r[4*k+2];
            const double red = 0.5/(invm[ai[k]] + invm[aj[k]]);                     /* reducedMasses, :246-252 */
            if (constrain_velocities) {
                delta[k] = -2*red*rrpr/r[4*k+3];                                     /* :277-280 */
                if (fabs(delta[k]) <= tol) converged++;
            }
            else {
                const double rp2 = rp[0]*rp[0] + rp[1]*rp[1] + rp[2]*rp[2];
                const double d2 = dist[k]*dist[k];
                delta[k] = red*(d2 - rp2)/rrpr;                                      /* :282-291 */
                if (rp2 >= lower*d2 && rp2 <= upper*d2) converged++;
            }
        }
        if (converged == ncon) break;
        it++;
        for (int k = 0; k < ncon; k++) {                                             /* :298-305 */
            double s = 0;
            for (int e = row_start[k]; e < row_start[k+1]; e++) s += val[e]*delta[col[e]];
            tmp[k] = s;
        }
        for (int k = 0; k < ncon; k++) {                                             /* :306-312 */
            for (int d = 0; d < 3; d++) {
                const double dr = r[4*k+d]*tmp[k];
                xp[3*ai[k]+d] += dr*invm[ai[k]];
                xp[3*aj[k]+d] -= dr*invm[aj[k]];
            }
        }
    }
    free(r); free(delta); free(tmp);
    return it;
}
