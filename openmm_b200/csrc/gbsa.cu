// gbsa.cu -- GBSAOBCForce: OBC II generalized Born implicit solvent with the ACE non-polar term, over the neighbour-list
// tiles (sm_90a).
//
// The model (Onufriev, Bashford and Case, Proteins 55:383, 2004; ACE term of Schaefer, Bartels and Karplus, 1998), with
// rho = R - 0.009 nm the offset radius and s the scale factor of an atom:
//   Born sum     S_i = sum_{j != i, r_ij <= cutoff} I(r_ij, rho_i, s_j rho_j)      (asymmetric: i and j each gain their own term)
//   I(r, rho, sr) = [l - u + r/4 (u^2 - l^2) + ln(u/l)/(2r) + sr^2/(4r) (l^2 - u^2)] (+ 2 (1/rho - l) when rho < sr - r),
//                   l = 1/max(rho, |r - sr|), u = 1/(r + sr), zero unless rho < r + sr
//   Born radius  Psi_i = rho_i S_i/2, T_i = tanh(Psi - 0.8 Psi^2 + 4.85 Psi^3), B_i = 1/(1/rho_i - T_i/R_i)
//   energy       E = sum_i 4 pi gamma_SA (R_i + 0.14)^2 (R_i/B_i)^6 + sum_{i <= j} w_ij f q_i q_j/sqrt(r^2 + B_i B_j exp(-r^2/(4 B_i B_j)))
//                with f = -ONE_4PI_EPS0 (1/eps_solute - 1/eps_solvent), w_ii = 1/2, w_ij = 1, and with a cutoff the pair
//                term shifted by -f q_i q_j/cutoff (i != j)
// Forces: the explicit r dependence of the GB pairs (k_gb_pairs) plus the chain rule through the Born radii: dE/dB_i (ACE,
// self and pair terms) times dB_i/dS_i = B_i^2 C_i/2 times dS_i/dr_ij (k_gb_chain), the same closed forms the Reference
// platform evaluates (ReferenceObc.cpp is the behaviour matched, tests/gbsa_harness.py the double-precision restatement).
//
// Pairs.  The tile list of the current neighbour list (NbDev::list, built this evaluation) holds every pair within the padded
// cutoff exactly once: i-block ib's diagonal tile holds the atoms of block ib itself (flushed on its own, build_tiles_iblock)
// and every other tile of ib holds atoms of j-blocks > ib (candidates start at jb >= ib).  So a pair (tile i-slot si, j-slot
// sj) of a tile is counted iff sj > si, sj is a real slot (>= 0) and si < natoms -- the tile's exclusion mask is NOT used:
// OBC counts bonded and excluded pairs like any other.  The sorted order is fixed for the whole evaluation, because the chain
// is launched after this evaluation's list check and build; parameters are read in user order through sorig.  The passes
// never touch NbDev::forceS (owned by k_pair / k_fold_sorted, which may run beside them): forces go straight into the
// user-order 2^32 fixed-point buffer through integer atomics, so the result does not depend on the order of the tiles.
//
// Numerics.  The pair passes run in double.  The Born integral and its derivative are differences of nearly equal terms
// (l - u, ln(u/l)) that lose most of their digits in fp32 for bonded and nearest-neighbour pairs, and the Born radius of a
// buried atom amplifies an error of S_i many times; the per-pair partial sums of a warp are then converted to fixed point.
#include "engine.h"
#include "../../include/b200md.h"
#include <algorithm>

#define FULL 0xffffffffu
#define GB_OFFSET 0.009
#define GB_PROBE 0.14
#define GB_ALPHA 1.0
#define GB_BETA 0.8
#define GB_GAMMA 4.85

// I(r, rho_i, s_j rho_j) of the header, 0 when the scaled sphere of j does not reach the offset sphere of i
__device__ __forceinline__ double obc_integral(double r, double rInv, double rho, double sr) {
    if (rho >= r + sr) return 0.0;
    const double l = 1.0/fmax(rho, fabs(r - sr)), u = 1.0/(r + sr);
    const double l2 = l*l, u2 = u*u;
    double t = l - u + 0.25*r*(u2 - l2) + 0.5*rInv*log(u/l) + 0.25*sr*sr*rInv*(l2 - u2);
    if (rho < sr - r) t += 2.0*(1.0/rho - l);
    return t;
}

// dI/dr divided by r, as the force of the chain rule uses it (0 when I is)
__device__ __forceinline__ double obc_integral_deriv(double r, double r2Inv, double rho, double sr) {
    if (rho >= r + sr) return 0.0;
    const double l = 1.0/fmax(rho, fabs(r - sr)), u = 1.0/(r + sr);
    return 0.125*(1.0 + sr*sr*r2Inv)*(l*l - u*u) + 0.25*log(u/l)*r2Inv;
}

// pass 1: the Born sums
__global__ void __launch_bounds__(256) k_gb_born(NbDev nb, GbsaDev gb) {
    const int src = ((threadIdx.x & 31) + 1) & 31;
    walk_tiles(nb, [&](const ListDev& L, int, int si, int ai, int sj, int aj) {
        const float4 pi = L.sposq[si];
        const double2 ri = ai >= 0 ? gb.radius[ai] : make_double2(1.0, 0.0);
        float4 pj = L.sposq[max(sj, 0)];
        double2 rj = aj >= 0 ? gb.radius[aj] : make_double2(1.0, 0.0);
        double sumI = 0.0, sumJ = 0.0;
        for (int k = 0; k < 32; k++) {
            if (ai >= 0 && sj > si) {
                const double3 d = tile_delta(nb.box, pi, pj);
                const double r2 = d.x*d.x + d.y*d.y + d.z*d.z;
                if (!gb.useCutoff || r2 <= gb.cutoff2) {
                    const double r = sqrt(r2), rInv = 1.0/r;
                    sumI += obc_integral(r, rInv, ri.x, rj.y);
                    sumJ += obc_integral(r, rInv, rj.x, ri.y);
                }
            }
            pj.x = __shfl_sync(FULL, pj.x, src); pj.y = __shfl_sync(FULL, pj.y, src); pj.z = __shfl_sync(FULL, pj.z, src);
            rj.x = shfl_d(rj.x, src); rj.y = shfl_d(rj.y, src);
            sj = __shfl_sync(FULL, sj, src); aj = __shfl_sync(FULL, aj, src);
            sumJ = shfl_d(sumJ, src);
        }
        if (ai >= 0) add_fixed(&gb.bornSum[ai], sumI);
        if (aj >= 0) add_fixed(&gb.bornSum[aj], sumJ);
    });
}

__device__ __forceinline__ void gb_energy_add(const NbDev& nb, double e) {
    for (int off = 16; off > 0; off >>= 1) e += __shfl_xor_sync(FULL, e, off);
    if ((threadIdx.x & 31) == 0 && e != 0.0) atomicAdd(&nb.energy[EN_GB], e);
}

// pass 2, per atom in double: Born radius, chain factor, the ACE term and the self term (energy and their dE/dB); the Born
// sum is zeroed for the next evaluation once read
template <bool ENERGY>
__global__ void __launch_bounds__(256) k_gb_radii(NbDev nb, GbsaDev gb) {
    const int a = blockIdx.x*blockDim.x + threadIdx.x;
    double e = 0.0;
    if (a < nb.natoms) {
        const double S = (double) gb.bornSum[a]*(1.0/B200MD_FORCE_SCALE);
        gb.bornSum[a] = 0;
        const double rho = gb.radius[a].x, R = gb.atomRadius[a];
        const double psi = 0.5*rho*S;
        const double T = tanh(psi*(GB_ALPHA + psi*(-GB_BETA + GB_GAMMA*psi)));
        const double B = 1.0/(1.0/rho - T/R);
        const double C = rho*(GB_ALPHA - 2.0*GB_BETA*psi + 3.0*GB_GAMMA*psi*psi)*(1.0 - T*T)/R;
        double dEdB = 0.0;
        if (B > 0.0) {
            const double x = R/B, x2 = x*x;
            const double sa = gb.surfaceFactor*(R + GB_PROBE)*(R + GB_PROBE)*x2*x2*x2;
            e += sa;
            dEdB -= 6.0*sa/B;
        }
        const double q = gb.charge[a];
        const double G = gb.prefactor*q*q/B;         // i = j: r = 0, denominator B
        e += 0.5*G;
        dEdB -= 0.5*G/B;
        gb.bornR[a] = B; gb.chain[a] = C;
        gb.dEdB[a] = __double2ll_rn(dEdB*B200MD_FORCE_SCALE);
    }
    if (ENERGY) gb_energy_add(nb, e);
}

// pass 3: the GB pair terms -- energy, the explicit r-dependent forces, and dE/dB of both atoms
template <bool ENERGY>
__global__ void __launch_bounds__(256) k_gb_pairs(NbDev nb, GbsaDev gb) {
    const int src = ((threadIdx.x & 31) + 1) & 31;
    double e = 0.0;
    const double shift = gb.useCutoff ? 1.0/gb.cutoff : 0.0;
    walk_tiles(nb, [&](const ListDev& L, int, int si, int ai, int sj, int aj) {
        const float4 pi = L.sposq[si];
        const double qi = ai >= 0 ? gb.prefactor*gb.charge[ai] : 0.0, bi = ai >= 0 ? gb.bornR[ai] : 1.0;
        float4 pj = L.sposq[max(sj, 0)];
        double qj = aj >= 0 ? gb.charge[aj] : 0.0, bj = aj >= 0 ? gb.bornR[aj] : 1.0;
        double fix = 0.0, fiy = 0.0, fiz = 0.0, fjx = 0.0, fjy = 0.0, fjz = 0.0, dI = 0.0, dJ = 0.0;
        for (int k = 0; k < 32; k++) {
            if (ai >= 0 && sj > si) {
                const double3 d = tile_delta(nb.box, pi, pj);
                const double r2 = d.x*d.x + d.y*d.y + d.z*d.z;
                if (!gb.useCutoff || r2 <= gb.cutoff2) {
                    const double a2 = bi*bj, D = 0.25*r2/a2, ex = exp(-D);
                    const double den2 = r2 + a2*ex, den2Inv = 1.0/den2;
                    const double qq = qi*qj;
                    const double G = qq*sqrt(den2Inv);
                    const double dGdr = -G*(1.0 - 0.25*ex)*den2Inv;
                    const double dGda2 = -0.5*G*ex*(1.0 + D)*den2Inv;
                    fix += d.x*dGdr; fiy += d.y*dGdr; fiz += d.z*dGdr;
                    fjx -= d.x*dGdr; fjy -= d.y*dGdr; fjz -= d.z*dGdr;
                    dI += dGda2*bj; dJ += dGda2*bi;
                    if (ENERGY) e += G - qq*shift;
                }
            }
            pj.x = __shfl_sync(FULL, pj.x, src); pj.y = __shfl_sync(FULL, pj.y, src); pj.z = __shfl_sync(FULL, pj.z, src);
            qj = shfl_d(qj, src); bj = shfl_d(bj, src);
            sj = __shfl_sync(FULL, sj, src); aj = __shfl_sync(FULL, aj, src);
            fjx = shfl_d(fjx, src); fjy = shfl_d(fjy, src); fjz = shfl_d(fjz, src); dJ = shfl_d(dJ, src);
        }
        if (ai >= 0) {
            add_fixed(&nb.force[ai], fix); add_fixed(&nb.force[ai + nb.npad], fiy); add_fixed(&nb.force[ai + 2*nb.npad], fiz);
            add_fixed(&gb.dEdB[ai], dI);
        }
        if (aj >= 0) {
            add_fixed(&nb.force[aj], fjx); add_fixed(&nb.force[aj + nb.npad], fjy); add_fixed(&nb.force[aj + 2*nb.npad], fjz);
            add_fixed(&gb.dEdB[aj], dJ);
        }
    });
    if (ENERGY) gb_energy_add(nb, e);
}

// pass 4, per atom: dE/dB_i times B_i^2 C_i
__global__ void __launch_bounds__(256) k_gb_fold(NbDev nb, GbsaDev gb) {
    const int a = blockIdx.x*blockDim.x + threadIdx.x;
    if (a >= nb.natoms) return;
    const double B = gb.bornR[a];
    gb.bornForce[a] = (double) gb.dEdB[a]*(1.0/B200MD_FORCE_SCALE)*B*B*gb.chain[a];
}

// pass 5: the forces of the chain rule through the Born sums of both atoms of every pair
__global__ void __launch_bounds__(256) k_gb_chain(NbDev nb, GbsaDev gb) {
    const int src = ((threadIdx.x & 31) + 1) & 31;
    walk_tiles(nb, [&](const ListDev& L, int, int si, int ai, int sj, int aj) {
        const float4 pi = L.sposq[si];
        const double2 ri = ai >= 0 ? gb.radius[ai] : make_double2(1.0, 0.0);
        const double bfi = ai >= 0 ? gb.bornForce[ai] : 0.0;
        float4 pj = L.sposq[max(sj, 0)];
        double2 rj = aj >= 0 ? gb.radius[aj] : make_double2(1.0, 0.0);
        double bfj = aj >= 0 ? gb.bornForce[aj] : 0.0;
        double fix = 0.0, fiy = 0.0, fiz = 0.0, fjx = 0.0, fjy = 0.0, fjz = 0.0;
        for (int k = 0; k < 32; k++) {
            if (ai >= 0 && sj > si) {
                const double3 d = tile_delta(nb.box, pi, pj);
                const double r2 = d.x*d.x + d.y*d.y + d.z*d.z;
                if (!gb.useCutoff || r2 <= gb.cutoff2) {
                    const double r = sqrt(r2), rInv = 1.0/r, r2Inv = rInv*rInv;
                    const double de = (bfi*obc_integral_deriv(r, r2Inv, ri.x, rj.y) + bfj*obc_integral_deriv(r, r2Inv, rj.x, ri.y))*rInv;
                    fix -= d.x*de; fiy -= d.y*de; fiz -= d.z*de;
                    fjx += d.x*de; fjy += d.y*de; fjz += d.z*de;
                }
            }
            pj.x = __shfl_sync(FULL, pj.x, src); pj.y = __shfl_sync(FULL, pj.y, src); pj.z = __shfl_sync(FULL, pj.z, src);
            rj.x = shfl_d(rj.x, src); rj.y = shfl_d(rj.y, src); bfj = shfl_d(bfj, src);
            sj = __shfl_sync(FULL, sj, src); aj = __shfl_sync(FULL, aj, src);
            fjx = shfl_d(fjx, src); fjy = shfl_d(fjy, src); fjz = shfl_d(fjz, src);
        }
        if (ai >= 0) { add_fixed(&nb.force[ai], fix); add_fixed(&nb.force[ai + nb.npad], fiy); add_fixed(&nb.force[ai + 2*nb.npad], fiz); }
        if (aj >= 0) { add_fixed(&nb.force[aj], fjx); add_fixed(&nb.force[aj + nb.npad], fjy); add_fixed(&nb.force[aj + 2*nb.npad], fjz); }
    });
}

void launch_gbsa(const NbDev& nb, const GbsaDev& gb, bool energy, cudaStream_t s) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // the pair passes spread over the tiles (DHFR-GBSA has ~80 i-blocks for 132 SMs); launched at the high priority of the
    // chains that run beside the tile kernel (launch_high), so their CTAs take the SM slots the tile kernel hands back
    const dim3 tiles(sms*4), atoms((nb.natoms + 255)/256), block(256);
    launch_high(k_gb_born, tiles, block, 0, s, nb, gb);
    if (energy) launch_high(k_gb_radii<true>, atoms, block, 0, s, nb, gb);
    else launch_high(k_gb_radii<false>, atoms, block, 0, s, nb, gb);
    if (energy) launch_high(k_gb_pairs<true>, tiles, block, 0, s, nb, gb);
    else launch_high(k_gb_pairs<false>, tiles, block, 0, s, nb, gb);
    launch_high(k_gb_fold, atoms, block, 0, s, nb, gb);
    launch_high(k_gb_chain, tiles, block, 0, s, nb, gb);
}
