// custom_nonbonded.cu -- CustomNonbondedForce: user-written pair potentials E(r, p1, p2) over the neighbour-list tiles (sm_90a).
//
// Every object's energy and dE/dr are expression programs (custom_interp.h, class B200MD_CUSTOM_NONBONDED): VAR 0 is r, PARAM k
// the first particle's parameter k and PARAM P+k the second's, and the DISCRETE opcodes read the Discrete1D/2D/3DFunction tables
// (CHARMM36's acoef(type1, type2)/r^12 - bcoef(type1, type2)/r^6, NBFIX tables).  The pair interaction is that of
// ReferenceCustomNonbondedIxn::calculateOneIxn: pairs with r < cutoff (every pair with NoCutoff), the minimum image with
// CutoffPeriodic, and with a switching distance s the energy and dE/dr multiplied through by S = 1 - 10 x^3 + 15 x^4 - 6 x^5,
// x = (r - s)/(cutoff - s), for r > s.  The long-range correction is added on the host (b200md_set_custom_nonbonded_lrc).
//
// Pairs.  One warp per tile of the current neighbour list (walk_tiles, engine.h), as the generalized Born sweeps of gbsa.cu
// walk it, but reading the tile's exclusion mask, and passing the j side through the lanes once per object (so the i atom's
// parameters of each object are read once per tile).  Bit k of lane i's mask word is the pair with the j atom the tile holds in
// lane k, and it is clear for an excluded pair, for j <= i in the diagonal tile and for padding.  Lane i holds the j atom of
// lane (i + k) & 31 after k rotations.  The list is built with the force's exclusions (the NonbondedForce's exceptions, which
// validateSystem requires to be the same pairs, or the force's own when there is no NonbondedForce).  Every object is
// evaluated in this one walk of the tiles, each only if its force group is in the evaluation's mask.
//
// Numerics.  The programs run in double on the double minimum-image displacement of the fp32 coordinates; the per-lane force
// sums go into the user-order 2^32 fixed-point buffer through integer atomics (never NbDev::forceS), so forces are
// bit-reproducible and do not depend on the order of the tiles or on what runs beside the kernel.
#include "engine.h"
#include "custom_interp.h"
#include "../../include/b200md.h"

#define FULL 0xffffffffu

template <bool ENERGY>
__global__ void __launch_bounds__(256) k_custom_nonbonded(NbDev nb, CnbDev cn) {
    const int lane = threadIdx.x & 31;
    const int src = (lane + 1) & 31;
    const CustomTables tables = {cn.ntables, cn.tableDims, cn.tableStart, cn.tableValues};
    const CustomBox box = {1.0, 0.0, 1.0, 0.0, 0.0, 1.0};      // not read: these programs hold no PERIODIC_DIST
    double e = 0.0;
    walk_tiles(nb, [&](const ListDev& L, int t, int si, int ai, int sj, int aj) {
        const int mi = L.tileMask[t];
        const unsigned int mask = mi < 0 ? FULL : L.maskPool[mi*32 + lane];
        const float4 pi = L.sposq[si];
        double fix = 0.0, fiy = 0.0, fiz = 0.0, fjx = 0.0, fjy = 0.0, fjz = 0.0;
        // one pass of the j side through the lanes per object: the i atom's parameters are read once per object and tile
        for (int o = 0; o < cn.nobj; o++) {
            if (!((cn.groupMask >> cn.group[o]) & 1u)) continue;
            const int np = cn.nparams[o];
            const double sw = cn.switchDist[o];
            const int b0 = cn.progStart[2*o], b1 = cn.progStart[2*o + 1], b2 = cn.progStart[2*o + 2];
            double par[B200MD_CUSTOM_MAX_PARAMS];
            if (ai >= 0) for (int q = 0; q < np; q++) par[q] = cn.params[((size_t) o*nb.npad + ai)*cn.stride + q];
            float4 pj = L.sposq[max(sj, 0)];
            int ajr = aj;
            for (int k = 0; k < 32; k++) {
                if (ai >= 0 && ajr >= 0 && ((mask >> ((lane + k) & 31)) & 1u)) {
                    const double3 d = tile_delta(nb.box, pi, pj);
                    const double r2 = d.x*d.x + d.y*d.y + d.z*d.z;
                    if (!cn.useCutoff || r2 < cn.cutoff2) {
                        const double r = sqrt(r2);
                        for (int q = 0; q < np; q++) par[np + q] = cn.params[((size_t) o*nb.npad + ajr)*cn.stride + q];
                        double dE = custom_run<B200MD_CUSTOM_MAX_STACK, false, true>(cn.code, cn.imm, b1, b2, &r, par, cn.globals, box, false, &tables);
                        // the energy program only where its value may be used: the energy, or the switching function's chain rule
                        // (for every pair of an object with a switching distance: a condition on r would split the warp)
                        if (ENERGY || sw >= 0.0) {
                            double E = custom_run<B200MD_CUSTOM_MAX_STACK, false, true>(cn.code, cn.imm, b0, b1, &r, par, cn.globals, box, false, &tables);
                            if (sw >= 0.0 && r > sw) {
                                const double w = 1.0/(cn.cutoff - sw), x = (r - sw)*w;
                                const double S = 1.0 + x*x*x*(-10.0 + x*(15.0 - 6.0*x));
                                const double dS = x*x*(-30.0 + x*(60.0 - 30.0*x))*w;
                                dE = dE*S + E*dS;
                                E *= S;
                            }
                            if (ENERGY) e += E;
                        }
                        const double f = dE/r;            // the force on i is f (x_j - x_i), on j its negative
                        fix += d.x*f; fiy += d.y*f; fiz += d.z*f;
                        fjx -= d.x*f; fjy -= d.y*f; fjz -= d.z*f;
                    }
                }
                pj.x = __shfl_sync(FULL, pj.x, src); pj.y = __shfl_sync(FULL, pj.y, src); pj.z = __shfl_sync(FULL, pj.z, src);
                ajr = __shfl_sync(FULL, ajr, src);
                fjx = shfl_d(fjx, src); fjy = shfl_d(fjy, src); fjz = shfl_d(fjz, src);
            }
        }
        if (ai >= 0) { add_fixed(&nb.force[ai], fix); add_fixed(&nb.force[ai + nb.npad], fiy); add_fixed(&nb.force[ai + 2*nb.npad], fiz); }
        if (aj >= 0) { add_fixed(&nb.force[aj], fjx); add_fixed(&nb.force[aj + nb.npad], fjy); add_fixed(&nb.force[aj + 2*nb.npad], fjz); }
    });
    if (ENERGY) {
        for (int off = 16; off > 0; off >>= 1) e += __shfl_xor_sync(FULL, e, off);
        if (lane == 0 && e != 0.0) atomicAdd(&nb.energy[EN_CNB], e);
    }
}

void launch_custom_nonbonded(const NbDev& nb, const CnbDev& cn, bool energy, cudaStream_t s) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // spread over the tiles like the generalized Born sweeps, at the high priority of the chains beside the tile kernel
    const dim3 tiles(sms*4), block(256);
    if (energy) launch_high(k_custom_nonbonded<true>, tiles, block, 0, s, nb, cn);
    else launch_high(k_custom_nonbonded<false>, tiles, block, 0, s, nb, cn);
}
