// cv.cu -- CustomCVForce on the device side.  The collective variables are evaluated by an inner context (an ordinary engine on
// the same device, one force group per variable); the host evaluates the energy expression and its derivatives dE/dCV_i.
//   k_cv_copy_state: the outer context's continuous user-order positions (hi + lo in mixed precision) into the inner context,
//                    as b200md_set_positions would upload them (cellOffset zeroed, the charge in posq.w kept).
//   k_cv_combine:    force += sum_i d_i F_i over the CV slots in a fixed order, F_i the inner context's fixed-point forces of
//                    variable i, added through the 2^32 fixed-point integer atomics.
#include "engine.h"
#include "../../include/b200md.h"
#include <algorithm>

__global__ void __launch_bounds__(128) k_cv_copy_state(NbDev from, NbDev to, int natoms) {
    const int a = blockIdx.x*blockDim.x + threadIdx.x;
    if (a >= natoms) return;
    const float4 h = from.posq[a];
    double x = h.x, y = h.y, z = h.z;
    if (from.posqCorr) { const float4 l = from.posqCorr[a]; x = pos_join(h.x, l.x); y = pos_join(h.y, l.y); z = pos_join(h.z, l.z); }
    const int kx = from.cellOffset[a], ky = from.cellOffset[a + from.npad], kz = from.cellOffset[a + 2*from.npad];
    x += kx*from.box.dax + ky*(double) from.box.bx + kz*(double) from.box.cx;
    y += ky*from.box.dby + kz*(double) from.box.cy;
    z += kz*from.box.dcz;
    float hx, hy, hz, lx, ly, lz;
    pos_split(x, hx, lx); pos_split(y, hy, ly); pos_split(z, hz, lz);
    to.posq[a] = make_float4(hx, hy, hz, to.posq[a].w);
    if (to.posqCorr) to.posqCorr[a] = make_float4(lx, ly, lz, 0.f);
    to.cellOffset[a] = 0; to.cellOffset[a + to.npad] = 0; to.cellOffset[a + 2*to.npad] = 0;
}

void launch_cv_copy_state(const NbDev& from, const NbDev& to, int natoms, cudaStream_t s) {
    launch_high(k_cv_copy_state, std::max(1, (natoms + 127)/128), 128, 0, s, from, to, natoms);
}

__global__ void __launch_bounds__(128) k_cv_combine(NbDev nb, CvDev cv) {
    const int t = blockIdx.x*blockDim.x + threadIdx.x;
    if (t >= 3*nb.npad) return;
    const size_t stride = 3*(size_t) nb.npad;
    double s = 0.0;
    for (int i = 0; i < cv.n; i++) s += cv.coeff[i]*(double) cv.forces[i*stride + t];
    const long long v = __double2ll_rn(s);
    if (v != 0) atomicAdd((unsigned long long*) &nb.force[t], (unsigned long long) v);
}

void launch_cv_combine(const NbDev& nb, const CvDev& cv, cudaStream_t s) {
    launch_high(k_cv_combine, (3*nb.npad + 127)/128, 128, 0, s, nb, cv);
}
