// custom_interp.h -- the interpreter of custom-term expression programs (B200MD_OP_*, include/b200md.h), one source for
// the device kernels (k_custom and k_compound, bonded.cu; k_custom_nonbonded, custom_nonbonded.cu) and the host (the program checks of engine.cu and the
// b200md_custom_*_probe calls).  A program is a Lepton ExpressionProgram flattened to (opcode, operand, immediate); this file
// restates ExpressionProgram::evaluate (ExpressionProgram.cpp:100-110), every Operation::evaluate (lepton/Operation.h) and,
// for PERIODIC_DIST and the POINT_* opcodes, ReferencePointDistanceFunction, ReferencePointAngleFunction and
// ReferencePointDihedralFunction (ReferencePointFunctions.cpp) and, for the DISCRETE opcodes, ReferenceDiscrete{1,2,3}DFunction
// (ReferenceTabulatedFunction.cpp) over a fixed-size double stack.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include "../../include/b200md.h"

#ifdef __CUDACC__
#define CUSTOM_HD __host__ __device__ __forceinline__
#else
#define CUSTOM_HD inline
#endif

// number of stack values an opcode consumes (Operation::getNumArguments); -1: not an opcode
CUSTOM_HD int custom_op_args(int op) {
    switch (op) {
        case B200MD_OP_CONST: case B200MD_OP_THETA: case B200MD_OP_PARAM: case B200MD_OP_GLOBAL: case B200MD_OP_VAR: return 0;
        case B200MD_OP_ADD: case B200MD_OP_SUB: case B200MD_OP_MUL: case B200MD_OP_DIV: case B200MD_OP_POW:
        case B200MD_OP_ATAN2: case B200MD_OP_MIN: case B200MD_OP_MAX: return 2;
        case B200MD_OP_SELECT: case B200MD_OP_DISCRETE3: return 3;
        case B200MD_OP_DISCRETE2: return 2;
        case B200MD_OP_PERIODIC_DIST: case B200MD_OP_POINT_DIST: return 6;
        case B200MD_OP_POINT_ANGLE: return 9;
        case B200MD_OP_POINT_DIHEDRAL: return 12;
        default: return op >= 0 && op < B200MD_OP_COUNT ? 1 : -1;
    }
}

// number of variables of a class (B200MD_CUSTOM_*) but a compound bond's (3 per particle of the expression): its derivative
// programs per expression
CUSTOM_HD int custom_num_vars(int cls) { return cls == B200MD_CUSTOM_EXTERNAL ? 3 : 1; }

// Operation::PowerConstant::evaluate: an integer exponent by repeated squaring, any other by pow
CUSTOM_HD double custom_pow_const(double x, double c) {
    int e = (int) c;
    if ((double) e != c) return pow(x, c);
    if (e < 0) { e = -e; x = 1.0/x; }
    double r = 1.0;
    while (e != 0) {
        if (e & 1) r *= x;
        x *= x;
        e >>= 1;
    }
    return r;
}

// The periodic box PERIODIC_DIST reduces by: a = (ax, 0, 0), b = (bx, by, 0), c = (cx, cy, cz), the reduced form of every
// OpenMM box.
struct CustomBox { double ax, bx, by, cx, cy, cz; };

// The minimum image of a displacement: reduced along c, b, a with floor(d/box_kk + 0.5), as ReferenceForce::getDeltaRPeriodic
// and the point functions of ReferencePointFunctions.cpp.
CUSTOM_HD void custom_min_image(double& dx, double& dy, double& dz, const CustomBox& box) {
    double s = floor(dz/box.cz + 0.5);
    dx -= s*box.cx; dy -= s*box.cy; dz -= s*box.cz;
    s = floor(dy/box.by + 0.5);
    dx -= s*box.bx; dy -= s*box.by;
    s = floor(dx/box.ax + 0.5);
    dx -= s*box.ax;
}

// ReferencePointDistanceFunction: a = the six arguments; which = -1 the distance, k in 0..5 its derivative by argument k.
CUSTOM_HD double custom_point_dist(const double* a, int which, const CustomBox& box, bool periodic) {
    double dx = a[0] - a[3], dy = a[1] - a[4], dz = a[2] - a[5];
    if (periodic) custom_min_image(dx, dy, dz, box);
    const double r = sqrt(dx*dx + dy*dy + dz*dz);
    if (which < 0) return r;
    if (r == 0.0) return 0.0;
    const double d = (which % 3) == 0 ? dx : (which % 3) == 1 ? dy : dz;
    return which < 3 ? d/r : -d/r;
}
CUSTOM_HD double custom_periodic_dist(const double* a, int which, const CustomBox& box) { return custom_point_dist(a, which, box, true); }

struct CustomVec { double x, y, z; };
CUSTOM_HD CustomVec custom_diff(const double* a, const double* b, const CustomBox& box, bool periodic) {
    CustomVec d = {a[0] - b[0], a[1] - b[1], a[2] - b[2]};
    if (periodic) custom_min_image(d.x, d.y, d.z, box);
    return d;
}
CUSTOM_HD CustomVec custom_cross(const CustomVec& a, const CustomVec& b) { return {a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x}; }
CUSTOM_HD double custom_dot(const CustomVec& a, const CustomVec& b) { return a.x*b.x + a.y*b.y + a.z*b.z; }
CUSTOM_HD double custom_comp(const CustomVec& a, int k) { return k == 0 ? a.x : k == 1 ? a.y : a.z; }

// ReferenceBondIxn::getAngleBetweenTwoVectors: the normed dot product (left 0 when it is 0, so a zero vector gives pi/2)
// clamped to [-1, 1]; within 0.01 of +-1 the angle comes from the cross product.
CUSTOM_HD double custom_angle_between(const CustomVec& u, const CustomVec& v) {
    double c = custom_dot(u, v);
    const double scale = custom_dot(u, u)*custom_dot(v, v);
    if (c != 0.0) c /= sqrt(scale);
    c = c > 1.0 ? 1.0 : c < -1.0 ? -1.0 : c;
    if (c > 0.99 || c < -0.99) {
        const CustomVec x = custom_cross(u, v);
        const double angle = asin(sqrt(custom_dot(x, x)/scale));
        return c < 0.0 ? 3.14159265358979323846 - angle : angle;
    }
    return acos(c);
}

// ReferencePointAngleFunction: a = the nine arguments (three points), the angle at the second point; which as above.
CUSTOM_HD double custom_point_angle(const double* a, int which, const CustomBox& box, bool periodic) {
    const CustomVec d12 = custom_diff(a + 3, a, box, periodic), d32 = custom_diff(a + 3, a + 6, box, periodic);
    if (which < 0) return custom_angle_between(d12, d32);
    const CustomVec cp = custom_cross(d12, d32);
    double len = sqrt(custom_dot(cp, cp));
    if (len < 1.0e-6) len = 1.0e-6;
    const CustomVec c0 = custom_cross(d12, cp), c2 = custom_cross(d32, cp);
    const double s0 = 1.0/(custom_dot(d12, d12)*len), s2 = -1.0/(custom_dot(d32, d32)*len);
    const int k = which % 3;
    const double g0 = custom_comp(c0, k)*s0, g2 = custom_comp(c2, k)*s2;
    return which < 3 ? -g0 : which < 6 ? g0 + g2 : -g2;
}

// ReferencePointDihedralFunction: a = the twelve arguments (four points); the sign is that of the first difference vector
// against the second normal (ReferenceBondIxn::getDihedralAngleBetweenThreeVectors); which as above.
CUSTOM_HD double custom_point_dihedral(const double* a, int which, const CustomBox& box, bool periodic) {
    const CustomVec d12 = custom_diff(a, a + 3, box, periodic), d32 = custom_diff(a + 6, a + 3, box, periodic),
                    d34 = custom_diff(a + 6, a + 9, box, periodic);
    const CustomVec c1 = custom_cross(d12, d32), c2 = custom_cross(d32, d34);
    if (which < 0) {
        const double angle = custom_angle_between(c1, c2);
        return custom_dot(d12, c2) < 0.0 ? -angle : angle;
    }
    const double n32 = custom_dot(d32, d32), r32 = sqrt(n32);
    const double f0 = -r32/custom_dot(c1, c1), f3 = r32/custom_dot(c2, c2);
    const double f1 = custom_dot(d12, d32)/n32, f2 = custom_dot(d34, d32)/n32;
    const int k = which % 3;
    const double i0 = f0*custom_comp(c1, k), i3 = f3*custom_comp(c2, k);
    const double s = f1*i0 - f2*i3;
    return which < 3 ? -i0 : which < 6 ? i0 - s : which < 9 ? i3 + s : -i3;
}

// The Discrete1D/2D/3DFunction tables of a context (b200md_set_custom_tables): table t has dims[t] = (dimensions, xsize, ysize,
// zsize) and the values [start[t], start[t+1]) of values, x fastest.
struct CustomTables { int n; const int4* dims; const int* start; const double* values; };

// A DISCRETE instruction of nargs arguments a[] and operand t: table t at the arguments rounded to the nearest integer, as
// ReferenceDiscrete{1,2,3}DFunction::evaluate, or NaN for an index outside the table (the Reference platform throws there; the
// NaN reaches the energy and the forces instead of a clamped, silently wrong value).  Operand -1 is a derivative: 0.
CUSTOM_HD double custom_discrete(const double* a, int nargs, int t, const CustomTables& tb) {
    if (t < 0) return 0.0;
    const int4 d = tb.dims[t];
    const double x = round(a[0]), y = nargs > 1 ? round(a[1]) : 0.0, z = nargs > 2 ? round(a[2]) : 0.0;
    if (!(x >= 0.0 && x < d.y && y >= 0.0 && y < d.z && z >= 0.0 && z < d.w)) return NAN;
    return tb.values[tb.start[t] + (int) x + d.y*((int) y + d.z*(int) z)];
}

// Program [begin, end) of `code` (x = opcode, y = operand) and `imm`, at the term's variables vars[] (THETA reads vars[0]).
// Argument k of an operation is st[sp + k]: argument 0 is the value pushed last, as in ExpressionProgram::evaluate.  The
// program must have passed custom_check_program (no underflow, depth <= STACK, one value left, VAR operands within the
// class's variables).  STACK is the capacity of the stack (B200MD_CUSTOM_MAX_STACK; B200MD_CUSTOM_COMPOUND_MAX_STACK for a
// compound bond); POINTS: the program may hold POINT_* instructions (a compound bond's), which take the minimum image iff
// `periodic`.  Without POINTS their code is not generated: the other classes' programs cannot hold them.  TABLES: the program
// may hold DISCRETE instructions (a custom nonbonded force's), which read `tables`; likewise not generated without it.
template <int STACK, bool POINTS, bool TABLES = false>
CUSTOM_HD double custom_run(const int2* code, const double* imm, int begin, int end, const double* vars, const double* params,
                            const double* globals, const CustomBox& box, bool periodic = false, const CustomTables* tables = nullptr) {
    double st[STACK];
    int sp = STACK;
    for (int pc = begin; pc < end; pc++) {
        const int2 in = code[pc];
        const int nargs = custom_op_args(in.x);
        const double a = nargs > 0 ? st[sp] : 0.0;
        const double b = nargs > 1 ? st[sp + 1] : 0.0;
        double r;
        switch (in.x) {
            case B200MD_OP_CONST: r = imm[pc]; break;
            case B200MD_OP_THETA: r = vars[0]; break;
            case B200MD_OP_VAR: r = vars[in.y]; break;
            case B200MD_OP_PARAM: r = params[in.y]; break;
            case B200MD_OP_GLOBAL: r = globals[in.y]; break;
            case B200MD_OP_ADD: r = a + b; break;
            case B200MD_OP_SUB: r = a - b; break;
            case B200MD_OP_MUL: r = a*b; break;
            case B200MD_OP_DIV: r = a/b; break;
            case B200MD_OP_POW: r = pow(a, b); break;
            case B200MD_OP_NEG: r = -a; break;
            case B200MD_OP_SQRT: r = sqrt(a); break;
            case B200MD_OP_EXP: r = exp(a); break;
            case B200MD_OP_LOG: r = log(a); break;
            case B200MD_OP_SIN: r = sin(a); break;
            case B200MD_OP_COS: r = cos(a); break;
            case B200MD_OP_SEC: r = 1.0/cos(a); break;
            case B200MD_OP_CSC: r = 1.0/sin(a); break;
            case B200MD_OP_TAN: r = tan(a); break;
            case B200MD_OP_COT: r = 1.0/tan(a); break;
            case B200MD_OP_ASIN: r = asin(a); break;
            case B200MD_OP_ACOS: r = acos(a); break;
            case B200MD_OP_ATAN: r = atan(a); break;
            case B200MD_OP_ATAN2: r = atan2(a, b); break;
            case B200MD_OP_SINH: r = sinh(a); break;
            case B200MD_OP_COSH: r = cosh(a); break;
            case B200MD_OP_TANH: r = tanh(a); break;
            case B200MD_OP_ERF: r = erf(a); break;
            case B200MD_OP_ERFC: r = erfc(a); break;
            case B200MD_OP_STEP: r = a >= 0.0 ? 1.0 : 0.0; break;
            case B200MD_OP_DELTA: r = a == 0.0 ? 1.0 : 0.0; break;
            case B200MD_OP_SQUARE: r = a*a; break;
            case B200MD_OP_CUBE: r = a*a*a; break;
            case B200MD_OP_RECIP: r = 1.0/a; break;
            case B200MD_OP_ADD_CONST: r = a + imm[pc]; break;
            case B200MD_OP_MUL_CONST: r = a*imm[pc]; break;
            case B200MD_OP_POW_CONST: r = custom_pow_const(a, imm[pc]); break;
            case B200MD_OP_MIN: r = b < a ? b : a; break;             // std::min(a, b)
            case B200MD_OP_MAX: r = a < b ? b : a; break;             // std::max(a, b)
            case B200MD_OP_ABS: r = fabs(a); break;
            case B200MD_OP_FLOOR: r = floor(a); break;
            case B200MD_OP_CEIL: r = ceil(a); break;
            case B200MD_OP_PERIODIC_DIST: r = custom_periodic_dist(st + sp, in.y, box); break;
            case B200MD_OP_SELECT: r = a != 0.0 ? b : st[sp + 2]; break;
            default:
                if (TABLES && in.x >= B200MD_OP_DISCRETE1) r = custom_discrete(st + sp, nargs, in.y, *tables);
                else if (!POINTS) r = 0.0;
                else if (in.x == B200MD_OP_POINT_DIST) r = custom_point_dist(st + sp, in.y, box, periodic);
                else if (in.x == B200MD_OP_POINT_ANGLE) r = custom_point_angle(st + sp, in.y, box, periodic);
                else r = custom_point_dihedral(st + sp, in.y, box, periodic);
                break;
        }
        sp += nargs - 1;
        st[sp] = r;
    }
    return st[STACK - 1];
}

// The checks of one program [begin, end) of class cls (B200MD_CUSTOM_*) that make custom_run safe: known opcodes, the
// variables of the class only (a torsion or an angle: THETA; a bond: VAR 0; an external: VAR 0..2 and PERIODIC_DIST with an
// operand in -1..5; a compound bond of nparticles particles: VAR 0..3 nparticles-1 and the POINT_* opcodes with an operand
// from -1 to their number of arguments - 1), PARAM operands < param_stride, GLOBAL operands < nglobals (nglobals < 0: not
// checked yet), no stack underflow, depth <= the class's stack capacity, exactly one value left, at most
// B200MD_CUSTOM_MAX_CODE instructions.  A custom nonbonded program reads VAR 0 (r) and may hold the DISCRETE opcodes, with an
// operand from -1 to ntables - 1 (ntables < 0: not checked yet); they are unknown opcodes for every other class.  nullptr if the program passes, else the reason.  An opcode of another class's is an
// unknown opcode for a torsion or an angle program, as is a POINT_* opcode for every class but the compound bond.  A centroid
// bond's program (of nparticles group centres) is checked as a compound bond's.
inline const char* custom_check_program(int cls, const int2* code, int begin, int end, int param_stride, int nglobals, int nparticles = 0,
                                        int ntables = -1) {
    const bool torsion = cls == B200MD_CUSTOM_TORSION, bond = cls == B200MD_CUSTOM_BOND, angle = cls == B200MD_CUSTOM_ANGLE,
               centroid = cls == B200MD_CUSTOM_CENTROID, compound = cls == B200MD_CUSTOM_COMPOUND || centroid,
               nonbonded = cls == B200MD_CUSTOM_NONBONDED;
#define CUSTOM_WHY(what) (torsion ? "custom torsion program: " what : bond ? "custom bond program: " what : \
                          angle ? "custom angle program: " what : centroid ? "custom centroid program: " what : \
                          compound ? "custom compound program: " what : nonbonded ? "custom nonbonded program: " what : \
                          "custom external program: " what)
    if (end <= begin) return CUSTOM_WHY("empty program");
    if (end - begin > B200MD_CUSTOM_MAX_CODE) return CUSTOM_WHY("more than 256 instructions");
    const int numVars = compound ? 3*nparticles : custom_num_vars(cls);
    int depth = 0;
    for (int pc = begin; pc < end; pc++) {
        const int op = code[pc].x, arg = code[pc].y;
        const int nargs = custom_op_args(op);
        const bool point = op == B200MD_OP_POINT_DIST || op == B200MD_OP_POINT_ANGLE || op == B200MD_OP_POINT_DIHEDRAL;
        const bool table = op == B200MD_OP_DISCRETE1 || op == B200MD_OP_DISCRETE2 || op == B200MD_OP_DISCRETE3;
        if (nargs < 0 || ((torsion || angle) && (op == B200MD_OP_VAR || op == B200MD_OP_PERIODIC_DIST)) || (point && !compound) ||
            (table && !nonbonded))
            return CUSTOM_WHY("unknown opcode");
        if (!torsion && !angle && op == B200MD_OP_THETA) return CUSTOM_WHY("THETA outside a torsion program");
        if ((bond || compound || nonbonded) && op == B200MD_OP_PERIODIC_DIST) return CUSTOM_WHY("PERIODIC_DIST outside an external program");
        if (table && (arg < -1 || (ntables >= 0 && arg >= ntables))) return CUSTOM_WHY("table index out of range");
        if (op == B200MD_OP_VAR && (arg < 0 || arg >= numVars)) return CUSTOM_WHY("variable index out of range for the class");
        if (op == B200MD_OP_PERIODIC_DIST && (arg < -1 || arg > 5)) return CUSTOM_WHY("periodic distance operand outside -1..5");
        if (point && (arg < -1 || arg >= nargs)) return CUSTOM_WHY("point function operand out of range");
        if (op == B200MD_OP_PARAM && (arg < 0 || arg >= param_stride)) return CUSTOM_WHY("parameter index out of range");
        if (op == B200MD_OP_GLOBAL && (arg < 0 || (nglobals >= 0 && arg >= nglobals))) return CUSTOM_WHY("global parameter index out of range");
        if (depth < nargs) return CUSTOM_WHY("stack underflow");
        depth += 1 - nargs;
        if (compound && depth > B200MD_CUSTOM_COMPOUND_MAX_STACK) return CUSTOM_WHY("stack deeper than 32");
        if (!compound && depth > B200MD_CUSTOM_MAX_STACK) return CUSTOM_WHY("stack deeper than 16");
    }
    if (depth != 1) return CUSTOM_WHY("does not end with exactly one value");
#undef CUSTOM_WHY
    return nullptr;
}
