// custom_interp.h -- the interpreter of custom-term expression programs (B200MD_OP_*, include/b200md.h), one source for
// the device kernel (k_custom, bonded.cu) and the host (the program checks of engine.cu and b200md_custom_term_probe).  A
// program is a Lepton ExpressionProgram flattened to (opcode, operand, immediate); this file restates
// ExpressionProgram::evaluate (ExpressionProgram.cpp:100-110), every Operation::evaluate (lepton/Operation.h) and, for
// PERIODIC_DIST, ReferencePointDistanceFunction (ReferencePointFunctions.cpp) over a fixed-size double stack.
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
        case B200MD_OP_SELECT: return 3;
        case B200MD_OP_PERIODIC_DIST: return 6;
        default: return op >= 0 && op < B200MD_OP_COUNT ? 1 : -1;
    }
}

// number of variables of a class (B200MD_CUSTOM_*): its derivative programs per expression
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

// ReferencePointDistanceFunction (periodic): a = the six arguments; which = -1 the distance, k in 0..5 its derivative by
// argument k.  The minimum image reduces along c, b, a with floor(d/box_kk + 0.5), as ReferenceForce::getDeltaRPeriodic.
CUSTOM_HD double custom_periodic_dist(const double* a, int which, const CustomBox& box) {
    double dx = a[0] - a[3], dy = a[1] - a[4], dz = a[2] - a[5];
    double s = floor(dz/box.cz + 0.5);
    dx -= s*box.cx; dy -= s*box.cy; dz -= s*box.cz;
    s = floor(dy/box.by + 0.5);
    dx -= s*box.bx; dy -= s*box.by;
    s = floor(dx/box.ax + 0.5);
    dx -= s*box.ax;
    const double r = sqrt(dx*dx + dy*dy + dz*dz);
    if (which < 0) return r;
    if (r == 0.0) return 0.0;
    const double d = (which % 3) == 0 ? dx : (which % 3) == 1 ? dy : dz;
    return which < 3 ? d/r : -d/r;
}

// Program [begin, end) of `code` (x = opcode, y = operand) and `imm`, at the term's variables vars[] (THETA reads vars[0]).
// Argument k of an operation is st[sp + k]: argument 0 is the value pushed last, as in ExpressionProgram::evaluate.  The
// program must have passed custom_check_program (no underflow, depth <= B200MD_CUSTOM_MAX_STACK, one value left, VAR
// operands within the class's variables).
CUSTOM_HD double custom_run(const int2* code, const double* imm, int begin, int end, const double* vars, const double* params,
                            const double* globals, const CustomBox& box) {
    double st[B200MD_CUSTOM_MAX_STACK];
    int sp = B200MD_CUSTOM_MAX_STACK;
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
            default: r = a != 0.0 ? b : st[sp + 2]; break;            // SELECT
        }
        sp += nargs - 1;
        st[sp] = r;
    }
    return st[B200MD_CUSTOM_MAX_STACK - 1];
}

// The checks of one program [begin, end) of class cls (B200MD_CUSTOM_*) that make custom_run safe: known opcodes, the
// variables of the class only (a torsion: THETA; a bond: VAR 0; an external: VAR 0..2 and PERIODIC_DIST with an operand in
// -1..5), PARAM operands < param_stride, GLOBAL operands < nglobals (nglobals < 0: not checked yet), no stack underflow,
// depth <= B200MD_CUSTOM_MAX_STACK, exactly one value left, at most B200MD_CUSTOM_MAX_CODE instructions.  nullptr if the
// program passes, else the reason.  For a torsion program VAR and PERIODIC_DIST are unknown opcodes.
inline const char* custom_check_program(int cls, const int2* code, int begin, int end, int param_stride, int nglobals) {
    const bool torsion = cls == B200MD_CUSTOM_TORSION, bond = cls == B200MD_CUSTOM_BOND;
#define CUSTOM_WHY(what) (torsion ? "custom torsion program: " what : bond ? "custom bond program: " what : "custom external program: " what)
    if (end <= begin) return CUSTOM_WHY("empty program");
    if (end - begin > B200MD_CUSTOM_MAX_CODE) return CUSTOM_WHY("more than 256 instructions");
    int depth = 0;
    for (int pc = begin; pc < end; pc++) {
        const int op = code[pc].x, arg = code[pc].y;
        const int nargs = custom_op_args(op);
        if (nargs < 0 || (torsion && (op == B200MD_OP_VAR || op == B200MD_OP_PERIODIC_DIST))) return CUSTOM_WHY("unknown opcode");
        if (!torsion && op == B200MD_OP_THETA) return CUSTOM_WHY("THETA outside a torsion program");
        if (bond && op == B200MD_OP_PERIODIC_DIST) return CUSTOM_WHY("PERIODIC_DIST outside an external program");
        if (op == B200MD_OP_VAR && (arg < 0 || arg >= custom_num_vars(cls))) return CUSTOM_WHY("variable index out of range for the class");
        if (op == B200MD_OP_PERIODIC_DIST && (arg < -1 || arg > 5)) return CUSTOM_WHY("periodic distance operand outside -1..5");
        if (op == B200MD_OP_PARAM && (arg < 0 || arg >= param_stride)) return CUSTOM_WHY("parameter index out of range");
        if (op == B200MD_OP_GLOBAL && (arg < 0 || (nglobals >= 0 && arg >= nglobals))) return CUSTOM_WHY("global parameter index out of range");
        if (depth < nargs) return CUSTOM_WHY("stack underflow");
        depth += 1 - nargs;
        if (depth > B200MD_CUSTOM_MAX_STACK) return CUSTOM_WHY("stack deeper than 16");
    }
    if (depth != 1) return CUSTOM_WHY("does not end with exactly one value");
#undef CUSTOM_WHY
    return nullptr;
}
