// custom_interp.h -- the interpreter of custom-torsion expression programs (B200MD_OP_*, include/b200md.h), one source for
// the device kernel (k_custom_torsion, bonded.cu) and the host (the program checks of engine.cu and
// b200md_custom_program_probe).  A program is a Lepton ExpressionProgram flattened to (opcode, operand, immediate); this
// file restates ExpressionProgram::evaluate (ExpressionProgram.cpp:100-110) and every Operation::evaluate
// (lepton/Operation.h) over a fixed-size double stack.
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
        case B200MD_OP_CONST: case B200MD_OP_THETA: case B200MD_OP_PARAM: case B200MD_OP_GLOBAL: return 0;
        case B200MD_OP_ADD: case B200MD_OP_SUB: case B200MD_OP_MUL: case B200MD_OP_DIV: case B200MD_OP_POW:
        case B200MD_OP_ATAN2: case B200MD_OP_MIN: case B200MD_OP_MAX: return 2;
        case B200MD_OP_SELECT: return 3;
        default: return op >= 0 && op < B200MD_OP_COUNT ? 1 : -1;
    }
}

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

// Program [begin, end) of `code` (x = opcode, y = operand) and `imm`, at the dihedral theta.  Argument k of an operation is
// st[sp + k]: argument 0 is the value pushed last, as in ExpressionProgram::evaluate.  The program must have passed
// custom_check_program (no underflow, depth <= B200MD_CUSTOM_MAX_STACK, one value left).
CUSTOM_HD double custom_run(const int2* code, const double* imm, int begin, int end, double theta, const double* params,
                            const double* globals) {
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
            case B200MD_OP_THETA: r = theta; break;
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
            default: r = a != 0.0 ? b : st[sp + 2]; break;            // SELECT
        }
        sp += nargs - 1;
        st[sp] = r;
    }
    return st[B200MD_CUSTOM_MAX_STACK - 1];
}

// The checks of one program [begin, end) that make custom_run safe: known opcodes, PARAM operands < param_stride, GLOBAL
// operands < nglobals (nglobals < 0: not checked yet), no stack underflow, depth <= B200MD_CUSTOM_MAX_STACK, exactly one
// value left, at most B200MD_CUSTOM_MAX_CODE instructions.  nullptr if the program passes, else the reason.
inline const char* custom_check_program(const int2* code, int begin, int end, int param_stride, int nglobals) {
    if (end <= begin) return "custom torsion program: empty program";
    if (end - begin > B200MD_CUSTOM_MAX_CODE) return "custom torsion program: more than 256 instructions";
    int depth = 0;
    for (int pc = begin; pc < end; pc++) {
        const int op = code[pc].x, arg = code[pc].y;
        const int nargs = custom_op_args(op);
        if (nargs < 0) return "custom torsion program: unknown opcode";
        if (op == B200MD_OP_PARAM && (arg < 0 || arg >= param_stride)) return "custom torsion program: parameter index out of range";
        if (op == B200MD_OP_GLOBAL && (arg < 0 || (nglobals >= 0 && arg >= nglobals))) return "custom torsion program: global parameter index out of range";
        if (depth < nargs) return "custom torsion program: stack underflow";
        depth += 1 - nargs;
        if (depth > B200MD_CUSTOM_MAX_STACK) return "custom torsion program: stack deeper than 16";
    }
    if (depth != 1) return "custom torsion program: does not end with exactly one value";
    return nullptr;
}
