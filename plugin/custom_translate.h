// custom_translate.h -- CustomTorsionForce, CustomBondForce, CustomExternalForce, CustomAngleForce,
// CustomCompoundBondForce, CustomCentroidBondForce and CustomNonbondedForce expressions -> the instruction programs of
// b200md_set_custom_torsions / _bonds / _externals / _angles / _compound / _centroid / _nonbonded (B200MD_OP_*, include/b200md.h).  Lepton, part of the host's
// libOpenMM.so, parses, optimises and differentiates the expression exactly as the Reference platform does
// (ReferenceCalcCustom{Torsion,Bond,External,Angle,CompoundBond,CentroidBond}ForceKernel::initialize) and makes the stack program
// (ExpressionProgram); this file only maps every Lepton::Operation to one instruction.  Included by the plugin
// (B200Platform.cpp) and by its test C API (tests/custom_capi.cpp), so that both make the same programs.
#ifndef B200MD_CUSTOM_TRANSLATE_H_
#define B200MD_CUSTOM_TRANSLATE_H_
#include "openmm/OpenMMException.h"
#include "openmm/CustomCompoundBondForce.h"
#include "openmm/internal/CustomCompoundBondForceImpl.h"
#include "openmm/CustomCentroidBondForce.h"
#include "openmm/internal/CustomCentroidBondForceImpl.h"
#include "openmm/CustomNonbondedForce.h"
#include "openmm/TabulatedFunction.h"
#include "lepton/CustomFunction.h"
#include "lepton/ExpressionProgram.h"
#include "lepton/Operation.h"
#include "lepton/ParsedExpression.h"
#include "lepton/Parser.h"
#include "../include/b200md.h"
#include <map>
#include <string>
#include <vector>

// the Reference platform's evaluation of a TabulatedFunction as a Lepton function, exported by libOpenMM.so
// (platforms/reference/include/ReferenceTabulatedFunction.h)
extern "C" Lepton::CustomFunction* createReferenceTabulatedFunction(const OpenMM::TabulatedFunction& function);

namespace b200md_custom {

// An expression the platform cannot run although it is valid (a hard limit, a tabulated function): validateSystem refuses
// the System with it, so that the Context moves to another platform.
class Unsupported : public OpenMM::OpenMMException {
public:
    explicit Unsupported(const std::string& msg) : OpenMM::OpenMMException(msg) {}
};

struct Program {
    std::vector<int> op, arg;
    std::vector<double> imm;
};

// periodicdistance(x, y, z, x0, y0, z0) of a CustomExternalForce, for Lepton's parser: the programs compute it on the device
// (PERIODIC_DIST), so it is never evaluated here.  An expression that would have it evaluated while optimising (all six
// arguments constant) is refused.
class PeriodicDistancePlaceholder : public Lepton::CustomFunction {
public:
    int getNumArguments() const { return 6; }
    double evaluate(const double*) const { throw Unsupported("B200 platform: periodicdistance of constant arguments is not supported"); }
    double evaluateDerivative(const double*, const int*) const { throw Unsupported("B200 platform: periodicdistance of constant arguments is not supported"); }
    Lepton::CustomFunction* clone() const { return new PeriodicDistancePlaceholder(); }
};

// pointdistance, pointangle and pointdihedral of a CustomCompoundBondForce (6, 9 and 12 arguments), likewise: the device
// computes them (POINT_DIST, POINT_ANGLE, POINT_DIHEDRAL).
class PointFunctionPlaceholder : public Lepton::CustomFunction {
public:
    explicit PointFunctionPlaceholder(int numArguments) : numArguments(numArguments) {}
    int getNumArguments() const { return numArguments; }
    double evaluate(const double*) const { throw Unsupported("B200 platform: a point function of constant arguments is not supported"); }
    double evaluateDerivative(const double*, const int*) const { throw Unsupported("B200 platform: a point function of constant arguments is not supported"); }
    Lepton::CustomFunction* clone() const { return new PointFunctionPlaceholder(numArguments); }
private:
    int numArguments;
};

// One Lepton program as instructions.  Variables: variables[k] -> VAR k, or THETA for a torsion's "theta"; a per-term
// parameter -> PARAM (its index), a global parameter -> GLOBAL (its slot in globalSlot, the per-Context map shared by every
// custom force; a name seen for the first time gets the next slot).  Any other variable is an error, as on the Reference
// platform.  periodicdistance and its first derivatives -> PERIODIC_DIST, pointdistance / pointangle / pointdihedral and
// theirs -> POINT_DIST / POINT_ANGLE / POINT_DIHEDRAL (the parser knows these names only for the classes that have them).
// forceName names the class in messages; maxStack is the stack capacity of the class's interpreter.  tables (a custom nonbonded
// force's): the name of every discrete tabulated function -> (its table index, its number of arguments); it becomes DISCRETE1..3
// with the table as operand, any derivative of it DISCRETE with operand -1 (the value 0).
inline Program translateProgram(const Lepton::ExpressionProgram& prog, const std::vector<std::string>& variables, const std::string& forceName,
                                const std::vector<std::string>& paramNames, const std::vector<std::string>& globalNames,
                                std::map<std::string, int>& globalSlot, int maxStack = B200MD_CUSTOM_MAX_STACK,
                                const std::map<std::string, std::pair<int, int> >* tables = nullptr) {
    typedef Lepton::Operation Op;
    if (prog.getStackSize() > maxStack)
        throw Unsupported("B200 platform: a " + forceName + " expression needs a stack deeper than " + std::to_string(maxStack));
    if (prog.getNumOperations() > B200MD_CUSTOM_MAX_CODE)
        throw Unsupported("B200 platform: a " + forceName + " expression has more than 256 operations");
    Program out;
    for (int k = 0; k < prog.getNumOperations(); k++) {
        const Op& o = prog.getOperation(k);
        int code = -1, arg = 0;
        double imm = 0.0;
        switch (o.getId()) {
            case Op::CONSTANT: code = B200MD_OP_CONST; imm = dynamic_cast<const Op::Constant&>(o).getValue(); break;
            case Op::VARIABLE: {
                const std::string& name = o.getName();
                for (size_t v = 0; v < variables.size() && code < 0; v++)
                    if (variables[v] == name) { code = name == "theta" ? B200MD_OP_THETA : B200MD_OP_VAR; arg = (int) v; }
                for (size_t p = 0; p < paramNames.size() && code < 0; p++)
                    if (paramNames[p] == name) { code = B200MD_OP_PARAM; arg = (int) p; }
                for (size_t g = 0; g < globalNames.size() && code < 0; g++)
                    if (globalNames[g] == name) {
                        code = B200MD_OP_GLOBAL;
                        std::map<std::string, int>::iterator it = globalSlot.find(name);
                        if (it == globalSlot.end()) it = globalSlot.insert(std::make_pair(name, (int) globalSlot.size())).first;
                        arg = it->second;
                    }
                if (code < 0) throw OpenMM::OpenMMException("Unknown variable in expression: " + name);
                break;
            }
            case Op::CUSTOM: {
                const std::string& fn = o.getName();
                if (tables && tables->count(fn)) {
                    const std::pair<int, int>& t = tables->at(fn);
                    const std::vector<int>& order = dynamic_cast<const Op::Custom&>(o).getDerivOrder();
                    bool deriv = false;
                    for (int k : order) deriv = deriv || k != 0;
                    code = B200MD_OP_DISCRETE1 + t.second - 1;
                    arg = deriv ? -1 : t.first;
                    break;
                }
                code = fn == "periodicdistance" ? B200MD_OP_PERIODIC_DIST : fn == "pointdistance" ? B200MD_OP_POINT_DIST :
                       fn == "pointangle" ? B200MD_OP_POINT_ANGLE : fn == "pointdihedral" ? B200MD_OP_POINT_DIHEDRAL : -1;
                if (code < 0)
                    throw Unsupported("B200 platform: tabulated functions in a " + forceName + " expression are not supported");
                // getDerivOrder: all zero is the value, a single 1 the first derivative by that argument
                const std::vector<int>& order = dynamic_cast<const Op::Custom&>(o).getDerivOrder();
                int which = -1, total = 0;
                for (size_t k = 0; k < order.size(); k++) { total += order[k]; if (order[k] == 1) which = (int) k; }
                if (total > 1) throw Unsupported("B200 platform: second derivatives of " + fn + " are not supported");
                arg = total ? which : -1;
                break;
            }
            case Op::ADD: code = B200MD_OP_ADD; break;
            case Op::SUBTRACT: code = B200MD_OP_SUB; break;
            case Op::MULTIPLY: code = B200MD_OP_MUL; break;
            case Op::DIVIDE: code = B200MD_OP_DIV; break;
            case Op::POWER: code = B200MD_OP_POW; break;
            case Op::NEGATE: code = B200MD_OP_NEG; break;
            case Op::SQRT: code = B200MD_OP_SQRT; break;
            case Op::EXP: code = B200MD_OP_EXP; break;
            case Op::LOG: code = B200MD_OP_LOG; break;
            case Op::SIN: code = B200MD_OP_SIN; break;
            case Op::COS: code = B200MD_OP_COS; break;
            case Op::SEC: code = B200MD_OP_SEC; break;
            case Op::CSC: code = B200MD_OP_CSC; break;
            case Op::TAN: code = B200MD_OP_TAN; break;
            case Op::COT: code = B200MD_OP_COT; break;
            case Op::ASIN: code = B200MD_OP_ASIN; break;
            case Op::ACOS: code = B200MD_OP_ACOS; break;
            case Op::ATAN: code = B200MD_OP_ATAN; break;
            case Op::ATAN2: code = B200MD_OP_ATAN2; break;
            case Op::SINH: code = B200MD_OP_SINH; break;
            case Op::COSH: code = B200MD_OP_COSH; break;
            case Op::TANH: code = B200MD_OP_TANH; break;
            case Op::ERF: code = B200MD_OP_ERF; break;
            case Op::ERFC: code = B200MD_OP_ERFC; break;
            case Op::STEP: code = B200MD_OP_STEP; break;
            case Op::DELTA: code = B200MD_OP_DELTA; break;
            case Op::SQUARE: code = B200MD_OP_SQUARE; break;
            case Op::CUBE: code = B200MD_OP_CUBE; break;
            case Op::RECIPROCAL: code = B200MD_OP_RECIP; break;
            case Op::ADD_CONSTANT: code = B200MD_OP_ADD_CONST; imm = dynamic_cast<const Op::AddConstant&>(o).getValue(); break;
            case Op::MULTIPLY_CONSTANT: code = B200MD_OP_MUL_CONST; imm = dynamic_cast<const Op::MultiplyConstant&>(o).getValue(); break;
            case Op::POWER_CONSTANT: code = B200MD_OP_POW_CONST; imm = dynamic_cast<const Op::PowerConstant&>(o).getValue(); break;
            case Op::MIN: code = B200MD_OP_MIN; break;
            case Op::MAX: code = B200MD_OP_MAX; break;
            case Op::ABS: code = B200MD_OP_ABS; break;
            case Op::FLOOR: code = B200MD_OP_FLOOR; break;
            case Op::CEIL: code = B200MD_OP_CEIL; break;
            case Op::SELECT: code = B200MD_OP_SELECT; break;
        }
        if (code < 0) throw Unsupported("B200 platform: operation '" + o.getName() + "' in a " + forceName + " expression is not supported");
        out.op.push_back(code); out.arg.push_back(arg); out.imm.push_back(imm);
    }
    return out;
}

namespace detail {
// The energy program of a parsed expression and one derivative program per variable, in order (expr.differentiate(variable)
// .optimize()).  The global slots new names take are committed to globalSlot only when every program translates.
inline void translatePrograms(const Lepton::ParsedExpression& expr, const std::vector<std::string>& variables, const std::string& forceName,
                              int maxStack, const std::vector<std::string>& paramNames, const std::vector<std::string>& globalNames,
                              std::map<std::string, int>& globalSlot, std::vector<Program>& programs,
                              const std::map<std::string, std::pair<int, int> >* tables = nullptr) {
    std::map<std::string, int> slots = globalSlot;
    std::vector<Program> out(1, translateProgram(expr.createProgram(), variables, forceName, paramNames, globalNames, slots, maxStack, tables));
    for (const std::string& v : variables)
        out.push_back(translateProgram(expr.differentiate(v).optimize().createProgram(), variables, forceName, paramNames, globalNames, slots,
                                       maxStack, tables));
    programs.swap(out);
    globalSlot.swap(slots);
}
} // namespace detail

// The energy program and one derivative program per variable of one expression: Parser::parse(energy).optimize(), and the
// same expression .differentiate(variable).optimize() for every variable in order.  periodic: periodicdistance is a function
// of the expression (a CustomExternalForce).  perTerm names a term in messages ("torsion", "bond", "particle").
inline void translateExpression(const std::string& energy, const std::vector<std::string>& variables, const std::string& forceName,
                                const std::string& perTerm, bool periodic, const std::vector<std::string>& paramNames,
                                const std::vector<std::string>& globalNames, std::map<std::string, int>& globalSlot,
                                std::vector<Program>& programs) {
    if ((int) paramNames.size() > B200MD_CUSTOM_MAX_PARAMS)
        throw Unsupported("B200 platform: a " + forceName + " with more than 16 per-" + perTerm + " parameters is not supported");
    PeriodicDistancePlaceholder pd;
    std::map<std::string, Lepton::CustomFunction*> functions;
    if (periodic) functions["periodicdistance"] = &pd;
    detail::translatePrograms(Lepton::Parser::parse(energy, functions).optimize(), variables, forceName, B200MD_CUSTOM_MAX_STACK, paramNames,
                              globalNames, globalSlot, programs);
}

// A CustomCompoundBondForce: its energy program and the derivative programs by x1, y1, z1, x2, .. (1 + 3 particles per bond).
// CustomCompoundBondForceImpl::prepareExpression (libOpenMM.so) turns distance, angle and dihedral into the point functions, as
// for the Reference platform; the expression is then an ordinary function of the coordinates.
inline void translateCompound(const OpenMM::CustomCompoundBondForce& force, std::map<std::string, int>& globalSlot, std::vector<Program>& programs) {
    const int numParticles = force.getNumParticlesPerBond();
    if (numParticles > B200MD_CUSTOM_MAX_PARTICLES)
        throw Unsupported("B200 platform: a CustomCompoundBondForce with more than 8 particles per bond is not supported");
    if (force.getNumPerBondParameters() > B200MD_CUSTOM_MAX_PARAMS)
        throw Unsupported("B200 platform: a CustomCompoundBondForce with more than 16 per-bond parameters is not supported");
    if (force.getNumTabulatedFunctions() > 0)
        throw Unsupported("B200 platform: tabulated functions in a CustomCompoundBondForce expression are not supported");
    PointFunctionPlaceholder distance(6), angle(9), dihedral(12);
    std::map<std::string, Lepton::CustomFunction*> functions;
    functions["pointdistance"] = &distance; functions["pointangle"] = &angle; functions["pointdihedral"] = &dihedral;
    std::vector<std::string> variables, paramNames, globalNames;
    for (int i = 1; i <= numParticles; i++)
        for (const char* axis : {"x", "y", "z"}) variables.push_back(axis + std::to_string(i));
    for (int i = 0; i < force.getNumPerBondParameters(); i++) paramNames.push_back(force.getPerBondParameterName(i));
    for (int i = 0; i < force.getNumGlobalParameters(); i++) globalNames.push_back(force.getGlobalParameterName(i));
    detail::translatePrograms(OpenMM::CustomCompoundBondForceImpl::prepareExpression(force, functions), variables, "CustomCompoundBondForce",
                              B200MD_CUSTOM_COMPOUND_MAX_STACK, paramNames, globalNames, globalSlot, programs);
}

// A CustomCentroidBondForce: the programs of a compound bond of the same expression, by x1, y1, z1, x2, .. of the group
// centres (1 + 3 groups per bond).  CustomCentroidBondForceImpl::prepareExpression turns distance, angle and dihedral of
// g1, g2, .. into the point functions of those coordinates, as for the Reference platform.
inline void translateCentroid(const OpenMM::CustomCentroidBondForce& force, std::map<std::string, int>& globalSlot, std::vector<Program>& programs) {
    const int numGroups = force.getNumGroupsPerBond();
    if (numGroups > B200MD_CUSTOM_MAX_PARTICLES)
        throw Unsupported("B200 platform: a CustomCentroidBondForce with more than 8 groups per bond is not supported");
    if (force.getNumPerBondParameters() > B200MD_CUSTOM_MAX_PARAMS)
        throw Unsupported("B200 platform: a CustomCentroidBondForce with more than 16 per-bond parameters is not supported");
    if (force.getNumTabulatedFunctions() > 0)
        throw Unsupported("B200 platform: tabulated functions in a CustomCentroidBondForce expression are not supported");
    PointFunctionPlaceholder distance(6), angle(9), dihedral(12);
    std::map<std::string, Lepton::CustomFunction*> functions;
    functions["pointdistance"] = &distance; functions["pointangle"] = &angle; functions["pointdihedral"] = &dihedral;
    std::vector<std::string> variables, paramNames, globalNames;
    for (int i = 1; i <= numGroups; i++)
        for (const char* axis : {"x", "y", "z"}) variables.push_back(axis + std::to_string(i));
    for (int i = 0; i < force.getNumPerBondParameters(); i++) paramNames.push_back(force.getPerBondParameterName(i));
    for (int i = 0; i < force.getNumGlobalParameters(); i++) globalNames.push_back(force.getGlobalParameterName(i));
    detail::translatePrograms(OpenMM::CustomCentroidBondForceImpl::prepareExpression(force, functions), variables, "CustomCentroidBondForce",
                              B200MD_CUSTOM_COMPOUND_MAX_STACK, paramNames, globalNames, globalSlot, programs);
}

// The Discrete1D/2D/3DFunction tables of b200md_set_custom_tables: table t has dims[4t] dimensions of sizes dims[4t+1 ..]
// (unused ones 1) and the values [start[t], start[t+1]), x fastest.
struct Tables {
    std::vector<int> dims, start = std::vector<int>(1, 0);
    std::vector<double> values;
    int count() const { return (int) start.size() - 1; }
    void add(int ndim, int xsize, int ysize, int zsize, const std::vector<double>& v) {
        dims.insert(dims.end(), {ndim, xsize, ysize, zsize});
        values.insert(values.end(), v.begin(), v.end());
        start.push_back((int) values.size());
    }
};

// A CustomNonbondedForce: the energy program and dE/dr (VAR 0 = r), with p1 of per-particle parameter k as PARAM k and p2 as
// PARAM P+k (P parameters).  Its Discrete1D/2D/3DFunction tables are appended to `tables` and read by DISCRETE instructions;
// for parsing (and Lepton's constant folding) they are the Reference platform's functions, as in
// ReferenceCalcCustomNonbondedForceKernel::initialize.  Continuous functions are refused: they need splines on the device.
inline void translateNonbonded(const OpenMM::CustomNonbondedForce& force, std::map<std::string, int>& globalSlot, std::vector<Program>& programs,
                               Tables& tables) {
    const int numParams = force.getNumPerParticleParameters();
    if (numParams > B200MD_CUSTOM_MAX_PARAMS/2)
        throw Unsupported("B200 platform: a CustomNonbondedForce with more than 8 per-particle parameters is not supported");
    Tables mine = tables;
    std::map<std::string, std::pair<int, int> > index;
    for (int i = 0; i < force.getNumTabulatedFunctions(); i++) {
        const OpenMM::TabulatedFunction& f = force.getTabulatedFunction(i);
        std::vector<double> v;
        int xs = 1, ys = 1, zs = 1, nd = 0;
        if (const OpenMM::Discrete1DFunction* d = dynamic_cast<const OpenMM::Discrete1DFunction*>(&f)) { d->getFunctionParameters(v); xs = (int) v.size(); nd = 1; }
        else if (const OpenMM::Discrete2DFunction* d = dynamic_cast<const OpenMM::Discrete2DFunction*>(&f)) { d->getFunctionParameters(xs, ys, v); nd = 2; }
        else if (const OpenMM::Discrete3DFunction* d = dynamic_cast<const OpenMM::Discrete3DFunction*>(&f)) { d->getFunctionParameters(xs, ys, zs, v); nd = 3; }
        else throw Unsupported("B200 platform: continuous tabulated functions in a CustomNonbondedForce expression are not supported");
        index[force.getTabulatedFunctionName(i)] = std::make_pair(mine.count(), nd);
        mine.add(nd, xs, ys, zs, v);
    }
    std::map<std::string, Lepton::CustomFunction*> functions;
    for (int i = 0; i < force.getNumTabulatedFunctions(); i++)
        functions[force.getTabulatedFunctionName(i)] = createReferenceTabulatedFunction(force.getTabulatedFunction(i));
    std::vector<std::string> paramNames, globalNames;
    for (const char* suffix : {"1", "2"})
        for (int i = 0; i < numParams; i++) paramNames.push_back(force.getPerParticleParameterName(i) + suffix);
    for (int i = 0; i < force.getNumGlobalParameters(); i++) globalNames.push_back(force.getGlobalParameterName(i));
    try {
        detail::translatePrograms(Lepton::Parser::parse(force.getEnergyFunction(), functions).optimize(), {"r"}, "CustomNonbondedForce",
                                  B200MD_CUSTOM_MAX_STACK, paramNames, globalNames, globalSlot, programs, &index);
    } catch (...) {
        for (auto& f : functions) delete f.second;
        throw;
    }
    for (auto& f : functions) delete f.second;
    tables = mine;
}

} // namespace b200md_custom
#endif
