// custom_translate.h -- CustomTorsionForce expression -> the instruction programs of b200md_set_custom_torsions (B200MD_OP_*,
// include/b200md.h).  Lepton, part of the host's libOpenMM.so, parses, optimises and differentiates the expression exactly as
// the Reference platform does (ReferenceCalcCustomTorsionForceKernel::initialize, ReferenceKernels.cpp:807-809) and makes
// the stack program (ExpressionProgram); this file only maps every Lepton::Operation to one instruction.  Included by the
// plugin (B200Platform.cpp) and by its test C API (tests/custom_torsion_capi.cpp), so that both make the same programs.
#ifndef B200MD_CUSTOM_TRANSLATE_H_
#define B200MD_CUSTOM_TRANSLATE_H_
#include "openmm/OpenMMException.h"
#include "lepton/ExpressionProgram.h"
#include "lepton/Operation.h"
#include "lepton/ParsedExpression.h"
#include "lepton/Parser.h"
#include "../include/b200md.h"
#include <map>
#include <string>
#include <vector>

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

// One Lepton program as instructions.  Variables: "theta" -> THETA, a per-torsion parameter -> PARAM (its index), a global
// parameter -> GLOBAL (its slot in globalSlot, the per-Context map shared by every CustomTorsionForce; a name seen for the
// first time gets the next slot).  Any other variable is an error, as on the Reference platform.
inline Program translateProgram(const Lepton::ExpressionProgram& prog, const std::vector<std::string>& paramNames,
                                const std::vector<std::string>& globalNames, std::map<std::string, int>& globalSlot) {
    typedef Lepton::Operation Op;
    if (prog.getStackSize() > B200MD_CUSTOM_MAX_STACK)
        throw Unsupported("B200 platform: a CustomTorsionForce expression needs a stack deeper than 16");
    if (prog.getNumOperations() > B200MD_CUSTOM_MAX_CODE)
        throw Unsupported("B200 platform: a CustomTorsionForce expression has more than 256 operations");
    Program out;
    for (int k = 0; k < prog.getNumOperations(); k++) {
        const Op& o = prog.getOperation(k);
        int code = -1, arg = 0;
        double imm = 0.0;
        switch (o.getId()) {
            case Op::CONSTANT: code = B200MD_OP_CONST; imm = dynamic_cast<const Op::Constant&>(o).getValue(); break;
            case Op::VARIABLE: {
                const std::string& name = o.getName();
                if (name == "theta") { code = B200MD_OP_THETA; break; }
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
            case Op::CUSTOM: throw Unsupported("B200 platform: tabulated functions in a CustomTorsionForce expression are not supported");
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
        if (code < 0) throw Unsupported("B200 platform: operation '" + o.getName() + "' in a CustomTorsionForce expression is not supported");
        out.op.push_back(code); out.arg.push_back(arg); out.imm.push_back(imm);
    }
    return out;
}

// The energy program and the dE/dtheta program of one expression: Parser::parse(energy).optimize(), and the same expression
// .differentiate("theta").optimize().
inline void translateExpression(const std::string& energy, const std::vector<std::string>& paramNames,
                                const std::vector<std::string>& globalNames, std::map<std::string, int>& globalSlot,
                                Program& energyProgram, Program& derivProgram) {
    if ((int) paramNames.size() > B200MD_CUSTOM_MAX_PARAMS)
        throw Unsupported("B200 platform: a CustomTorsionForce with more than 16 per-torsion parameters is not supported");
    const Lepton::ParsedExpression expr = Lepton::Parser::parse(energy).optimize();
    std::map<std::string, int> slots = globalSlot;      // committed only when both programs translate
    energyProgram = translateProgram(expr.createProgram(), paramNames, globalNames, slots);
    derivProgram = translateProgram(expr.differentiate("theta").optimize().createProgram(), paramNames, globalNames, slots);
    globalSlot.swap(slots);
}

} // namespace b200md_custom
#endif
