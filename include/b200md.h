/* b200md.h -- the C-ABI of the CUDA-native (sm_90a) OpenMM hot path (libb200md.so).
 *
 * This is the drop-in boundary.  Plain pointers and sizes only: no C++ types, no torch types.  Every entry
 * point replaces one method of the reference's abstract kernel interfaces (olla/include/openmm/kernels.h in
 * pandegroup/openmm 7.6-dev); the OpenMM Platform plugin (plugin/, libOpenMMB200.so) is a thin C++ adapter that
 * forwards those virtual methods to the functions below, and the Python host mirror (openmm_b200/) binds the same
 * functions through ctypes.  Units follow OpenMM: nm, ps, amu, kJ/mol, elementary charges, Kelvin.
 *
 * All functions return 0 on success and a negative code on failure; b200md_last_error() gives the message
 * (the plugin turns it into an OpenMMException, OpenMMException.h).  There is NO CPU fallback anywhere:
 * if the CUDA device or kernels are unavailable every call fails loudly.
 *
 * Host arrays are caller-owned, double precision, atom-major ([natoms][3]) in the USER's atom order; the
 * engine keeps its own device-resident, spatially sorted fp32/fixed-point state.
 */
#ifndef B200MD_H_
#define B200MD_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200md_ctx b200md_ctx;

/* ---- NonbondedForce::NonbondedMethod (openmmapi/include/openmm/NonbondedForce.h:114-143) ---- */
#define B200MD_NB_NOCUTOFF            0
#define B200MD_NB_CUTOFF_NONPERIODIC  1
#define B200MD_NB_CUTOFF_PERIODIC     2
#define B200MD_NB_EWALD               3   /* not implemented: b200md_set_nonbonded fails */
#define B200MD_NB_PME                 4
#define B200MD_NB_LJPME               5   /* not implemented */

/* ---- which terms b200md_compute evaluates (force groups are mapped onto these by the plugin) ---- */
#define B200MD_TERM_BONDS      1
#define B200MD_TERM_ANGLES     2
#define B200MD_TERM_TORSIONS   4
#define B200MD_TERM_NB_DIRECT  8    /* includeDirect  of CalcNonbondedForceKernel::execute (kernels.h:588) */
#define B200MD_TERM_NB_RECIP   16   /* includeReciprocal */
#define B200MD_TERM_RB_TORSIONS 32
#define B200MD_TERM_CMAP       64
#define B200MD_TERM_CUSTOM_TORSIONS 128
#define B200MD_TERM_ALL        255

/* ---- the bonded classes: kind argument of b200md_set_bonded_groups and b200md_update_bonded_params ---- */
#define B200MD_BONDED_BONDS           0
#define B200MD_BONDED_ANGLES          1
#define B200MD_BONDED_TORSIONS        2
#define B200MD_BONDED_RB_TORSIONS     3
#define B200MD_BONDED_CMAP            4
#define B200MD_BONDED_CUSTOM_TORSIONS 5

/* ---- instructions of a custom-torsion expression program (b200md_set_custom_torsions) ----
 * One instruction = (opcode, operand index, double immediate).  A program is the flat stack program of a Lepton
 * ExpressionProgram (lepton/ExpressionProgram.h), one instruction per Lepton::Operation, in the same order and with the same
 * argument order: an operation of k arguments reads them from the top of the stack, argument 0 being the value pushed LAST,
 * and replaces them with its result (ExpressionProgram::evaluate).  Each opcode computes exactly what the Operation of the
 * same name computes.  THETA pushes the dihedral in (-pi, pi], PARAM k the term's k-th parameter, GLOBAL s the context's
 * global value in slot s; CONST, ADD_CONST, MUL_CONST and POW_CONST take their constant from the immediate. */
enum {
    B200MD_OP_CONST = 0, B200MD_OP_THETA, B200MD_OP_PARAM, B200MD_OP_GLOBAL,
    B200MD_OP_ADD, B200MD_OP_SUB, B200MD_OP_MUL, B200MD_OP_DIV, B200MD_OP_POW, B200MD_OP_NEG, B200MD_OP_SQRT, B200MD_OP_EXP,
    B200MD_OP_LOG, B200MD_OP_SIN, B200MD_OP_COS, B200MD_OP_SEC, B200MD_OP_CSC, B200MD_OP_TAN, B200MD_OP_COT, B200MD_OP_ASIN,
    B200MD_OP_ACOS, B200MD_OP_ATAN, B200MD_OP_ATAN2, B200MD_OP_SINH, B200MD_OP_COSH, B200MD_OP_TANH, B200MD_OP_ERF,
    B200MD_OP_ERFC, B200MD_OP_STEP, B200MD_OP_DELTA, B200MD_OP_SQUARE, B200MD_OP_CUBE, B200MD_OP_RECIP, B200MD_OP_ADD_CONST,
    B200MD_OP_MUL_CONST, B200MD_OP_POW_CONST, B200MD_OP_MIN, B200MD_OP_MAX, B200MD_OP_ABS, B200MD_OP_FLOOR, B200MD_OP_CEIL,
    B200MD_OP_SELECT,
    B200MD_OP_COUNT
};
/* hard limits of a custom-torsion program: stack depth, instructions per program, parameters per term */
#define B200MD_CUSTOM_MAX_STACK  16
#define B200MD_CUSTOM_MAX_CODE   256
#define B200MD_CUSTOM_MAX_PARAMS 16

/* ---- integrators (kernels.h:1033-1060 Verlet, :1160-1188 Langevin, :1192-1220 LangevinMiddle) ---- */
#define B200MD_INT_VERLET          0
#define B200MD_INT_LANGEVIN        1
#define B200MD_INT_LANGEVIN_MIDDLE 2

typedef struct b200md_nonbonded_desc {
    int    method;               /* B200MD_NB_*                                                         */
    double cutoff;               /* NonbondedForce::getCutoffDistance                                    */
    int    use_switch;           /* getUseSwitchingFunction                                              */
    double switch_distance;      /* getSwitchingDistance                                                 */
    double rf_dielectric;        /* getReactionFieldDielectric (CutoffPeriodic / CutoffNonPeriodic)      */
    double ewald_alpha;          /* PME: alpha from NonbondedForceImpl::calcPMEParameters (:144-184)     */
    int    grid[3];              /* PME grid; each dim must factor into radices <= 16 (see DESIGN.md)    */
    double dispersion_coefficient; /* NonbondedForceImpl::calcDispersionCorrection (:236-310); 0 = off   */
    int    exceptions_periodic;  /* getExceptionsUsePeriodicBoundaryConditions                           */
} b200md_nonbonded_desc;

/* ---------------------------------------------------------------------------------------------------
 * Life cycle.  Replaces Platform::contextCreated / contextDestroyed (olla/include/openmm/Platform.h)
 * and the per-Context PlatformData of the reference CUDA platform (CudaPlatform.cpp:232-257).        */
int  b200md_create(b200md_ctx** out, int device, int natoms);
void b200md_destroy(b200md_ctx* ctx);
const char* b200md_last_error(const b200md_ctx* ctx);      /* ctx may be NULL: error of the last failed create */
const char* b200md_version(void);

/* ---------------------------------------------------------------------------------------------------
 * System definition (all before b200md_finalize).                                                    */
/* System::getParticleMass; mass 0 = immovable particle (ReferenceStochasticDynamics.cpp:101).       */
int b200md_set_masses(b200md_ctx* ctx, const double* mass);
/* CalcNonbondedForceKernel::initialize (kernels.h:577): per-particle charge, sigma, epsilon.         */
int b200md_set_nonbonded(b200md_ctx* ctx, const b200md_nonbonded_desc* desc,
                         const double* charge, const double* sigma, const double* epsilon);
/* NonbondedForce exceptions: EVERY exception is an exclusion; those with chargeProd != 0 or eps != 0
 * are additionally evaluated as 1-4 pairs (ReferenceKernels.cpp:885-895).                            */
int b200md_set_exceptions(b200md_ctx* ctx, int n, const int* p1, const int* p2,
                          const double* charge_prod, const double* sigma, const double* epsilon);
/* CalcHarmonicBondForceKernel::initialize (kernels.h:289), E = k/2 (r-r0)^2.                         */
int b200md_set_bonds(b200md_ctx* ctx, int n, const int* p1, const int* p2, const double* length, const double* k);
/* CalcHarmonicAngleForceKernel::initialize (kernels.h:359), E = k/2 (theta-theta0)^2.                */
int b200md_set_angles(b200md_ctx* ctx, int n, const int* p1, const int* p2, const int* p3, const double* angle, const double* k);
/* CalcPeriodicTorsionForceKernel::initialize (kernels.h:429), E = k (1+cos(n phi - phase)).          */
int b200md_set_torsions(b200md_ctx* ctx, int n, const int* p1, const int* p2, const int* p3, const int* p4,
                        const int* periodicity, const double* phase, const double* k);
/* CalcRBTorsionForceKernel::initialize (kernels.h:464), E = sum_{n=0..5} c[i][n] cos^n(phi - pi).                 */
int b200md_set_rb_torsions(b200md_ctx* ctx, int n, const int* p1, const int* p2, const int* p3, const int* p4, const double* c);
/* CalcCMAPTorsionForceKernel::initialize (kernels.h:499): nmaps maps of size[m] x size[m] points, given as the bicubic
 * spline coefficients of CMAPTorsionForceImpl::calcMapDerivatives, maps one after the other, [size^2 patches][16] each;
 * n terms, term i uses map[i] and the two dihedrals atoms[i][0..3] and atoms[i][4..7].                                */
int b200md_set_cmap(b200md_ctx* ctx, int nmaps, const int* size, const double* coeff, int n, const int* map, const int* atoms);
/* CalcCustomTorsionForceKernel::initialize (kernels.h:521): nprog expressions as instruction programs (B200MD_OP_*), program
 * 2p the energy of expression p and program 2p+1 its derivative dE/dtheta; program q is the instructions
 * [prog_start[q], prog_start[q+1]) of op / arg / imm (prog_start has 2*nprog+1 entries).  n terms: term i evaluates
 * expression prog[i] on the dihedral atoms[4i..4i+3] with the parameters params[i*param_stride ..].  Every program is
 * checked here (opcodes, operand indices, the stack simulated on the host); GLOBAL operands are checked against the number
 * of global values at finalize.  Single GPU only.                                                                        */
int b200md_set_custom_torsions(b200md_ctx* ctx, int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                               int param_stride, int n, const int* prog, const int* atoms, const double* params);
/* The global parameter values the GLOBAL instructions read (slot s = values[s]).  Before finalize it sets the number of
 * slots; after it, a stream-ordered copy of n == that number of values into the same device buffer, so a captured step
 * graph keeps running with the new values and is never instantiated again.                                               */
int b200md_set_custom_globals(b200md_ctx* ctx, int n, const double* values);
/* Force group (Force::getForceGroup, openmmapi/include/openmm/Force.h) of every bonded term, so that
 * several Force objects of one class may live in different groups (ContextImpl::calcForcesAndEnergy,
 * ContextImpl.cpp:293-308; tests/TestLocalEnergyMinimizer.h:234 testForceGroups).  kind: B200MD_BONDED_*; default
 * group 0.  group[i] | 0x80 marks a term of a Force with usesPeriodicBoundaryConditions(): its
 * difference vectors take the minimum image (ReferenceForce::getDeltaRPeriodic, ReferenceForce.cpp:90-101).          */
int b200md_set_bonded_groups(b200md_ctx* ctx, int kind, int n, const int* group);
/* System::getConstraintParameters; supported topologies: 3-atom rigid molecules (SETTLE,
 * ReferenceConstraints.cpp:69-146) and X-H_n clusters, n<=3 (SHAKE, common IntegrationUtilities.cpp:204-277). */
int b200md_set_constraints(b200md_ctx* ctx, int n, const int* p1, const int* p2, const double* distance);
/* Dry run of the constraint classification, without a context or a device: 0 if every constraint is supported, else -1
 * with the reason in msg.  Platform::contextCreated calls it so that an unsupported System is refused THERE, where
 * ContextImpl can still fall back to another platform (ContextImpl.cpp:152-166).                                      */
int b200md_check_constraints(int natoms, const double* mass, int n, const int* p1, const int* p2, const double* distance,
                             char* msg, int msglen);
/* The host half of the CCMA setup (ReferenceCCMAAlgorithm's constructor, ReferenceCCMAAlgorithm.cpp:42-202), without a
 * context or a device: which constraints form general networks, their connected components, and the approximate inverse of
 * the coupling matrix in CSR form (angles = the HarmonicAngleForce terms, as ReferenceConstraints.cpp:163-177 collects
 * them).  out_order[k] = index, in the caller's arrays, of CCMA constraint k (component by component); row_start has
 * *out_nccma + 1 entries.  Returns the number of non-zeros, -2 if cap is too small, -1 on error.  Test hook.            */
int b200md_ccma_setup_probe(int natoms, const double* mass, int ncon, const int* p1, const int* p2, const double* distance,
                            int nangles, const int* a1, const int* a2, const int* a3, const double* theta0,
                            int* out_ncomp, int* out_nccma, int* out_order, int* row_start, int* col, float* val, int cap);
/* RemoveCMMotionKernel (kernels.h:1464-1483); frequency <= 0 disables.                               */
int b200md_set_cm_remover(b200md_ctx* ctx, int frequency);
/* RemoveCMMotionKernel::execute (kernels.h:1483): subtract the centre-of-mass velocity now.          */
int b200md_remove_cm_motion(b200md_ctx* ctx);
/* Precision of the integration state (the Precision platform property).  SINGLE (default): fp32 positions and velocities.
 * MIXED: positions kept as fp32 hi + fp32 lo (about 48 bits), velocities, integration and constraints in double; the force
 * kernels read the fp32 hi part either way.  Before b200md_finalize, single-GPU contexts only (not after b200md_comm_init
 * with world > 1, not on a b200md_pme_create context).                                                                   */
#define B200MD_PRECISION_SINGLE 0
#define B200MD_PRECISION_MIXED  1
int b200md_set_precision(b200md_ctx* ctx, int precision);
int b200md_get_precision(b200md_ctx* ctx);      /* B200MD_PRECISION_*, or -1 for a NULL context */
/* Build exclusion lists, constraint clusters, PME plans; allocate the device state.                  */
int b200md_finalize(b200md_ctx* ctx);
/* CalcNonbondedForceKernel::copyParametersToContext (kernels.h:595), after finalize.                 */
int b200md_update_nonbonded_params(b200md_ctx* ctx, const double* charge, const double* sigma, const double* epsilon,
                                   int nexc, const double* exc_charge_prod, const double* exc_sigma, const double* exc_epsilon,
                                   double dispersion_coefficient);

/* Calc{HarmonicBond,HarmonicAngle,PeriodicTorsion}ForceKernel::copyParametersToContext (kernels.h:305,375,445):
 * same topology, new parameters. kind B200MD_BONDED_BONDS (a=length,b=k), _ANGLES (a=angle,b=k), _TORSIONS (a=phase,b=k). */
int b200md_update_bonded_params(b200md_ctx* ctx, int kind, int n, const double* a, const double* b, const int* periodicity);
/* CalcRBTorsionForceKernel::copyParametersToContext (kernels.h:480): same torsions, new c[n][6].                     */
int b200md_update_rb_torsion_params(b200md_ctx* ctx, int n, const double* c);
/* CalcCMAPTorsionForceKernel::copyParametersToContext (kernels.h:515): same number of maps and map sizes, same terms
 * (atoms); new coefficients and new map index per term.                                                              */
int b200md_update_cmap_params(b200md_ctx* ctx, int nmaps, const int* size, const double* coeff, int n, const int* map);
/* CalcCustomTorsionForceKernel::copyParametersToContext (kernels.h:544): same terms, same program per term, new parameters
 * params[n][param_stride], written into the same device buffers.                                                         */
int b200md_update_custom_torsion_params(b200md_ctx* ctx, int n, const double* params);
/* Test hook, no context and no device: program `which` of a b200md_set_custom_torsions program set, checked as that call
 * checks it (nglobals = the number of global slots), evaluated at (theta, params, globals) on the host by the interpreter
 * source the device kernel runs.  0 and *out on success, -1 with the reason in msg.                                       */
int b200md_custom_program_probe(int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                                int param_stride, int nglobals, int which, double theta, const double* params,
                                const double* globals, double* out, char* msg, int msglen);

/* ---------------------------------------------------------------------------------------------------
 * UpdateStateDataKernel (kernels.h:125-214).                                                         */
int b200md_set_box(b200md_ctx* ctx, const double a[3], const double b[3], const double c[3]);
int b200md_get_box(b200md_ctx* ctx, double a[3], double b[3], double c[3]);

/* ---------------------------------------------------------------------------------------------------
 * ApplyMonteCarloBarostatKernel (kernels.h:1425-1459), for MonteCarloBarostat and MonteCarloAnisotropicBarostat.  The host
 * half (MonteCarloBarostatImpl) stays the caller's: it evaluates the energy, calls b200md_scale_coordinates, sets the scaled
 * box with b200md_set_box, evaluates again and on rejection calls b200md_restore_coordinates and sets the old box.  One rank
 * only: all three fail in a multi-GPU context.                                                        */
/* ApplyMonteCarloBarostatKernel::initialize: the molecules of ContextImpl::getMolecules(), in that order, as CSR
 * (start[nmol+1], atoms[start[nmol]]).                                                                */
int b200md_set_barostat_molecules(b200md_ctx* ctx, int nmol, const int* start, const int* atoms);
/* ApplyMonteCarloBarostatKernel::scaleCoordinates: save the positions and the force buffer, then move every molecule's centre
 * into the first periodic box of the CURRENT box and scale it by (sx, sy, sz) (ReferenceMonteCarloBarostat.cpp:67-103).
 * b200md_get_positions then returns the wrapped, scaled coordinates.                                  */
int b200md_scale_coordinates(b200md_ctx* ctx, double sx, double sy, double sz);
/* ApplyMonteCarloBarostatKernel::restoreCoordinates: positions and forces as before the last scale, bit for bit. */
int b200md_restore_coordinates(b200md_ctx* ctx);
int b200md_set_positions(b200md_ctx* ctx, const double* xyz);
int b200md_get_positions(b200md_ctx* ctx, double* xyz);   /* continuous (unwrapped) trajectory, like the Reference platform's:
                                                             * internal molecule wrapping is undone (DESIGN.md section 4, "Long runs") */
int b200md_set_velocities(b200md_ctx* ctx, const double* xyz);
int b200md_get_velocities(b200md_ctx* ctx, double* xyz);
int b200md_get_forces(b200md_ctx* ctx, double* xyz);        /* forces of the last b200md_compute.  b200md_step zeroes the force
                                                             * buffer inside its fused integrate kernel: after a step the
                                                             * forces (and the half-step-shifted kinetic energy of the
                                                             * leapfrog integrators, which needs them) are only valid after
                                                             * another b200md_compute -- Context::getState does exactly that */
int b200md_set_time(b200md_ctx* ctx, double t);
double b200md_get_time(b200md_ctx* ctx);
int64_t b200md_get_step_count(b200md_ctx* ctx);
/* createCheckpoint / loadCheckpoint (kernels.h:208-214): opaque blob; size query with buf == NULL.  A blob is loaded only
 * into a context of the precision that wrote it.                                                     */
int64_t b200md_checkpoint_save(b200md_ctx* ctx, void* buf, int64_t capacity);
int b200md_checkpoint_load(b200md_ctx* ctx, const void* buf, int64_t size);

/* ---------------------------------------------------------------------------------------------------
 * CalcForcesAndEnergyKernel::beginComputation/finishComputation + every Calc*ForceKernel::execute
 * (kernels.h:81-118, :298, :368, :438, :588) in one call: zero the force buffer, (re)build the tile
 * neighbour list if any atom moved more than half the padding, evaluate the selected terms.
 * energy (may be NULL) receives the potential energy of the selected terms.                          */
int b200md_compute(b200md_ctx* ctx, int terms, int want_forces, double* energy);
/* the same with the `groups` bit mask of CalcForcesAndEnergyKernel::beginComputation (kernels.h:96): a bond / angle /
 * torsion is evaluated iff its class is in `terms` AND bit (its force group) of bonded_group_mask is set.            */
int b200md_compute_groups(b200md_ctx* ctx, int terms, unsigned int bonded_group_mask, int want_forces, double* energy);

/* ---------------------------------------------------------------------------------------------------
 * Integrate*StepKernel::initialize/execute/computeKineticEnergy (kernels.h:1033-1060, 1160-1220),
 * ApplyConstraintsKernel::apply/applyToVelocities (kernels.h:220-246).                              */
int b200md_set_integrator(b200md_ctx* ctx, int kind, double dt, double temperature, double friction,
                          int seed, double constraint_tol);
/* n full MD steps (forces + integrate + constraints), enqueued as CUDA graphs with no host sync.     */
int b200md_step(b200md_ctx* ctx, int nsteps);
/* the integrator half only (the plugin calls b200md_compute itself via ContextImpl::calcForcesAndEnergy) */
int b200md_integrate_only(b200md_ctx* ctx);
int b200md_kinetic_energy(b200md_ctx* ctx, double* ke);
int b200md_apply_constraints(b200md_ctx* ctx, double tol);
int b200md_apply_velocity_constraints(b200md_ctx* ctx, double tol);
int b200md_synchronize(b200md_ctx* ctx);

/* ---------------------------------------------------------------------------------------------------
 * Multi-GPU (one process per GPU).  The caller creates an NCCL unique id on rank 0 (b200md_comm_unique_id),
 * broadcasts the 128 bytes by any means (torch.distributed in bench.py) and hands it to every rank.
 * mode 0: replicated atoms, tile list and PME atoms sharded, one int64 all-reduce of the forces per step. */
int b200md_comm_unique_id(void* id128);
/* Test hook, no context and no device: the ownership cuts b200md_finalize makes for `world` ranks (atom_lo, unit_lo: world + 1
 * entries; rank q owns the atoms [atom_lo[q], atom_lo[q+1]) = whole integration units).  Returns the number of units.   */
int b200md_ownership_probe(int natoms, const double* mass, int ncon, const int* p1, const int* p2, const double* distance,
                           int world, int* atom_lo, int* unit_lo);
int b200md_comm_init(b200md_ctx* ctx, int rank, int world, const void* id128);

/* ---------------------------------------------------------------------------------------------------
 * Introspection for tests, bench and roofline accounting.                                            */
typedef struct b200md_stats {
    int64_t natoms, padded_atoms, num_blocks;
    int64_t num_tiles;            /* 32x32 tiles in the current neighbour list                 */
    int64_t num_mask_tiles;       /* tiles carrying an exclusion / validity mask               */
    int64_t list_builds;          /* neighbour-list rebuilds so far                            */
    int64_t force_evals;          /* b200md_compute + b200md_step evaluations                   */
    int64_t kernel_launches;      /* kernels launched (or replayed inside graphs) so far        */
    int64_t pairs_in_cutoff;      /* filled by b200md_count_pairs (diagnostic kernel)           */
    int     pme_grid[3];
    double  ewald_alpha;
    int     overflow;             /* sticky: tile capacity exceeded at some point               */
    int64_t graph_instantiations; /* executable step graphs instantiated so far (a box change updates them in place) */
} b200md_stats;
int b200md_get_stats(b200md_ctx* ctx, b200md_stats* out);
/* mean device time (ms) of named phases measured with CUDA events on the engine's stream:
 * phase: 0 pair kernel, 1 pme spread, 2 fft+convolution, 3 pme gather, 4 integrate+constrain, 5 list build,
 * 6 bonded+exceptions (k_bonded and, with custom torsions, k_custom_torsion), 7 custom torsions alone (k_custom_torsion).
 * Runs `reps` isolated launches of that phase on the current state.                                  */
int b200md_time_phase(b200md_ctx* ctx, int phase, int reps, double* ms_mean);
/* stand-alone 3-D FFT entry (the bespoke FFT alone, for parity against fftpack / numpy):
 * in: real [nx][ny][nz] floats (host), out: complex [nx][ny][nz/2+1] (re,im) floats (host).          */
int b200md_fft3d_r2c(int device, int nx, int ny, int nz, const float* in, float* out);
int b200md_fft3d_c2r(int device, int nx, int ny, int nz, const float* in, float* out);
void* b200md_cuda_stream(b200md_ctx* ctx);

/* ---------------------------------------------------------------------------------------------------
 * Stand-alone reciprocal-space PME (SURVEY.md 8f rank 3): the narrow drop-in behind the reference's
 * CalcPmeReciprocalForceKernel (olla/include/openmm/kernels.h:1493-1557), the hook through which the CPU platform
 * (CpuKernels.cpp:620-690) and the CUDA platform (CudaKernels.cpp:746-760, UseCpuPme) outsource reciprocal space to
 * plugins/cpupme.  plugin/libOpenMMB200Pme.so registers a kernel of that name that forwards to these two calls.
 *   create: CalcPmeReciprocalForceKernel::initialize(gridx, gridy, gridz, numParticles, alpha, deterministic);
 *           every grid dimension must factor into radices <= 13 (the caller rounds up, as cpupme does);
 *   exec:   beginComputation + finishComputation: posq = [natoms][4] floats (x, y, z, charge in e: IO::getPosq),
 *           box = the three periodic box vectors row by row, force4 = [natoms][4] floats (IO::setForce layout, 4th
 *           element untouched), *energy = reciprocal-space energy WITHOUT the Ewald self term (as cpupme returns it).
 * Destroy with b200md_destroy.                                                                       */
int b200md_pme_create(b200md_ctx** out, int device, int natoms, int nx, int ny, int nz, double alpha);
int b200md_pme_exec(b200md_ctx* ctx, const float* posq, const double box[9], int include_energy, float* force4, double* energy);

#ifdef __cplusplus
}
#endif
#endif
