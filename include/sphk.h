/* sphk.h -- C-ABI of the native SPH kernel library (libsphk.so, H100: sm_90a).
 *
 * The reference (zhai-xiao/CPP-Fluid-Particles) has no FFI/plugin boundary: its boundary is the C++
 * class API SPHSystem / BaseSolver / SPHParticles / DArray compiled into one executable.  This
 * header is the boundary a maintainer binds to: ONE entry point per reference launch site on the
 * hot path SPHSystem::step() (each declaration cites the reference code it replaces, paths relative
 * to /root/reference/src).  The reference-shaped C++ classes in cpp-fluid-particles_b200/host/ are
 * written purely on top of these calls (see INTEGRATION.md).
 *
 * Conventions
 *  - Plain C: raw DEVICE pointers, ints, floats, PODs.  No torch / thrust / C++ types.
 *  - "float3 arrays" are packed xyz triplets, 12-byte stride, exactly the reference's float3 DArrays.
 *  - Every function returns 0 on success or a negative SPHK_ERR_* / positive cudaError_t value, and
 *    never throws.  Nothing synchronises the host unless stated (the reference syncs on every Thrust
 *    call; here only sphk_reduce_abs_sum and sphk_synchronize do).
 *  - All work is enqueued on the stream given to sphk_create (a cudaStream_t passed as void*).
 *  - There is NO CPU fallback: without a CUDA device sphk_create fails with SPHK_ERR_NO_DEVICE.
 *  - The library never allocates or frees API-visible arrays; sphk_ctx owns only scratch (sort
 *    buffers, packed 32-byte particle records, neighbour lists).
 *
 * Record coherence rule: sphk_neighbor_search() packs the particle set into 32-byte records
 * {x,y,z,s | vx,vy,vz,m} that the sweep kernels gather; every sphk_* call that changes pos / vel writes
 * both the API array and the record.  If the caller edits pos / vel itself between calls it must call
 * sphk_neighbor_search (or sphk_refresh) before the next sweep.  A scalar array passed to a sweep that
 * gathers it from neighbours (stiffness, lambda) is mirrored into the records unless the previous sphk_*
 * call produced it; arrays modified behind the library's back need sphk_refresh.
 */
#ifndef SPHK_H_
#define SPHK_H_

#ifdef __cplusplus
extern "C" {
#endif

#define SPHK_VERSION 1

enum {
    SPHK_OK = 0,
    SPHK_ERR_INVALID = -1,    /* bad argument */
    SPHK_ERR_NO_DEVICE = -2,  /* no CUDA device / driver: there is no CPU path */
    SPHK_ERR_CAPACITY = -3,   /* n exceeds the capacity given to sphk_create */
    SPHK_ERR_STATE = -4,      /* call order violated (e.g. sweep before neighbour search) */
    SPHK_ERR_ALLOC = -5,
    SPHK_ERR_COMM = -6        /* multi-GPU: NCCL missing / failed, or a neighbour's message did not arrive */
};

typedef struct sphk_ctx sphk_ctx;

/* Uniform grid, CUDAFunctions.cuh:64-78: cell (x,y,z) -> (x*cs.y + y)*cs.z + z, z fastest. */
typedef struct sphk_grid {
    int   cell_size[3];
    float cell_length;
    int   origin[3];   /* cell coordinates of this context's cell (0,0,0) in the global grid: all zero for a
                          single-GPU system; a slab rank covers global x-planes [origin[0], origin[0]+cell_size[0]) */
} sphk_grid;

/* One SPHParticles object (SPHParticles.h:56-59 + Particles.h:47-48): device pointers. */
typedef struct sphk_particles {
    float* pos;            /* float3[n]   getPosPtr()          */
    float* vel;            /* float3[n]   getVelPtr()  (NULL allowed for boundaries) */
    float* mass;           /* float[n]    getMassPtr()         */
    float* density;        /* float[n]    getDensityPtr()      */
    float* pressure;       /* float[n]    getPressurePtr()     */
    int*   particle2cell;  /* int[n]      getParticle2Cell()   */
    int    n;
} sphk_particles;

/* What every solver step receives (BaseSolver.h:22-26): both particle sets + their cell ranges. */
typedef struct sphk_scene {
    sphk_particles fluid;
    sphk_particles boundary;
    const int* cell_start_fluid;     /* int[ncells+1] */
    const int* cell_start_boundary;  /* int[ncells+1] */
    float radius;                    /* sphSmoothingRadius */
} sphk_scene;

enum {
    SPHK_OPT_NEIGHBOR_LIST = 1,  /* 1: sweeps walk a per-step neighbour list while positions are
                                    unchanged since the search (WCSPH, DFSPH); 0: always walk the
                                    27 cells.  default 1 */
    SPHK_OPT_LIST_CAPACITY = 2,  /* max neighbours kept per particle; particles with more fall back
                                    to the cell walk individually.  A multiple of 4 in [8, 1024], for the int32 lists and
                                    the tile lists alike (a tile list is padded to whole 8-slot batches).  default 96 */
    SPHK_OPT_STAGED_LIST_BUILD = 10, /* 1 (default): the list builder stages each tile's 9 + 9 candidate windows in shared memory
                                    (cp.async.bulk + mbarrier) and tests candidates from there; 0: candidates read from global memory */
    SPHK_OPT_PATCH = 11,         /* experiment (default 0 = off): S > 0 makes the 4 warps of a list-sweep block take their
                                    32-particle chunks from 4 runs that lie S chunks apart in the sorted order instead of 4
                                    consecutive chunks -- with S = chunks per cell column, a block covers 4 adjacent columns x 4 cells
                                    in z, a smaller neighbour footprint per block (L1 reuse).  Results are unchanged. */
    SPHK_OPT_SIMPLE_LIST_BUILD = 6, /* 1: build the list with the generic cell walk (reference for the tuned builder) */
    SPHK_OPT_LIST_SKIN = 5,      /* neighbour-list skin in 1/1000 of the radius (default 0).  With a skin the list
                                    stays valid while sphk_pbd_delta_pos_apply moves particles by less than skin/2
                                    (tracked on the device; beyond that every sweep falls back to the cell walk) */
    SPHK_OPT_TILE = 9            /* 1: tile lists.  A tile = 128 consecutive particles; the particles any of them can interact
                                    with lie in 9 + 9 contiguous windows of the sorted fluid / boundary records
                                    (CUDAFunctions.cuh:68: z is the fastest cell dimension), which every sweep stages into
                                    shared memory with cp.async.bulk behind an mbarrier; neighbour lists hold 16-bit slots of the
                                    staged windows (half the list traffic, no L1 misses on the gathers).
                                    0 (default): per-particle int32 lists gathered from global memory through L1 -- the faster
                                    of the two for the 2M-particle DFSPH step (DESIGN.md section 4.3): random 16-byte
                                    shared-memory reads cost what L1 hits cost, and the staged tiles cap the occupancy of the
                                    velocity sweeps at 4 blocks per SM */
};

/* ---- lifetime ------------------------------------------------------------------------------ */
int  sphk_create(sphk_ctx** ctx, int max_fluid, int max_boundary, const sphk_grid* grid, void* stream);
void sphk_destroy(sphk_ctx* ctx);
int  sphk_set_option(sphk_ctx* ctx, int option, int value);
/* re-target the context at another (sub-)grid with the same cell length (a slab rank whose cuts moved): both particle
 * sets must be searched again before the next sweep; capacities and buffers are kept (the sort scratch is sized at creation
 * for any grid) */
int  sphk_set_grid(sphk_ctx* ctx, const sphk_grid* grid);
int  sphk_synchronize(sphk_ctx* ctx);
const char* sphk_error_string(int code);
/* number of kernels this library has launched on ctx since creation (bench.py's gpu_launches) */
long long sphk_launch_count(const sphk_ctx* ctx);
/* account for kernels replayed from a captured CUDA graph (the host-side counter does not see them) */
int  sphk_add_launches(sphk_ctx* ctx, long long n);
/* rcp.approx(cell_length) as the device computes it (bit pattern as float): lets a CPU checker
 * reproduce the GPU cell hash bit-for-bit */
int  sphk_device_rcp(sphk_ctx* ctx, float x, float* out_host);

/* ---- neighbour search: SPHSystem::neighborSearch, SPHSystem.cu:114-127 ------------------------
 * Replaces mapParticles2Cells_CUDA (CUDAFunctions.cuh:72-78), two thrust::sort_by_key with float3
 * payloads (SPHSystem.cu:119,121), thrust::fill + countingInCell_CUDA + thrust::exclusive_scan
 * (SPHSystem.cu:123-125).  Bit-exact contract: particle2cell (left in PRE-sort order, quirk Q2), the
 * stable-sort permutation applied to pos and vel, and cell_start[ncells+1].
 * which = 0: the fluid set (p = &scene->fluid, cell_start = cell_start_fluid);
 * which = 1: the boundary set (searched once at construction, SPHSystem.cu:69). */
int sphk_neighbor_search(sphk_ctx* ctx, int which, const sphk_particles* p, int* cell_start);

/* Applies the permutation of the last fluid neighbour search to a solver-private history array, in
 * place: replaces DFSPHSolver.cu:170-171 (denWarmStiff, width 1) and PBDSolver.cu:84-85
 * (fluidPosLast, width 3), which re-sort with particle2cell as keys and rely on sort stability. */
int sphk_permute(sphk_ctx* ctx, float* array, int width, int n);

/* Re-packs the shadows from the API arrays without re-sorting (after caller-side edits).  Boundary records take the
 * boundary velocities of body particles when bodies are defined (sphk_bodies_init); static records keep v = 0. */
int sphk_refresh(sphk_ctx* ctx, const sphk_scene* scene);

/* computeBoundaryMass_CUDA, SPHSystem.cu:79-112: mass_b = rhoB / max(eps, sum_k W(|x_b - x_k|)). */
int sphk_boundary_mass(sphk_ctx* ctx, const sphk_particles* boundary, const int* cell_start_boundary,
                       float rho_boundary, float radius);

/* Particles::advect, Particles.cu:28-36: pos += dt * vel on raw arrays (no context needed: the public method of the
 * class API; the solvers' own advection is the fused sphk_advect).  `stream` is a cudaStream_t or NULL. */
int sphk_particles_advect(float* pos, const float* vel, int n, float dt, void* stream);

/* thrust::fill, SPHSystem.cu:73 / BasicSPHSolver.cu:78 */
int sphk_fill(sphk_ctx* ctx, float* array, int n, float value);

/* ---- WCSPH: BasicSPHSolver.cu -------------------------------------------------------------- */
/* force(): vel += dt*G, BasicSPHSolver.cu:227-235 */
int sphk_gravity(sphk_ctx* ctx, const sphk_scene* s, float dt, const float G[3]);
/* viscosity_CUDA + thrust::transform(vel += deltaV), BasicSPHSolver.cu:183-225.  delta_v (float3[n])
 * is the reference's bufferFloat3 and receives visc*a*dt as in the reference. */
int sphk_viscosity(sphk_ctx* ctx, const sphk_scene* s, float* delta_v, float rho0, float visc, float dt);
/* computeColorGrad_CUDA, BasicSPHSolver.cu:277-330 */
int sphk_color_grad(sphk_ctx* ctx, const sphk_scene* s, float* color_grad, float rho0, float rho_boundary);
/* surfaceTensionAndAirPressure_CUDA, BasicSPHSolver.cu:332-381 */
int sphk_surface(sphk_ctx* ctx, const sphk_scene* s, const float* color_grad, float dt, float rho0,
                 float surface_tension, float air_pressure);
/* thrust::fill(density,0) + computeDensity_CUDA, BasicSPHSolver.cu:32-83 */
int sphk_density(sphk_ctx* ctx, const sphk_scene* s);
/* computePressure_CUDA, BasicSPHSolver.cu:103-111 */
int sphk_pressure(sphk_ctx* ctx, const sphk_scene* s, float rho0, float stiff);
/* pressureForce_CUDA, BasicSPHSolver.cu:113-165 */
int sphk_pressure_force(sphk_ctx* ctx, const sphk_scene* s, float dt);
/* Particles::advect (Particles.cu:28-36) + enforceBoundary_CUDA(pos,vel) (BasicSPHSolver.cu:85-101) */
int sphk_advect(sphk_ctx* ctx, const sphk_scene* s, float dt, const float space[3]);

/* ---- fused sweeps: the same quantities as the per-launch-site entries above, computed in fewer passes over the
 * neighbour lists (each neighbour record is gathered once for two operators).  Every quantity is formed by the
 * same operations in the same order as in its own sweep.  The class layer uses these by default. */
/* computeDensity_CUDA + computeColorGrad_CUDA (both depend on positions and masses only) */
int sphk_fused_density_color_grad(sphk_ctx* ctx, const sphk_scene* s, float* color_grad, float rho0, float rho_boundary);
/* computeDensityAlpha_CUDA + computeColorGrad_CUDA */
int sphk_fused_dfsph_density_alpha_color_grad(sphk_ctx* ctx, const sphk_scene* s, float* alpha, float* color_grad,
                                              float rho0, float rho_boundary);
/* computeDensityAlpha_CUDA (+ computeColorGrad_CUDA when color_grad != NULL) + the first computeDivergenceError_CUDA of
 * DFSPHSolver::correctDivergenceError (DFSPHSolver.cu:341), which reads the velocities the density sweep leaves
 * untouched and, per particle, the density and alpha that particle has just computed. */
int sphk_fused_dfsph_density_alpha_div_error(sphk_ctx* ctx, const sphk_scene* s, float* alpha, float* color_grad_or_null,
                                             float rho0, float rho_boundary, float* error, float* stiff, float dt);
/* viscosity_CUDA (+ vel += deltaV) followed by surfaceTensionAndAirPressure_CUDA.  delta_v and color_grad must be
 * distinct buffers (the reference reuses one buffer for both because it runs them one after the other). */
int sphk_fused_viscosity_surface(sphk_ctx* ctx, const sphk_scene* s, float* delta_v, const float* color_grad,
                                 float rho0, float visc, float dt, float surface_tension, float air_pressure);

/* ---- DFSPH: DFSPHSolver.cu ----------------------------------------------------------------- */
/* computeDensityAlpha_CUDA, DFSPHSolver.cu:212-259 */
int sphk_dfsph_density_alpha(sphk_ctx* ctx, const sphk_scene* s, float* alpha);
/* computeDivergenceError_CUDA, DFSPHSolver.cu:261-306 */
int sphk_dfsph_div_error(sphk_ctx* ctx, const sphk_scene* s, const float* alpha, float* error,
                         float* stiff, float dt, float rho0);
/* correctDivergenceError_CUDA, DFSPHSolver.cu:308-329 */
int sphk_dfsph_div_correct(sphk_ctx* ctx, const sphk_scene* s, const float* stiff);
/* computeDensityError_CUDA, DFSPHSolver.cu:74-116.  warm_accumulate (may be NULL) additionally does
 * warm[i] += stiff[i], i.e. the thrust::transform of DFSPHSolver.cu:199-203 fused in. */
int sphk_dfsph_den_error(sphk_ctx* ctx, const sphk_scene* s, const float* alpha, float* error,
                         float* stiff, float dt, float rho0, float* warm_accumulate);
/* correctDensityError_CUDA, DFSPHSolver.cu:118-158 */
int sphk_dfsph_den_correct(sphk_ctx* ctx, const sphk_scene* s, const float* stiff, float dt);
/* thrust::reduce(error, abs_plus), DFSPHSolver.cu:206,360.  Synchronises; result to *host_out. */
int sphk_reduce_abs_sum(sphk_ctx* ctx, const float* x, int n, float* host_out);
/* Device-side control of an adaptive solver loop: the loop tests of DFSPHSolver.cu:187 / :347
 *     while ((iter < min_iter || totalError > threshold) && iter < max_iter) { body; ++iter; [totalError = reduce] }
 * evaluated on the device.  The host enqueues max_iter bodies; between sphk_loop_begin and sphk_loop_end every sweep
 * returns at once when the loop has ended, so no error sum travels to the host and the launch sequence is fixed (a
 * CUDA graph can replay it).  sphk_loop_next ends one iteration: ++iter, totalError = sum |error| (the same fixed-shape
 * reduction as sphk_reduce_abs_sum) from iteration reduce_from_iter on (DFSPHSolver.cu:205: the density loop reduces
 * from its second iteration), then the loop test.  slot: 0 or 1.  threshold = errorThreshold * num * rho0. */
int sphk_loop_begin(sphk_ctx* ctx, int slot, int min_iter, int max_iter, float threshold, int reduce_from_iter);
int sphk_loop_next(sphk_ctx* ctx, int slot, const float* error, int n);
int sphk_loop_end(sphk_ctx* ctx, int slot);
/* iterations the loop executed and its last error sum (synchronises) */
int sphk_loop_iterations(sphk_ctx* ctx, int slot, int* iterations_host, float* last_total_host);
/* cudaMemcpy D2D of a float array, DFSPHSolver.cu:185 */
int sphk_copy(sphk_ctx* ctx, float* dst, const float* src, int n_floats);

/* ---- PBD: PBDSolver.cu --------------------------------------------------------------------- */
/* computeDensityLambda_CUDA, PBDSolver.cu:127-168 (incl. the `bool rho0` quirk Q4) */
int sphk_pbd_density_lambda(sphk_ctx* ctx, const sphk_scene* s, float* lambda, float rho0, float relaxation);
/* computeDeltaPos_CUDA + thrust::transform(pos += dpos) + enforceBoundary_CUDA(pos),
 * PBDSolver.cu:170-256.  delta_pos (float3[n]) receives dp/rho0 as in the reference. */
int sphk_pbd_delta_pos_apply(sphk_ctx* ctx, const sphk_scene* s, const float* lambda, float* delta_pos,
                             float rho0, const float space[3]);
/* thrust::transform(vel = (pos - posLast)/dt), PBDSolver.cu:55-60 */
int sphk_pbd_velocity_from_positions(sphk_ctx* ctx, const sphk_scene* s, const float* pos_last, float dt);
/* XSPHViscosity_CUDA, PBDSolver.cu:89-125; Jacobi (the reference updates in place and races, Q5) */
int sphk_pbd_xsph(sphk_ctx* ctx, const sphk_scene* s, float c, float rho0);

/* XSPHViscosity_CUDA + computeColorGrad_CUDA in one pass over the neighbour list (the colour gradient reads positions and
 * masses only, which PBD does not change after its projection) */
int sphk_fused_pbd_xsph_color_grad(sphk_ctx* ctx, const sphk_scene* s, float c, float rho0, float* color_grad, float rho_boundary);

/* ---- vorticity confinement (no reference counterpart: Macklin & Mueller 2013, section 5; DESIGN.md section 2.2) ----------
 * Puts back the rotation the discretisation and the viscosity (XSPH, artificial viscosity) smear out.  Fluid neighbours
 * only, V_j = m_j / rho0, gradW_ij the kernel gradient at x_i - x_j:
 *   omega_i = sum_j V_j (v_i - v_j) x gradW_ij                  (rigid rotation v = W x x: +2 W in the bulk)
 *   eta_i   = sum_j V_j (|omega_j| - |omega_i|) gradW_ij,  N_i = eta_i / max(|eta_i|, eps)
 *   v_i    += dt * eps_conf * (N_i x omega_i)
 * The class layer forms omega from the velocities its viscosity / XSPH sweep reads and confines right after the surface
 * sweep (BasicSPHSolver::setVorticityConfinement).  All entries return SPHK_ERR_INVALID for NULL or aliased buffers,
 * rho0 <= 0, and (confinement) eps_conf < 0 or NaN. */
/* omega (float3[n]) and omega_norm = |omega| (float[n]).  No reference counterpart. */
int sphk_vorticity(sphk_ctx* ctx, const sphk_scene* s, float* omega, float* omega_norm, float rho0);
/* vel += dt * eps * (N x omega) for fluid particles; API array and records.  omega_norm is mirrored into the records
 * (the neighbour scalar) first.  No reference counterpart. */
int sphk_vorticity_confinement(sphk_ctx* ctx, const sphk_scene* s, const float* omega, const float* omega_norm, float eps,
                               float dt, float rho0);
/* sphk_fused_viscosity_surface + sphk_vorticity in one sweep; omega is formed from the velocities before the viscosity
 * update, exactly as sphk_vorticity called before sphk_fused_viscosity_surface forms it.  No reference counterpart. */
int sphk_fused_viscosity_surface_vorticity(sphk_ctx* ctx, const sphk_scene* s, float* delta_v, const float* color_grad,
                                           float rho0, float visc, float dt, float surface_tension, float air_pressure,
                                           float* omega, float* omega_norm);
/* sphk_pbd_xsph (+ the colour gradient of sphk_fused_pbd_xsph_color_grad when color_grad_or_null != NULL) + sphk_vorticity
 * in one sweep, omega from the velocities before XSPH.  No reference counterpart. */
int sphk_fused_pbd_xsph_vorticity(sphk_ctx* ctx, const sphk_scene* s, float c, float rho0, float* color_grad_or_null,
                                  float rho_boundary, float* omega, float* omega_norm);

/* ---- implicit viscosity (no reference counterpart: Weiler, Koschier, Brand & Bender 2018; DESIGN.md section 2.5) ------------
 * Solves A v = b for the new fluid velocities, v* = the velocities entering the solve, d = x_i - x_j, g = the kernel gradient
 * factor (gradW_ij = g d, g <= 0), R = support radius:
 *   c_ij    = -10 nu V_j g / (r^2 + 0.01 R^2),  V_j = m_j / rho0   (boundary pairs: nu_boundary and m_b / rho_boundary)
 *   (A v)_i = D_i v_i - dt sum_j c_ij d (d . v_j)                         (fluid neighbours)
 *   D_i     = I + dt sum_j c_ij d d^T + dt sum_b c_ib d d^T
 *   b_i     = v*_i + dt sum_b c_ib d (d . v_b)                            (v_b: 0, or a kinematic body's velocity)
 * A is self-adjoint in <u,w>_M = sum m_i u_i . w_i with eigenvalues >= 1.  Preconditioned CG in that inner product with the
 * block-Jacobi preconditioner D_i^-1, x0 = v*, m-weighted dot products in double in a fixed shape; the loop ends at the first
 * of |b - A v|_M <= tol |b|_M, <r,z>_M = 0 (a fluid at rest comes out unchanged) and max_iter iterations.  The loop test runs on
 * the device: max_iter iterations are enqueued, the ones after the end return at once (no host synchronisation; a step graph
 * replays it).  The solution goes to the API velocities and the records.  `work` = caller-owned device floats,
 * sphk_implicit_viscosity_work_floats(n) of them for n fluid particles (so nothing is allocated inside a captured step).
 * SPHK_ERR_INVALID: NULL or aliased buffers, nu or nu_boundary < 0 / not finite, rho0 or rho_boundary <= 0, tol <= 0 or NaN,
 * max_iter < 1 or > SPHK_IMPLICIT_VISCOSITY_MAX_ITER, dt < 0.  SPHK_ERR_STATE: an active range is set (slab ranks), or
 * nu_boundary > 0 with dynamic bodies declared (sphk_bodies_set_dynamics: the viscous wall force is not part of their reaction).
 * Every one of the max_iter iterations is enqueued (6 launches each, a matvec sweep over all particles among them) and a
 * captured step graph holds them all; the ones after the end cost about 20-30 us each on the 2M-particle scenes, so max_iter
 * should not be far above the iterations a scene needs (DESIGN.md section 2.5). */
#define SPHK_IMPLICIT_VISCOSITY_MAX_ITER 1000
long long sphk_implicit_viscosity_work_floats(int n);
int sphk_implicit_viscosity(sphk_ctx* ctx, const sphk_scene* s, float* work, float nu, float nu_boundary, float dt, float rho0,
                            float rho_boundary, float tol, int max_iter);
/* iterations and final relative residual |r|_M / |b|_M of the last sphk_implicit_viscosity (0, 0 before the first), kept by the
 * context (the workspace may be freed after the solve); synchronises */
int sphk_implicit_viscosity_stats(sphk_ctx* ctx, int* iterations, float* rel_residual);
/* The two sweeps of the solve, one call each (per-element tests): D_i (float[6n], {xx, yy, zz, xy, xz, yz}) and b_i (float3[n]);
 * (A p)_i (float3[n]) from D (float[6n]) and p (float3[n]).  The matvec leaves the records' velocities as the API array holds
 * them.  Same validation as sphk_implicit_viscosity. */
int sphk_visc_implicit_setup(sphk_ctx* ctx, const sphk_scene* s, float* d_out, float* b_out, float nu, float nu_boundary, float dt,
                             float rho0, float rho_boundary);
int sphk_visc_implicit_matvec(sphk_ctx* ctx, const sphk_scene* s, const float* d_in, const float* p_in, float* ap_out, float nu,
                              float dt, float rho0);

/* ---- non-Newtonian viscosity (no reference counterpart; DESIGN.md section 2.9) -----------------------------------------------
 * The implicit viscosity solve above with a per-particle kinematic viscosity nu_i = model(gamma_dot_i), frozen for the step (one
 * Picard linearisation: gamma_dot from v*, the velocities entering the solve).
 *   shear rate: G_i = sum_j V_j (v_j - v_i) (x) gradW_ij, M_i = -sum_j V_j g d d^T (boundary neighbours only when beta > 0, with
 *               V_b = m_b / rho_boundary and the record's velocity), grad v_i = G_i M_i^-1 -- or G_i 3 / tr M_i where
 *               det M_i < 0.01 (tr M_i / 3)^3 --, E = (grad v + grad v^T) / 2, gamma_dot = sqrt(2 E:E)
 *   models (double, rounded to float once, clamped to [nu_min, nu_max]; stresses kinematic, i.e. divided by rho0):
 *     SPHK_RHEOLOGY_CROSS            params {nu0, nu_inf, lambda, m}:  nu = nu_inf + (nu0 - nu_inf) / (1 + (lambda gamma_dot)^m)
 *     SPHK_RHEOLOGY_HERSCHEL_BULKLEY params {K, n, tau_y, m_reg}:     nu = K gamma_dot^(n-1) + tau_y (1 - exp(-m_reg gamma_dot)) / gamma_dot
 *                                                                      (tau_y m_reg at gamma_dot = 0)
 *   pairs: fluid c_ij with nu_ij = (nu_i + nu_j) / 2 (so m_i c_ij = m_j c_ji: the PCG applies unchanged), boundary nu_ib = beta nu_i
 *   (beta = 0: free slip; 1: no-slip with the fluid's own viscosity).
 * nu_max must be finite: it bounds the largest eigenvalue of A and so the iterations the solve needs.  nu_field = caller-owned
 * device float[n]: receives nu_i.  work = sphk_rheology_work_floats(n) device floats.
 * SPHK_ERR_INVALID: NULL or aliased buffers, a non-finite parameter, nu_min < 0, nu_min > nu_max, a parameter outside its model's
 * range (Cross: nu0, nu_inf, lambda >= 0, m > 0; HB: K >= 0, n > 0, tau_y >= 0, m_reg >= 0), an unknown model, beta < 0, rho0 or
 * rho_boundary <= 0, tol <= 0, max_iter outside [1, SPHK_IMPLICIT_VISCOSITY_MAX_ITER].  SPHK_ERR_STATE: an active range (slab
 * ranks), or beta > 0 with dynamic bodies declared. */
#define SPHK_RHEOLOGY_CROSS 1
#define SPHK_RHEOLOGY_HERSCHEL_BULKLEY 2
typedef struct sphk_rheology {
    int model;
    float params[6];          /* the model's parameters in the order above; the unused ones must be finite (0) */
    float nu_min, nu_max;
} sphk_rheology;
long long sphk_rheology_work_floats(int n);
int sphk_non_newtonian_viscosity(sphk_ctx* ctx, const sphk_scene* s, float* work, float* nu_field, const sphk_rheology* rheology,
                                 float beta, float dt, float rho0, float rho_boundary, float tol, int max_iter);
/* of the last sphk_non_newtonian_viscosity (0 before the first; the shear statistics also of a later sphk_shear_rate): PCG
 * iterations and |r|_M / |b|_M, max gamma_dot, min and max nu, and the particles at the nu_max clamp; any pointer may be NULL.
 * Synchronises. */
int sphk_non_newtonian_stats(sphk_ctx* ctx, int* iterations, float* rel_residual, float* gamma_max, float* nu_min, float* nu_max,
                             int* n_at_max);
/* Per-element entries (tests): the shear sweep alone (gamma_dot, nu; optionally grad v as float[9n] row-major d v_a / d x_b and
 * int[n] = 1 where the scalar normalisation replaced M_i^-1); the model on a given gamma_dot array (no scene needed); the setup and
 * matvec sweeps with an explicit nu array (the matvec leaves the records' velocities as the API array holds them). */
int sphk_shear_rate(sphk_ctx* ctx, const sphk_scene* s, float* gamma_out, float* nu_out, float* grad_out_or_null,
                    int* flag_out_or_null, const sphk_rheology* rheology, float beta, float rho0, float rho_boundary);
int sphk_rheology_eval(sphk_ctx* ctx, const sphk_rheology* rheology, const float* gamma, float* nu_out, int n);
int sphk_visc_field_setup(sphk_ctx* ctx, const sphk_scene* s, float* d_out, float* b_out, const float* nu, float beta, float dt,
                          float rho0, float rho_boundary);
int sphk_visc_field_matvec(sphk_ctx* ctx, const sphk_scene* s, const float* d_in, const float* p_in, float* ap_out, const float* nu,
                           float dt, float rho0);

/* ---- heat transfer (no reference counterpart; DESIGN.md section 2.10) ----------------------------------------------------------
 * Every fluid particle carries a temperature T_i (a caller-owned device float[n] in the fluid's current order).  With d = x_i - x_j,
 * r = |d|, f = the kernel gradient factor (grad W = d f, f <= 0), eta^2 = 0.0025 R^2:
 *   dT_i/dt = sum_j c_ij (T_j - T_i),   c_ij = -2 alpha V_j f r^2 / (r^2 + eta^2) >= 0
 *   fluid neighbour: V_j = m_j / rho0 (so m_i c_ij = m_j c_ji: sum m T is conserved); boundary neighbour of group g (0 = the static
 *   walls, b + 1 = body b): V_b = m_b / rho_boundary, alpha -> h_g alpha, T_j -> T_g.  Groups at or past n_groups are adiabatic.
 * One substep k of K (dt_k = dt / K, K from sphk_heat_substeps): T += dt_k dT/dt (Jacobi: the sweep reads the old T only); on the
 * last substep the buoyancy v += -beta (T - t_ref) G dt (the step's dt, the new T) on the API velocities and the records.
 * The sweep records max dt_k sum_j c_ij and the count of particles above 1 (the discrete maximum principle holds below 1):
 * statistics, not a clamp.
 * SPHK_ERR_INVALID: NULL or aliased buffers, alpha < 0, a non-finite beta or t_ref, a group with a non-finite T or h < 0, n_groups
 * outside [0, SPHK_THERMAL_GROUPS], rho0 or rho_boundary <= 0, dt < 0, K < 1 or k outside [0, K).  SPHK_ERR_STATE: an active range
 * (slab ranks), or n_groups above 1 + the bodies of the context. */
#define SPHK_BODY_LIMIT 64                              /* bodies per context (sphk_bodies_init) */
#define SPHK_THERMAL_GROUPS (1 + SPHK_BODY_LIMIT)
typedef struct sphk_thermal_group {
    float t;                  /* temperature of the group's boundary particles */
    float h;                  /* relative conductance >= 0 (0: adiabatic) */
} sphk_thermal_group;
typedef struct sphk_thermal {
    float alpha;              /* diffusivity >= 0 (m^2/s in the scene's units) */
    float beta;               /* expansion coefficient of the buoyancy term */
    float t_ref;              /* temperature without buoyancy */
    int n_groups;             /* entries of groups[] in use */
    sphk_thermal_group groups[SPHK_THERMAL_GROUPS];
} sphk_thermal;
/* Host only, no context: the substep count K = max(1, ceil(dt S)), S = SPHK_HEAT_COP alpha (1 + h_max) / R^2 (h_max over the groups in
 * use), so that dt_k sum_j c_ij <= 1 in the scenes DESIGN.md section 2.10 derives SPHK_HEAT_COP from.  SPHK_ERR_INVALID for a bad
 * setting, radius <= 0, dt < 0 or non-finite, or K above 65536. */
#define SPHK_HEAT_COP 100.0
int sphk_heat_substeps(const sphk_thermal* thermal, float radius, float dt, int* substeps);
/* substep k of K of a step of length dt; work = n device floats (dT/dt); gravity = {gx, gy, gz} (host) */
int sphk_heat_step(sphk_ctx* ctx, const sphk_scene* s, const sphk_thermal* thermal, float* temperature, float* work, float dt, int k,
                   int substeps, float rho0, float rho_boundary, const float* gravity);
/* per element (tests): dT/dt of every particle; the statistics with dt_sub as dt_k */
int sphk_heat_conduction(sphk_ctx* ctx, const sphk_scene* s, const sphk_thermal* thermal, const float* temperature, float* dtdt_out,
                         float dt_sub, float rho0, float rho_boundary);
/* Statistics of the last step's substeps (0 before the first: the largest dt_k sum_j c_ij and the particle-substeps above 1), and,
 * when temperature and mass are given, min T, max T and sum m T (double) over n particles by a fixed-shape reduction (the same
 * bits for the same input).  Any output pointer may be NULL.  Synchronises. */
int sphk_heat_stats(sphk_ctx* ctx, const float* temperature, const float* mass, int n, float* max_courant, int* violators,
                    float* t_min, float* t_max, double* heat);
/* Temperature-dependent viscosity nu_i = clamp(nu_ref exp(-e (T_i - t_ref)), nu_min, nu_max) (double, rounded once; nu_max finite),
 * solved by the per-particle-nu PCG of section 2.9 (walls with beta nu_i); iterations and residual in
 * sphk_implicit_viscosity_stats.  work = sphk_implicit_viscosity_work_floats(n) floats, nu_field = n floats (receives nu_i).
 * SPHK_ERR_INVALID as sphk_non_newtonian_viscosity, and nu_ref < 0 or a non-finite e or t_ref; SPHK_ERR_STATE: slab ranks, beta > 0
 * with dynamic bodies. */
typedef struct sphk_viscosity_law {
    float nu_ref, e, t_ref, nu_min, nu_max;
} sphk_viscosity_law;
int sphk_thermal_viscosity(sphk_ctx* ctx, const sphk_scene* s, float* work, float* nu_field, const float* temperature,
                           const sphk_viscosity_law* law, float beta, float dt, float rho0, float rho_boundary, float tol,
                           int max_iter);
int sphk_thermal_viscosity_eval(sphk_ctx* ctx, const sphk_viscosity_law* law, const float* temperature, float* nu_out, int n);

/* ---- fluid-solid adhesion (Akinci et al. 2013; no reference counterpart; DESIGN.md section 2.11) -------------------------------
 * Every fluid particle i is pulled towards the boundary particles b near it; fluid pairs contribute nothing (the fluid's cohesion is
 * the surface tension of sphk_surface).  With x_ib = x_i - x_b, r = |x_ib|, g(b) the group of b (0 = the static walls, k + 1 = body
 * k) and m_b the boundary mass:
 *   a_i = - sum_b beta_g(b) Psi_b A(r) x_ib / r,   Psi_b = rho0 m_b / rho_boundary
 *   A(r) = 0.007 / R^3.25 (-4 r^2 / R + 6 r - 2 R)^(1/4)   for R/2 < r <= R, else 0
 *   v_i += dt a_i   (API velocities and records; a particle without such a pair gets no write)
 * Groups at or past n_groups do not adhere.  The sweep walks the boundary cell ranges around each particle's current cell (no
 * neighbour list), so every execution path gives the same bits.  When the context has declared dynamics (sphk_bodies_set_dynamics),
 * sphk_adhesion also gathers the reaction dt m_i beta_g Psi_k A x_ik / r and its moment into the bodies' impulse of the step
 * (sphk_bodies_integrate), like sphk_bodies_react.  The sweep counts the "wetted" particles (some pair in the band with beta > 0)
 * and the largest |a_i|.
 * SPHK_ERR_INVALID: NULL pointers, a non-finite or negative beta, n_groups outside [1, SPHK_ADHESION_GROUPS], rho0 or
 * rho_boundary <= 0, dt < 0 or non-finite.  SPHK_ERR_STATE: an active range (slab ranks), or n_groups above 1 + the bodies of the
 * context. */
#define SPHK_ADHESION_GROUPS (1 + SPHK_BODY_LIMIT)
typedef struct sphk_adhesion_setting {
    int n_groups;                           /* entries of beta[] in use */
    float beta[SPHK_ADHESION_GROUPS];       /* adhesion strength >= 0 of the static walls [0] and of body k [k + 1] */
} sphk_adhesion_setting;
int sphk_adhesion(sphk_ctx* ctx, const sphk_scene* s, const sphk_adhesion_setting* adhesion, float dt, float rho0, float rho_boundary);
/* per element (tests): a_i into accel (device float[3 n]) and the statistics; no velocity write, no reaction */
int sphk_adhesion_accel(sphk_ctx* ctx, const sphk_scene* s, const sphk_adhesion_setting* adhesion, float* accel, float rho0,
                        float rho_boundary);
/* the wetted count and the largest |a_i| of the last sphk_adhesion / sphk_adhesion_accel (0 before the first); either pointer
 * may be NULL.  Synchronises. */
int sphk_adhesion_stats(sphk_ctx* ctx, int* wetted, float* max_accel);

/* ---- kinematic rigid bodies (no reference counterpart; DESIGN.md section 2.3) ---------------------------------------------
 * A body is a rigid set of boundary particles given in body coordinates r_k, with a pose (centre c, unit quaternion q) and
 * a motion (linear velocity V, angular velocity Omega, both in the world frame).  Poses and motions live in device memory.
 * Layouts: pose = {cx, cy, cz, qx, qy, qz, qw} (scalar part LAST) per body, motion = {Vx, Vy, Vz, Ox, Oy, Oz} per body.
 *
 * sphk_bodies_init declares that the boundary slots [n_static, n) of the set that has NOT been searched yet belong to
 * n_bodies bodies (1..SPHK_MAX_BODIES = 64): body b owns slots [body_begin[b], body_begin[b+1]) with body_begin[0] = n_static,
 * body_begin[n_bodies] = boundary->n, non-decreasing; local_xyz holds r_k of slots n_static.. (host float3[n - n_static]).
 * pose and motion are host arrays (a non-unit quaternion is normalised, a zero one refused).  boundary->vel is required.
 * From then on every boundary search (sphk_neighbor_search(which = 1) too) places the body particles at their pose
 * (x_k = c + R(q) r_k, v_k = V + Omega x (x_k - c) into boundary->pos / vel), and carries the mass and {r_k, group} of every
 * particle with it; boundary records carry v_k for body particles and 0 for the static set.  sphk_boundary_mass sums
 * over the particle's own group only (the static set, or its body): m_b = rho_B / max(eps, sum_{k in group} W_bk).
 * Call it before the first boundary search (SPHK_ERR_STATE otherwise, and on a second call).  Synchronises.
 * A body particle that leaves the grid gets the out-of-grid cell (Q8) and stops interacting; nothing guards against it. */
int sphk_bodies_init(sphk_ctx* ctx, const sphk_particles* boundary, int n_static, int n_bodies, const int* body_begin,
                     const float* local_xyz, const float* pose, const float* motion);
/* New motions of all bodies (host float[6 * n_bodies]), enqueued on the stream as an ordinary copy: it takes effect at the
 * next sphk_bodies_step and does not change the launch sequence (a captured step graph stays valid).  The caller's buffer
 * may be reused on return (waits only while the previous change is still in the context's staging buffer). */
int sphk_bodies_set_motion(sphk_ctx* ctx, const float* motion_host);
/* One step of every body, before the fluid search: pose update (c += dt V; q = normalize(dq (x) q), dq the rotation by
 * |Omega| dt about Omega), placement, and the boundary search that carries mass and body frame (invalidates the lists as
 * a boundary search does).  dt > 0 and finite.  SPHK_ERR_STATE before sphk_bodies_init and the first boundary search. */
int sphk_bodies_step(sphk_ctx* ctx, const sphk_particles* boundary, int* cell_start_boundary, float dt);
/* current poses (host float[7 * n_bodies]); synchronises */
int sphk_bodies_get_pose(sphk_ctx* ctx, float* pose_host);
/* introspection: the carried {r_k, group} of every boundary slot in the current (sorted) order, device float4[n] (group
 * 0 = static, b + 1 = body b) */
int sphk_bodies_get_local(sphk_ctx* ctx, float* local_out);

/* ---- two-way coupled bodies (no reference counterpart; DESIGN.md section 2.4) ------------------------------------------------
 * The fluid pushes back on bodies: every sweep whose boundary term changes fluid momentum, c m_i m_k s_i gradW(x_i - x_k) for
 * a fluid particle i and a body particle k, is followed by sphk_bodies_react with its c; the body gathers the opposite
 * impulse J and its moment H about the body's centre.  sphk_bodies_integrate then moves the dynamic bodies at the end of the
 * step.
 *
 * sphk_bodies_set_dynamics declares the bodies' masses and principal moments, mass_inertia = {M, Ix, Iy, Iz} per body (host
 * float[4 * n_bodies]), the moments about the centre in body axes (the axes of r_k).  M > 0 makes a body dynamic and needs
 * I > 0; M = 0 keeps it kinematic ("held"), its reaction is still gathered and reported (a force sensor).  Mass units are
 * those of the fluid's momentum: a fluid particle of mass m0 stands for a volume spacing^3, so the fluid's mass per unit
 * volume is m0 / spacing^3 (about 9.57 in the reference's scenes), NOT rho0; a body of relative density REL and volume V has
 * M = REL * m0 / spacing^3 * V.  space = the domain size: dynamic bodies stay inside the fluid's clamp box
 * [0, 0.99 space] per axis (the corners of the body-frame bounding box of r_k; the centre is moved back and the outward
 * velocity zeroed at each pose update; no friction, no torque; bodies pass through each other).  Call it once, after
 * sphk_bodies_init and before the first sphk_bodies_step (SPHK_ERR_STATE otherwise).  Synchronises.
 * A system that never calls it launches nothing new. */
int sphk_bodies_set_dynamics(sphk_ctx* ctx, const float* mass_inertia, const float space[3]);
/* Gathers the reaction of the sweep just run, per body particle, from the fluid records' scalar s_i and positions and the
 * fluid masses (scene->fluid.mass):  c = -dt after sphk_pressure_force; 1 after sphk_dfsph_div_correct; 1/dt after
 * sphk_dfsph_den_correct (warm start included); 1/(rho0 dt) between sphk_pbd_density_lambda and sphk_pbd_delta_pos_apply.
 * Returns at once inside a device-controlled loop that has ended, like the sweeps.  Reads the records only.  SPHK_ERR_STATE
 * before sphk_bodies_set_dynamics and under an active range (slab ranks). */
int sphk_bodies_react(sphk_ctx* ctx, const sphk_scene* scene, float c);
/* End of step: the gathered {J, H} of every body become the reported impulse (sphk_bodies_get_impulse) and are cleared; a
 * dynamic body's motion becomes V += J / M + dt G, Omega = (R diag(I) R^T)^-1 (R diag(I) R^T Omega + H), R from the current
 * pose.  The next sphk_bodies_step moves it.  dt > 0, G finite.  While a tank motion is set (sphk_tank_set) G is replaced by the
 * R (G - a_w) of the last sphk_tank_force. */
int sphk_bodies_integrate(sphk_ctx* ctx, float dt, const float G[3]);
/* New motion {V, Omega} of one body (host float[6]), enqueued like sphk_bodies_set_motion; the other bodies keep their
 * device-side motion (the integrated one, for dynamic bodies). */
int sphk_bodies_set_body_motion(sphk_ctx* ctx, int body, const float motion[6]);
/* current motions (host float[6 * n_bodies]); synchronises */
int sphk_bodies_get_motion(sphk_ctx* ctx, float* motion_host);
/* {Jx, Jy, Jz, Hx, Hy, Hz} per body of the last integrated step (host float[6 * n_bodies]; J / dt is the mean force); synchronises */
int sphk_bodies_get_impulse(sphk_ctx* ctx, float* impulse_host);

/* ---- open boundaries: emitters and sinks (no reference counterpart; DESIGN.md section 2.6) ----------------------------------
 * The fluid set keeps capF slots (sphk_create's max_fluid) of which the first n are live; n changes between steps.
 * An emitter is a rectangular nozzle {origin o, direction d, speed u > 0, spacing s > 0, width W >= 1, height H >= 1}.  Its axes
 * (sphk_emitter_axes) are d normalised in double, e1 = normalize(d x y^) (normalize(d x x^) when |d . y^| > 0.9) and e2 = e1 x d,
 * all in double, rounded to float once.  A layer at offset delta is the W x H lattice
 *     x_ab = o + ((a - (W-1)/2) s) e1 + ((b - (H-1)/2) s) e2 + delta d      (float, in that order, no contraction)
 * with slot dst + k W H + b W + a for layer k; its particles get v = u d, mass m0, density 0, pressure 0.
 * A sink is an axis-aligned box {lo, hi}, lo < hi per axis: a live fluid particle with lo <= x < hi on all three axes is removed.
 *
 * The order of a step (the class layer's SPHSystem::step, engine.SphkSystem.step):
 *   1. sphk_sinks_apply over the n live slots: marks the particles inside a sink (position -1e6, velocity 0) and counts them;
 *   2. sphk_emit of the scheduled layers (sphk_emitter_advance) into slots [n, n + e), history slot included;
 *   3. the bodies' step, if any;
 *   4. sphk_neighbor_search over n + e slots: marked particles get the out-of-grid key and sort behind every live one (stable);
 *   5. L = n + e - removed (sphk_sinks_removed waits for the sinks' count only, so it overlaps the search), then
 *      sphk_fluid_set_count(L): permutes, lists and sweeps cover [0, L) from here on;
 *   6. the solver's step on L particles.
 * Removal happens before the search, so the L live particles are exactly the set a closed system built from the survivors plus
 * the emitted particles (in the same pre-sort order) would hold after its search.
 * All of these entries except the two host-only ones return SPHK_ERR_STATE under an active range (slab ranks). */
#define SPHK_MAX_EMITTERS 16
#define SPHK_MAX_SINKS 16
typedef struct sphk_emitter {
    float origin[3];
    float direction[3];   /* any length > 0: the library normalises it */
    float speed;          /* u > 0 */
    float spacing;        /* s > 0: lattice spacing within a layer and distance between layers */
    int   width, height;  /* W, H >= 1 */
} sphk_emitter;
/* Host only (no context, no device): {d, e1, e2} as float[9], the values sphk_emit uses.  SPHK_ERR_INVALID for a NULL pointer, a
 * non-finite value, |d| = 0, u <= 0, s <= 0, W or H < 1. */
int sphk_emitter_axes(const sphk_emitter* e, float axes_out[9]);
/* Host only: the emission schedule of one step, in double.  carry += u dt; while carry >= s: a layer with delta = carry - s,
 * carry -= s.  Layers are therefore exactly s apart along the stream, and several may come in one step.  *scheduled_out = the
 * layers due this step; the first min(scheduled, max_layers) deltas go to offsets_out (float[max_layers]); the rest are refused
 * (the caller counts them: a partial layer is never emitted, and their carry is spent all the same).  max_layers = the whole
 * layers that fit in the remaining capacity.  SPHK_ERR_INVALID: an invalid emitter (as sphk_emitter_axes), a NULL carry or
 * scheduled_out, offsets_out NULL with max_layers > 0, max_layers < 0, dt < 0 or not finite, a carry < 0 or not finite, or more than
 * 65536 layers due in one step. */
int sphk_emitter_advance(const sphk_emitter* e, double* carry, float dt, int max_layers, float* offsets_out, int* scheduled_out);
/* Writes n_layers layers of emitter e (offsets_host: their deltas, host float[n_layers]) into fluid slots [dst_begin,
 * dst_begin + n_layers W H): pos, vel, mass (= m0), density and pressure (= 0), and the solver's history slot of each:
 * history_kind 0 = none (history NULL), 1 = zero (width 1: DFSPH's warm-start stiffness), 2 = x - dt v (width 3: PBD's last
 * position, from which PBDSolver recovers v).  The slots must then be searched (sphk_neighbor_search over dst_begin + the new
 * particles): until then sweeps return SPHK_ERR_STATE.  SPHK_ERR_INVALID: NULL pointers, an invalid emitter, non-finite offsets,
 * m0 <= 0, dt < 0, n_layers < 0, dst_begin < 0, history_kind outside 0..2 or history NULL with kind != 0; SPHK_ERR_CAPACITY when
 * dst_begin + n_layers W H > max_fluid. */
int sphk_emit(sphk_ctx* ctx, const sphk_particles* fluid, int dst_begin, const sphk_emitter* e, int n_layers,
              const float* offsets_host, float m0, float dt, float* history, int history_kind);
/* Marks the live particles [0, fluid->n) inside any of the n_boxes sinks (boxes_host: float[6 n_boxes] = {lo.xyz, hi.xyz}): position
 * (-1e6, -1e6, -1e6), velocity 0; counts them (warp-aggregated integer adds: deterministic) into memory the context owns, then an
 * event.  Must be followed by a fluid search (sweeps return SPHK_ERR_STATE until then).  SPHK_ERR_INVALID: NULL pointers, n_boxes
 * outside 0..SPHK_MAX_SINKS, a non-finite bound or lo >= hi on some axis. */
int sphk_sinks_apply(sphk_ctx* ctx, const sphk_particles* fluid, const float* boxes_host, int n_boxes);
/* The count of the last sphk_sinks_apply; waits for that kernel only (not for work enqueued after it).  SPHK_ERR_STATE before the
 * first sphk_sinks_apply. */
int sphk_sinks_removed(sphk_ctx* ctx, int* removed_host);
/* Truncates the searched fluid set to its first L slots (the marked particles sorted behind them): nF = L for sphk_permute, the
 * lists and the sweeps.  Valid between a fluid search and the first sweep (SPHK_ERR_STATE otherwise, and for L > the searched
 * count; SPHK_ERR_INVALID for L < 0 or a NULL cell_start_fluid).  Enqueues a one-thread check that cell_start_fluid[ncells] == L:
 * a mismatch (a live particle had left the grid, or a marked one had not) sets a sticky bit read by sphk_open_check. */
int sphk_fluid_set_count(sphk_ctx* ctx, const int* cell_start_fluid, int L);
/* the sticky error bits of sphk_fluid_set_count's check (0 = fine; bit 0 = a count mismatch since the context was created);
 * synchronises */
int sphk_open_check(sphk_ctx* ctx, int* error_bits_host);

/* ---- CFL-adaptive time stepping (no reference counterpart; DESIGN.md section 2.8) ---------------------------------------------
 * The step-size rule {C, dt_min, dt_max, R, |G|}, host only, in double (sphk_time_step):
 *   v_b = v_max + |G| dt_prev;  dt_cfl = C R / v_b (dt_max when v_b = 0), clamped to [dt_min, dt_max] (SPHK_DT_MIN_CLAMP when
 *   dt_min binds); a v_max that is not finite gives dt_min (SPHK_DT_NONFINITE).  With remaining > 0 (the rest of a frame):
 *   remaining <= dt_cfl gives dt = remaining (SPHK_DT_FRAME_END: the frame ends with this step, which may be shorter than
 *   dt_min), remaining < 2 dt_cfl gives dt = remaining / 2 (no sliver step at the end of the frame).  remaining <= 0: no frame.
 *   The result is rounded to float once; that float is the dt every kernel of the step receives.
 * The speed bound of a step (sphk_step_speed) is computed on the device after the step's last velocity write. */
typedef struct sphk_time_step_rule {
    double cfl;        /* C > 0 (relative to the support radius R) */
    double dt_min;     /* 0 < dt_min <= dt_max */
    double dt_max;
    double radius;     /* R > 0 */
    double gravity;    /* |G| >= 0 */
} sphk_time_step_rule;
#define SPHK_DT_MIN_CLAMP 1
#define SPHK_DT_NONFINITE 2
#define SPHK_DT_FRAME_END 4
/* Host only (no context, no device).  SPHK_ERR_INVALID: NULL pointers, a rule field that is not finite or out of range,
 * v_max < 0 (NaN and +inf are accepted and flagged), dt_prev < 0 or not finite, remaining not finite. */
int sphk_time_step(const sphk_time_step_rule* r, double v_max, double dt_prev, double remaining, float* dt_out, int* flags_out);
/* Enqueues the speed bound of the current state: max |v| over the live fluid particles [0, fluid->n) (|v|^2 = (vx vx + vy vy) +
 * vz vz in float, no contraction; warp and block maxima, one atomicMax on the float bits per block: order-independent), particles
 * with a non-finite velocity component counted (warp-aggregated adds) and left out of the max; with with_bodies != 0 also
 * |V| + |Omega| r_max per body from the device-resident motions (r_max = max_k |r_k|, from sphk_bodies_init; a non-finite motion
 * is counted and left out).  The result goes to memory the context owns, then by an asynchronous copy to pinned memory, then an
 * event.  SPHK_ERR_INVALID: NULL pointers, fluid->n < 0 or > max_fluid; SPHK_ERR_STATE: with_bodies without sphk_bodies_init, or
 * an active range is set (slab ranks: the bound would need a global maximum). */
int sphk_step_speed(sphk_ctx* ctx, const sphk_particles* fluid, int with_bodies);
/* Waits for the copy of the last sphk_step_speed only; v_max_host = float[2] {fluid max |v|, body max |V| + |Omega| r_max} (0 for
 * an empty set), *nonfinite_host = the particles and bodies left out.  SPHK_ERR_STATE before the first sphk_step_speed. */
int sphk_step_speed_result(sphk_ctx* ctx, float* v_max_host, int* nonfinite_host);

/* Builds the per-step neighbour list now (sweeps otherwise build it lazily on first use). */
int sphk_build_neighbor_list(sphk_ctx* ctx, const sphk_scene* s);

/* ---- scene generation on the device: initSPHSystem(), main.cpp:73-116 (SURVEY 8f-4) ---------------------------------------
 * The dam-break scene without a host-side particle array: positions are bit-identical to the host code's (same float
 * operations in the same order, no contraction) and in the reference's push order.
 * fluid block nx * ny * nz at `origin` with `spacing` (main.cpp:76-85: y outermost, then x, z innermost), restricted to the
 * x-columns [j_begin, j_begin + j_count) -- a slab rank generates only its own columns; pos_out: float3[ny * j_count * nz]. */
int sphk_scene_fluid_block(float* pos_out, int nx, int ny, int nz, const float origin[3], float spacing, int j_begin, int j_count,
                           void* stream);
/* six-face boundary shell of the box `space` on the lattice 2 * cell_size (main.cpp:89-116); pos_out: float3[count] */
long long sphk_scene_boundary_count(const int cell_size[3]);
int sphk_scene_boundary_shell(float* pos_out, const int cell_size[3], const float space[3], void* stream);

/* ---- scenes from triangle meshes (no reference counterpart; DESIGN.md section 2.12) -----------------------------------------
 * A mesh is float3 vertices and int3 triangles (counter-clockwise seen from outside on a closed mesh).  None of these entries
 * needs an sphk_ctx; all are safe before sphk_create.  Every entry checks all of its arguments before anything is launched or
 * allocated: NULL or overlapping buffers, counts <= 0, a triangle index outside [0, nv) and a non-finite vertex or parameter give
 * SPHK_ERR_INVALID.
 * sphk_mesh_transform: host only, v_out = scale * v_in + t per coordinate in float (multiply, then add; no contraction) -- the one
 *   place a mesh transform is computed, so every layer gets the same bits.
 * sphk_mesh_properties: host only, in double.  flags bit SPHK_MESH_CLOSED: every edge is shared by exactly two triangles that
 *   run it in opposite directions (and nt >= 4).  out = {area, V, centroid xyz, inertia tensor per unit density about the centroid
 *   {xx, yy, zz, xy, xz, yz}, principal moments ascending (3), the rotation from the principal (body) axes to the world as a unit
 *   quaternion (x, y, z, w)} by the divergence theorem; the body axes have det +1, each of the first two has its largest component
 *   positive, and w >= 0.  A closed mesh with reversed winding gives the same outputs (|V|, the tensor's sign flipped with V).  An
 *   open mesh reports the area only (the rest 0). */
#define SPHK_MESH_PROPS 18
#define SPHK_MESH_CLOSED 1
#define SPHK_MESH_INSIDE 1        /* sphk_mesh_classify flag bits */
#define SPHK_MESH_NEAR 2
typedef struct sphk_mesh sphk_mesh;
int sphk_mesh_transform(const float* v_in, int nv, float scale, const float t[3], float* v_out);
int sphk_mesh_properties(const float* v, int nv, const int* tri, int nt, double out[SPHK_MESH_PROPS], int* flags);
/* Uploads the mesh (host arrays) and bins its triangles, in triangle-index order, into a 3D uniform grid (distance queries) and a
 * 2D (x, z) column grid (ray parity).  Every later call on the mesh runs on `stream`. */
int sphk_mesh_create(sphk_mesh** m, const float* v_host, int nv, const int* tri_host, int nt, void* stream);
void sphk_mesh_destroy(sphk_mesh* m);
/* Device arrays pos float3[n] -> flags_out int[n]: SPHK_MESH_INSIDE = odd number of crossings of the +y ray from the point
 * (watertight: exact orientation predicates in (x, z) and one fixed tie rule, so a ray through a shared edge or vertex counts
 * once); SPHK_MESH_NEAR = distance to the surface <= clearance (>= 0).  Asynchronous.  SPHK_ERR_INVALID also for an open mesh. */
int sphk_mesh_classify(const sphk_mesh* m, const float* pos, int n, float clearance, int* flags_out);
/* The lattice points origin + spacing * (j, i, k) (float multiply then add, as sphk_scene_fluid_block) over the mesh's bounding box
 * that are inside and not near (clearance), in the fluid block's order (i = y outermost, then j = x, k = z innermost).  pos_out:
 * device float3[capacity]; *count_host = the number of such points; when it exceeds capacity nothing is written.  Synchronises.
 * SPHK_ERR_INVALID also for an open mesh, spacing <= 0 and a lattice of more than 2^31 - 1 points over the box. */
int sphk_mesh_fill(const sphk_mesh* m, float spacing, const float origin[3], float clearance, float* pos_out, int capacity,
                   int* count_host);
/* A maximal Poisson-disk sampling of the surface (open meshes too) with minimum distance r: candidates on a barycentric lattice of
 * spacing <= r/4 per triangle (edges and vertices included), accepted in (cell, candidate) order in 27 colour phases of cells of
 * side >= r.  Every sample lies on a triangle, no two are closer than r, every surface point is within r + r/4 of a sample, and
 * the output (ordered by cell, then candidate) is the same on every call.  pos_out: device float3[capacity]; *count_host and
 * capacity as sphk_mesh_fill.  Synchronises.  SPHK_ERR_INVALID also for r <= 0 and more than 2^31 - 1 candidates. */
int sphk_mesh_sample_surface(const sphk_mesh* m, float r, float* pos_out, int capacity, int* count_host);

/* ---- probes and water-level gauges (no reference counterpart; DESIGN.md section 2.13) ------------------------------------------
 * SPH-interpolated fluid fields at points.  For a point x, over the fluid particles j with |x - x_j| <= R and rho_j > 0, with
 * V_j = m_j / rho_j and W the continuous cubic spline of radius R (W(0) > 0: no quirk Q1, so the interpolant does not jump when x
 * sits on a particle; boundary particles take no part):
 *   S(x) = sum_j V_j W (the Shepard sum),  n(x) = the count of those particles,
 *   A(x) = sum_j V_j A_j W / S  for A in {rho, v, p, T}   (so rho(x) = sum_j m_j W / S)
 * A record is 8 floats {S, rho, vx, vy, vz, p, T, n} (32 bytes, 16-byte aligned).  A point with no such particle, or outside the
 * grid, is dry: n = 0 and zeros (S = 0 with n > 0 -- every particle exactly at R -- also gives zero fields).  p is NaN when
 * pressure_or_null is NULL (only WCSPH keeps a pressure field), T is NaN when temperature_or_null is NULL.
 * A gauge is the segment a -> b with k samples a + (b - a) (i / (k - 1)), i = 0..k-1 (each operation rounded once).  With i* the
 * highest sample with S >= threshold, its level is the linear crossing of the threshold between i* and i* + 1, measured from a
 * along the segment; |b - a| when i* = k - 1 (overtopped); -1 when no sample is wet.  A gauge has no notion of up: orient it along
 * -G for a water level.
 * Every entry reads the API arrays pos, vel, mass, density (and the optional pressure and temperature arrays, in the fluid's
 * current order) as the caller left them and the fluid cell ranges of the last search -- not the packed records.  Reach: the cells
 * within 1 of the point's (2 when positions have moved since the search), so no particle may have moved more than one cell since
 * the search (the sphk_bodies_react / sphk_adhesion contract).  Particles outside the grid do not count; live particles only.
 * Refused before anything is enqueued: NULL pointers, a non-finite value, an output overlapping a scene array or an input
 * (SPHK_ERR_INVALID); the set not searched or sized otherwise, and an active range (slab ranks) (SPHK_ERR_STATE). */
#define SPHK_PROBE_FIELDS 8
#define SPHK_PROBE_LIMIT 4096                 /* probes of one series */
#define SPHK_GAUGE_LIMIT 64                   /* gauges of one series or call */
#define SPHK_GAUGE_MAX_SAMPLES 1024           /* samples per gauge (at least 2) */
#define SPHK_PROBE_CAPACITY_LIMIT 65536       /* rows of a series ring */
typedef struct sphk_gauge {
    float a[3], b[3];        /* the segment, a != b */
    int samples;             /* k in [2, SPHK_GAUGE_MAX_SAMPLES] */
} sphk_gauge;
/* records of n points (device float3[n]) into out (device float[8 n]).  The points are checked for finite values on the device
 * first, which synchronises. */
int sphk_probe_sample(sphk_ctx* ctx, const sphk_scene* s, const float* points, int n, const float* pressure_or_null,
                      const float* temperature_or_null, float* out);
/* records of the lattice origin + spacing (ix, iy, iz) (multiply then add, per axis), z fastest -- the cell hash's order -- into
 * out[nx][ny][nz][8].  spacing > 0 and finite, dims >= 1, at most 2^31 - 1 points. */
int sphk_probe_lattice(sphk_ctx* ctx, const sphk_scene* s, const float origin[3], float spacing, const int dims[3],
                       const float* pressure_or_null, const float* temperature_or_null, float* out);
/* levels of n_gauges (1..SPHK_GAUGE_LIMIT) gauges (host array) into out (device float[n_gauges]); threshold finite and > 0 */
int sphk_gauge_levels(sphk_ctx* ctx, const sphk_scene* s, const sphk_gauge* gauges, int n_gauges, float threshold, float* out);
/* A series: fixed probes (host float3[n_points], up to SPHK_PROBE_LIMIT) and gauges (host, up to SPHK_GAUGE_LIMIT; at least one of
 * the two) recorded into a device ring of `capacity` rows.  sphk_probes_record writes the row into slot (counter mod capacity) and
 * then advances the counter, both on the device: no argument changes from step to step, so the two launches can sit inside a
 * captured step graph.  sphk_probe_series_read (synchronises on the series' stream) gives the counter and copies the last
 * min(counter, capacity, max_rows) rows, oldest first: records [rows][n_points][8] and levels [rows][n_gauges]. */
typedef struct sphk_probe_series sphk_probe_series;
int sphk_probe_series_create(sphk_probe_series** series, const float* points_host, int n_points, const sphk_gauge* gauges_host,
                             int n_gauges, float threshold, int capacity, void* stream);
void sphk_probe_series_destroy(sphk_probe_series* series);
int sphk_probes_record(sphk_ctx* ctx, const sphk_scene* s, sphk_probe_series* series, const float* pressure_or_null,
                       const float* temperature_or_null);
int sphk_probe_series_read(sphk_probe_series* series, long long* counter, int max_rows, float* records_host, float* levels_host,
                           int* rows);

/* ---- checkpoints (no reference counterpart; DESIGN.md section 2.14) ------------------------------------------------------------
 * A checkpoint file holds the mutable state of one system as named sections of bytes.  The caller lists the sections (device or
 * host memory); the library appends the context's own body and open-boundary state ("ctx.*") and owns the format:
 *   header  "SPHKCKPT" | u32 version | u32 sections | u64 header bytes | u64 file bytes | u64 config hash |
 *           sphk_state_config (152 bytes) | sections x {char name[32], u64 offset, u64 bytes, u32 element size, u32 host,
 *           u64 checksum} | u32 CRC-32 (zlib) of every header byte before it | zero padding to 16
 *   payload every section at its (16-byte aligned) file offset, zero-padded to 16 bytes
 * Section checksum: the bytes as little-endian u64 words w_i (the last one zero-padded), h = sum_i splitmix64(w_i + (i + 1)
 * 0x9E3779B97F4A7C15) mod 2^64 (splitmix64's finaliser: z ^= z >> 30, z *= 0xBF58476D1CE4E5B9, z ^= z >> 27, z *= 0x94D049BB133111EB,
 * z ^= z >> 31).  The config hash is the checksum of the config record's bytes.
 * sphk_checkpoint_save packs the device sections into a device staging buffer in one launch on the context's stream (with their
 * checksums), copies the host sections at once, and returns: a copy stream moves the staging buffer to pinned host memory and a host
 * thread writes path.tmp, fsyncs and renames it to path.  The snapshot is the stream state at the call; later work on the stream
 * overlaps the copy and the write.  A save waits for the previous one to finish first (one pinned buffer).  sphk_checkpoint_wait
 * joins it and returns the result of the saves since the last wait (0, or the first error with its message).  The staging buffers are allocated at the first save or load and
 * freed by sphk_checkpoint_release or sphk_destroy.
 * Loading: sphk_state_open reads and checks a file on the host (magic, version, sizes, header CRC; no device needed).
 * sphk_checkpoint_load then compares the config record field by field and the section table (names, order, sizes) with the
 * system's, verifies the host checksums on the host and the device ones on the device after uploading, and only when everything
 * passed writes the sections.  A refused call writes nothing and names the field or section at fault in msg.
 * sphk_checkpoint_invalidate drops what the context derived from the state it had (neighbour list, search, record scalar tags,
 * DFSPH chunk activity and velocity epochs, last-step statistics): the next step rebuilds them. */
#define SPHK_STATE_VERSION 1
#define SPHK_STATE_MAX_SECTIONS 64
#define SPHK_STATE_NAME 32
typedef struct sphk_state_config {
    char solver[16];                 /* "wcsph", "dfsph", "pbd" */
    int capacity_fluid, capacity_boundary, n_boundary, n_bodies;
    int cell_size[3];
    int flags;                       /* 1 fused sweeps, 2 device loops, 4 open boundaries, 8 dynamic bodies, 16 adaptive dt */
    float space_size[3], cell_length, radius, dt, m0, rho0, rho_boundary, stiff, visc, surface_tension, air_pressure, gravity[3];
    float solver_args[4];            /* DFSPH: density / divergence thresholds, max iterations; PBD: max iterations, XSPH c, relaxation */
    unsigned long long bodies_hash;  /* body-local points, masses and inertias */
    unsigned long long open_hash;    /* emitters and sinks */
    unsigned long long settings_hash;/* vorticity, implicit viscosity, rheology, thermal, thermal viscosity, adhesion, adaptive rule */
} sphk_state_config;
typedef struct sphk_state_section {
    char name[SPHK_STATE_NAME];
    void* ptr;                       /* device memory (host = 0) or host memory (host = 1) */
    unsigned long long bytes;
    unsigned int elem_size;
    int host;
} sphk_state_section;
typedef struct sphk_state_file sphk_state_file;
int  sphk_state_checksum_host(const void* data, unsigned long long bytes, unsigned long long* out);
int  sphk_state_crc32_host(const void* data, unsigned long long bytes, unsigned int* out);
/* the same checksum of device memory, computed by the pack kernel (synchronises) */
int  sphk_state_checksum_device(sphk_ctx* ctx, const void* data, unsigned long long bytes, unsigned long long* out_host);
int  sphk_checkpoint_save(sphk_ctx* ctx, const char* path, const sphk_state_config* config, const sphk_state_section* sections,
                          int n_sections);
int  sphk_checkpoint_wait(sphk_ctx* ctx, char* msg, int msg_len);
int  sphk_checkpoint_release(sphk_ctx* ctx);
int  sphk_state_open(const char* path, sphk_state_file** file, char* msg, int msg_len);
void sphk_state_close(sphk_state_file* file);
/* bytes of a named section of an opened file (SPHK_ERR_INVALID: no such section) */
int  sphk_state_section_bytes(const sphk_state_file* file, const char* name, unsigned long long* bytes);
int  sphk_checkpoint_load(sphk_ctx* ctx, const sphk_state_file* file, const sphk_state_config* expect,
                          const sphk_state_section* sections, int n_sections, char* msg, int msg_len);
int  sphk_checkpoint_invalidate(sphk_ctx* ctx);

/* ---- tank motion (no reference counterpart; DESIGN.md section 2.15) ------------------------------------------------------------
 * The simulation frame is the tank's own frame: walls, grid, clamp box and every sweep stay where they are, and the tank's motion
 * enters as a body force.  At t = 0 the tank frame coincides with the world whenever theta(0) = 0.  G is gravity in the world.
 *   rotation about the unit axis n (fixed in the tank) through the pivot p (tank coordinates):
 *     theta(t) = e(t) Theta sin(w t + phi) + theta_s(t),   d theta_s / dt = e(t) Omega0,  theta_s(0) = 0
 *   translation, as the world acceleration of the pivot:
 *     a_w(t) = e(t) (a_c + sum_k A_k sin(w_k t + phi_k)),   k < n_harmonics <= SPHK_TANK_HARMONICS
 *   ramp: e(t) = min(1, t / T_r) (e = 1 when T_r = 0).  With s = sin(w t + phi), c = cos(w t + phi) and, before the ramp's end
 *   (t < T_r), e = t / T_r and e' = 1 / T_r, after it e = 1 and e' = 0:
 *     theta_s = Omega0 t^2 / (2 T_r)                       (t < T_r)
 *             = Omega0 (t - T_r / 2)                       (t >= T_r; Omega0 t when T_r = 0)
 *     thd  = e' Theta s + e Theta w c + e Omega0
 *     thdd = 2 e' Theta w c - e Theta w^2 s + e' Omega0
 * With Omega = thd n, R = Rot(n, -theta) (world vectors in tank axes) and r = x - p, one step of a fluid particle, every quantity
 * at t_n (the start of the step):
 *     v <- Rot(n, -2 thd dt) v + dt (R (G - a_w) - thdd n x r - thd^2 n x (n x r))
 * (Coriolis as an exact rotation of v: it never changes |v|; Euler; centrifugal).  It replaces the gravity kick sphk_gravity.
 * Refused by sphk_tank_set and sphk_tank_eval with SPHK_ERR_INVALID: a NULL pointer (motion NULL is a clear for sphk_tank_set), a
 * non-finite value in the fields in use, |n| = 0, w, w_k or T_r < 0, n_harmonics outside [0, SPHK_TANK_HARMONICS]. */
#define SPHK_TANK_HARMONICS 4
#define SPHK_TANK_STATE 9                   /* theta, thd, thdd, R (G - a_w) (3), a_w (3) */
typedef struct sphk_tank_motion {
    float axis[3];                          /* n, any length > 0 (normalised in double) */
    float pivot[3];                         /* p, tank coordinates */
    float roll_amplitude;                   /* Theta (rad) */
    float roll_omega;                       /* w >= 0 (rad/s) */
    float roll_phase;                       /* phi (rad) */
    float spin;                             /* Omega0 (rad/s) */
    float accel[3];                         /* a_c, world */
    int   n_harmonics;                      /* entries of the three arrays below in use; the rest are ignored */
    float harmonic_amplitude[SPHK_TANK_HARMONICS][3];   /* A_k, world */
    float harmonic_omega[SPHK_TANK_HARMONICS];          /* w_k >= 0 */
    float harmonic_phase[SPHK_TANK_HARMONICS];          /* phi_k */
    float ramp;                             /* T_r >= 0 */
} sphk_tank_motion;
/* Host only, no context: {theta, thd, thdd, R (G - a_w), a_w} at t >= 0, computed in double and rounded to float once -- the one
 * place the schedule is written down.  SPHK_ERR_INVALID also for t < 0 or not finite. */
int sphk_tank_eval(const sphk_tank_motion* motion, const float G[3], double t, float out[SPHK_TANK_STATE]);
/* Host only: a bound on the body force per unit mass over all t,
 *   |G| + |a_c| + sum_k |A_k| + r_max (|Theta| w^2 + (2 |Theta| w + |Omega0|) / T_r + (|Theta| w + |Theta| / T_r + |Omega0|)^2)
 * (the 1 / T_r terms 0 when T_r = 0), r_max = the distance from p to the farthest corner of the clamp box [0, 0.99 space].  It
 * bounds |G - a_w| + |r|_max (|thdd| + thd^2); Coriolis adds no speed.  The |G| of the adaptive step rule while a motion is set. */
int sphk_tank_accel_bound(const sphk_tank_motion* motion, const float G[3], const float space[3], double* bound_out);
/* Sets (NULL: clears) the context's motion; the frame time is kept (0 at the first setting).  Refusals change nothing:
 * SPHK_ERR_INVALID as above; SPHK_ERR_STATE under an active range (slab ranks) and for a rotation (Theta != 0 or Omega0 != 0) when
 * dynamic bodies are declared (a rigid body's angular equation in a rotating frame is not modelled; sphk_bodies_set_dynamics refuses
 * M > 0 under a rotating motion in turn).  The motion is passed to the kernels by value: a captured step graph must be captured again. */
int sphk_tank_set(sphk_ctx* ctx, const sphk_tank_motion* motion, const float G[3]);
/* The step's body force on the live fluid: one single-thread kernel evaluates the schedule in double at the device-resident frame
 * time t_n into the per-step state {Rot(n, -2 thd dt), dt R (G - a_w), thdd dt, thd^2 dt} and advances the frame time by (double)
 * dt (in the stream: a replayed step graph advances it too); one kernel per fluid particle applies the update above to the API
 * velocities and the records.  When the step's thd and thdd are both 0 the particle kernel does exactly sphk_gravity's arithmetic
 * with dt R (G - a_w) as its dt G (zero amplitudes give sphk_gravity's bits).  While a motion is set, sphk_bodies_integrate uses
 * R (G - a_w) of the last sphk_tank_force instead of its G.  SPHK_ERR_STATE without a motion; dt >= 0 and finite. */
int sphk_tank_force(sphk_ctx* ctx, const sphk_scene* scene, float dt);
/* The frame time (synchronises) and, when state_or_null is given, the state of the last sphk_tank_force as sphk_tank_eval gives it
 * (float[SPHK_TANK_STATE], zeros before the first); sphk_tank_set_time enqueues a new frame time (t >= 0, finite: a restore).
 * SPHK_ERR_STATE before the first sphk_tank_set. */
int sphk_tank_time(sphk_ctx* ctx, double* t, float* state_or_null);
int sphk_tank_set_time(sphk_ctx* ctx, double t);

/* ---- render export: generate_dots_CUDA, vbo.cu:26-44 (SURVEY 8f-2) -----------------------------------------------
 * dot[i] = pos[i]; colour[i] from density[i] (blue below 0.75, blend to white at 1.0, blend to pink above).  Plain
 * device buffers instead of a mapped GL vertex buffer; synchronises like the reference (vbo.cu:49). */
int sphk_export_dots(sphk_ctx* ctx, const sphk_particles* p, float* dot_xyz, float* color_rgb);

/* ---- multi-GPU slab support (no reference counterpart: the reference is single-GPU; SURVEY 8e) ----------------
 * A slab rank keeps [ghost-left | owned | ghost-right] particles in one sorted set (cpp-fluid-particles_b200/
 * slabs.py).  Sweeps compute only the active (owned) range; ghost values arrive by halo exchange of the API
 * arrays (contiguous slices) and are mirrored into the packed records. */
/* restrict every subsequent sweep to particles [begin, begin+count) of the fluid set (count<0: all) */
int sphk_set_active_range(sphk_ctx* ctx, int begin, int count);
/* the same with {begin, count} in DEVICE memory, read by the kernels themselves (NULL: back to the host-side range).  The
 * contents may change between sweeps (the neighbour lists are then built for all particles of the set) */
int sphk_set_active_range_device(sphk_ctx* ctx, const int* device_begin_count);
/* copy API data of particles [begin, begin+count) into the packed records: what is a bit mask -- 1: vel
 * (scene->fluid.vel), 2: neighbour scalar from `array` (float[n]), 4: pos (scene->fluid.pos; PBD ghosts moved by
 * their owner: counted against the neighbour-list skin like local moves) */
int sphk_push_range(sphk_ctx* ctx, const sphk_scene* s, int what, const float* array, int begin, int count);

/* The exchanges themselves (csrc/sphk_mg.cu).  One sphk_mg_comm per rank = one process per GPU; a rank talks to
 * ranks rank-1 ("left") and rank+1 ("right") only.  Everything is enqueued on the stream given to sphk_mg_init
 * (must be the sphk_ctx stream) and nothing synchronises the host unless stated.  Transports:
 *   NCCL point-to-point (resolved with dlopen at run time, so it is the process's one NCCL) for the once-per-step
 *   candidate exchange and as fallback; peer-memory mailboxes over NVLink (CUDA IPC) for the per-sweep halos:
 *   one kernel stores the boundary planes into the neighbours' memory, waits for theirs and unpacks them into the
 *   ghost slices and the packed records. */
typedef struct sphk_mg_comm sphk_mg_comm;
/* rank 0 creates the NCCL id; ship the 128 bytes to every rank by any side channel */
int  sphk_mg_unique_id(unsigned char id[128]);
/* collective over all ranks.  mailbox_floats > 0 also allocates this rank's halo mailboxes (payload capacity per
 * message, in floats; MUST be the same number on every rank -- sphk_mg_ipc_connect checks it) */
int  sphk_mg_init(sphk_mg_comm** comm, int rank, int world, const unsigned char id[128], void* stream, long long mailbox_floats);
void sphk_mg_destroy(sphk_mg_comm* comm);
/* CUDA IPC handle of this rank's mailboxes (64 bytes) / open the neighbours' (NULL where there is none) */
int  sphk_mg_ipc_handle(sphk_mg_comm* comm, unsigned char handle[64]);
int  sphk_mg_ipc_connect(sphk_mg_comm* comm, const unsigned char* left_handle64, const unsigned char* right_handle64);
/* halo transport: 0 = NCCL send/recv + sphk_push_range (default), 1 = peer-memory mailboxes (after ipc_connect) */
int  sphk_mg_set_transport(sphk_mg_comm* comm, int transport);
/* up to 8 ints to each neighbour and back (missing neighbour: zeros).  Synchronises the stream. */
int  sphk_mg_exchange_ints(sphk_mg_comm* comm, const int* to_left, const int* to_right, int* from_left, int* from_right, int count);
/* sum of one double over all ranks.  Synchronises the stream. */
int  sphk_mg_allreduce_sum(sphk_mg_comm* comm, double* inout_host);
/* NCCL: for every array a (widths[a] floats per particle) send particles send_left = {begin, count} of send_arrays[a]
 * to the left rank and send_right to the right rank; receive recv_left / recv_right = {begin, count} of
 * recv_arrays[a].  Counts must agree with the neighbours' (exchange them first).  One NCCL group. */
int  sphk_mg_exchange_slices(sphk_mg_comm* comm, int narrays, const float* const* send_arrays, float* const* recv_arrays,
                             const int* widths, const int send_left[2], const int send_right[2],
                             const int recv_left[2], const int recv_right[2]);
/* One halo of a per-particle API array (width 1 or 3 floats): ranges = {first_begin, first_count, last_begin,
 * last_count, ghostL_begin, ghostL_count, ghostR_begin, ghostR_count} in particles -- the first / last owned plane go
 * to the left / right rank, whose planes arrive in the ghost ranges and are mirrored into the packed records as
 * sphk_push_range(what) would (what = 0: an array no record mirrors; 1: array = scene->fluid.vel; 2: neighbour
 * scalar; 4: array = scene->fluid.pos). */
int  sphk_mg_halo(sphk_mg_comm* comm, sphk_ctx* ctx, const sphk_scene* s, int what, float* array, int width, const int ranges[8]);
/* Host-free variants (a slab rank's step without a single host synchronisation):
 * sphk_mg_plane_ranges: from the cell ranges of the freshly sorted local set (cell_start_fluid, plane_cells = cy*cz cells per
 * x-plane, w owned planes + 2 ghost planes) computes on the device, into device_out24: [0..7] the plane offsets, [8..15] the
 * halo ranges in sphk_mg_halo's layout, [16..17] the owned range {begin, count} (-> sphk_set_active_range_device),
 * [18..21] next step's candidate slices, [22..23] their counts (what the neighbours must learn); also copied to pinned host
 * memory for NEXT step's host-side sizing.  sphk_mg_halo_device: sphk_mg_halo with the ranges read from device memory
 * (mailbox transport).  sphk_mg_exchange_ints_async / sphk_mg_check_async: as the synchronising calls, device-resident input,
 * results into pinned host memory when the stream gets there. */
int  sphk_mg_plane_ranges(sphk_mg_comm* comm, const int* cell_start_fluid, int plane_cells, int w, int* device_out24, int* pinned_host_out24);
int  sphk_mg_halo_device(sphk_mg_comm* comm, sphk_ctx* ctx, const sphk_scene* s, int what, float* array, int width,
                         const int* device_ranges8, int max_particles);
int  sphk_mg_exchange_ints_async(sphk_mg_comm* comm, const int* device_to_left, const int* device_to_right, int count,
                                 int* pinned_from_left, int* pinned_from_right);
int  sphk_mg_check_async(sphk_mg_comm* comm, int* pinned_error_bits);
/* mailbox error word (0 = fine; bit 0/1 timed out waiting for left/right; bit 2/3 size mismatch from left/right; bit 4 more
 * strays than the routing capacity, see sphk_mg_strays_route).
 * Synchronises the stream. */
int  sphk_mg_check(sphk_mg_comm* comm, int* error_bits_host);
/* {bytes sent, messages sent} by this rank so far */
int  sphk_mg_stats(const sphk_mg_comm* comm, long long out_host[2]);
/* Strays: owned particles that crossed TWO OR MORE cell planes in x since the last search (the candidate exchange covers
 * one plane per step; the reference's own DFSPH benchmark setting shoots a few hundred particles across tens of planes
 * once the block hits the floor).  They are routed to every rank instead.  `arrays` are the carried per-particle arrays
 * (arrays[0] = positions, width 3; at most 4 arrays of width 1..3); a block is {int count, 3 pad, rows[capacity][sum of
 * widths]} = sphk_strays_block_floats floats.
 *   sphk_strays_collect: over the owned slots [own_begin, own_begin + own_count) of the set sorted by the last search
 *     (cell_start_fluid are ITS cell ranges; call before sphk_set_grid moves the window): rows of the strays into `block`,
 *     their positions out of the world (-1e6: dropped by the next search wherever a copy is held).
 *   sphk_mg_strays_route: all-gathers the blocks (NCCL) into `gathered` (world blocks) and appends world * capacity slots
 *     at dst_begin of `arrays` (the assembled set of the next search): the strays of rank 0, 1, ... -- the same order on
 *     every rank -- unused slots out of the world.  count > capacity (the surplus stayed in place) raises bit 4 of the
 *     error word of sphk_mg_check.  sphk_strays_append: the append alone, for blocks gathered through another channel.
 *   sphk_strays_counts: the per-rank counts of a gathered set (synchronises; introspection). */
long long sphk_strays_block_floats(int capacity, int narrays, const int* widths);
int  sphk_strays_collect(sphk_ctx* ctx, const int* cell_start_fluid, int own_begin, int own_count, int narrays,
                         float* const* arrays, const int* widths, float* block, int capacity);
int  sphk_strays_append(sphk_ctx* ctx, const float* gathered, int world, int capacity, int narrays, float* const* arrays,
                        const int* widths, int dst_begin);
int  sphk_mg_strays_route(sphk_mg_comm* comm, sphk_ctx* ctx, const float* block, float* gathered, int capacity, int narrays,
                          float* const* arrays, const int* widths, int dst_begin);
int  sphk_strays_counts(sphk_ctx* ctx, const float* gathered, int world, int capacity, int narrays, const int* widths, int* counts_host);

/* ---- introspection for parity tests --------------------------------------------------------- */
/* copies the stable-sort permutation of the last fluid search (perm[s] = pre-sort index) to device
 * memory `perm_out` (int[n]) */
int sphk_get_permutation(sphk_ctx* ctx, int* perm_out, int n);
/* raw copy of the current neighbour list (device to device): counts int[n]; entries int[capacity*max_fluid] in
 * the int4-packed layout nbr4[(k/4)*max_fluid + i].{x,y,z,w}.  Either pointer may be NULL. */
int sphk_get_neighbor_list(sphk_ctx* ctx, const sphk_scene* s, int* counts_out, int* entries_out);
/* raw copy of the current tile lists (SPHK_OPT_TILE = 1; device to device), building them first if needed:
 *   counts_out  int[n]: neighbour count, or capacity + 1 for a particle that walks the cells (its tile's windows exceed
 *               the staging capacity, or it lies outside the grid)
 *   slots_out   uint16[8 * ceil(capacity/8) * max_fluid]: batch b of particle i is the 8 slots at (b*max_fluid + i)*8.  A slot
 *               indexes the tile's staged windows (window w holds slots [pre_w, pre_w + count_w), pre_w = sum of the
 *               counts of the windows before it); the dummy slot T = sum of all 18 counts pads the last batch to 8
 *   windows_out int[2 * 18 * ceil(n/128)]: {first record, count} of the 9 fluid then 9 boundary windows of every tile of
 *               128 particles (record index of boundary particle b = max_fluid + b)
 * Any pointer may be NULL. */
int sphk_get_tile_lists(sphk_ctx* ctx, const sphk_scene* s, int* counts_out, unsigned short* slots_out, int* windows_out);
/* largest displacement of any particle since the skin list was built (PBD; synchronises) */
int sphk_get_skin_displacement(sphk_ctx* ctx, float* host_out);
/* neighbour-list statistics of the last build: host ints {max_count, overflow_particles, total} */
int sphk_list_stats(sphk_ctx* ctx, const sphk_scene* s, long long out_host[3]);

#ifdef __cplusplus
}
#endif
#endif /* SPHK_H_ */
