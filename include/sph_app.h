/* sph_app.h -- headless C facade over the reference-shaped C++ class API
 * (SPHSystem / BaseSolver / SPHParticles / DArray).
 *
 * The facade source (cpp-fluid-particles_b200/facade/sph_app.cpp) restates the ONLY call sites of
 * that API in the reference -- initSPHSystem() /root/reference/src/main.cpp:117-134 (particle
 * upload, solver choice, 16-argument SPHSystem constructor) and oneStep() main.cpp:300-306
 * (`float ms = pSystem->step()`) -- without GLUT/OpenGL.  The very same source file is compiled
 *   (1) by g++ against this repository's headers  -> libsphhost.so   (product: the native engine)
 *   (2) by nvcc against /root/reference/src headers + the unmodified reference .cu files
 *                                                 -> oracle/_ref/libsphref.so (parity oracle, B1)
 * which is the drop-in claim made concrete: identical call sites, two engines underneath.
 */
#ifndef SPH_APP_H_
#define SPH_APP_H_
#ifdef __cplusplus
extern "C" {
#endif

typedef struct sph_app sph_app;

typedef struct sph_app_params {
    float space[3];        /* spaceSize                       main.cpp:54  */
    float cell_length;     /* sphCellLength                   main.cpp:57  */
    float radius;          /* sphSmoothingRadius              main.cpp:56  */
    float dt;              /*                                 main.cpp:58  */
    float m0;              /* sphM0                           main.cpp:61  */
    float rho0;            /* sphRho0                         main.cpp:59  */
    float rho_boundary;    /* sphRhoBoundary                  main.cpp:60  */
    float stiff;           /* sphStiff                        main.cpp:62  */
    float visc;            /* sphVisc                         main.cpp:64  */
    float surface_tension; /* sphSurfaceTensionIntensity      main.cpp:65  */
    float air_pressure;    /* sphAirPressure                  main.cpp:66  */
    float gravity[3];      /* sphG                            main.cpp:63  */
    int   cell_size[3];    /* cellSize                        main.cpp:67  */
    int   solver;          /* 0 = BasicSPHSolver, 1 = DFSPHSolver, 2 = PBDSolver (main.cpp:69-71) */
    int   max_iter;        /* <=0: solver constructor default (DFSPHSolver.h:30 / PBDSolver.h:28) */
    float density_error_threshold;    /* DFSPH only; used when max_iter > 0 */
    float divergence_error_threshold; /* DFSPH only; used when max_iter > 0 */
} sph_app_params;

/* Builds SPHParticles for fluid and boundary from host xyz triplets, the chosen solver and the
 * SPHSystem (whose constructor already performs one step, SPHSystem.cu:76).  NULL on failure. */
sph_app* sph_app_create(const float* fluid_xyz, int n_fluid,
                        const float* boundary_xyz, int n_boundary,
                        const sph_app_params* params);
void  sph_app_destroy(sph_app* app);
/* One SPHSystem::step(); returns the milliseconds the system itself reports (SPHSystem.cu:151-157). */
float sph_app_step(sph_app* app);
int   sph_app_fluid_size(const sph_app* app);
int   sph_app_boundary_size(const sph_app* app);
/* Device->host copies through the public accessors (getPosPtr, getVelPtr, getDensityPtr,
 * getPressurePtr, getMassPtr, getParticle2Cell).  Any pointer may be NULL.  Returns 0 on success. */
int   sph_app_download_fluid(sph_app* app, float* pos_xyz, float* vel_xyz, float* density,
                             float* pressure, float* mass, int* particle2cell);
int   sph_app_download_boundary(sph_app* app, float* pos_xyz, float* mass, int* particle2cell);
/* Host->device overwrite of fluid pos / vel through getPosPtr / getVelPtr (either may be NULL).  An adaptive system measures its
 * speed bound again, so the next step's dt sees the uploaded state. */
int   sph_app_upload_fluid(sph_app* app, const float* pos_xyz, const float* vel_xyz);
/* Pipelined host-buffer stepping: one call = "advance the particle state held in HOST memory (pos_in, vel_in) by one
 * SPHSystem::step() and deliver pos / vel / density of the result to HOST memory".  The upload of this batch and the
 * download of the previous result overlap the previous batch's step (copy stream + device staging; the step itself
 * only adds device-to-device copies), so a stream of batches costs one step per batch instead of step + PCIe time.
 * Host buffers should be pinned (cudaHostAlloc / torch pin_memory) and must stay valid until sph_app_wait() returns;
 * results of batch k are complete after the call that submits batch k+2, or after sph_app_wait().  Output pointers
 * may be NULL.  Returns 0 on success. */
int   sph_app_submit(sph_app* app, const float* pos_in_xyz, const float* vel_in_xyz,
                     float* pos_out_xyz, float* vel_out_xyz, float* density_out);
/* Steps every submitted batch that has not run yet and waits for all downloads. */
int   sph_app_wait(sph_app* app);
/* Introspection / switches of this repository's engine (return 1 on the reference build of the facade):
 * iteration counts of the last DFSPH step; option 1 = device-side loop tests for adaptive DFSPH (default on; 0 = the
 * reference's host loop with one error sum read back per iteration), 2 = fused sweeps (default on), 3 = step graph. */
int   sph_app_dfsph_iterations(sph_app* app, int* divergence_iters, int* density_iters);
int   sph_app_set_option(sph_app* app, int option, int value);
/* 1 when the next step replays a captured step graph, 0 when it launches kernels one by one, -1 on the reference build */
int   sph_app_step_graph_active(sph_app* app);
/* Vorticity confinement of strength eps >= 0 in every following step (BasicSPHSolver::setVorticityConfinement; 0 = off,
 * the default).  No reference counterpart: returns 1 on the reference build, and for eps < 0 or NaN. */
int   sph_app_set_vorticity(sph_app* app, float eps);
/* Implicit viscosity in every following step (BasicSPHSolver::setImplicitViscosity; DESIGN.md section 2.5): kinematic viscosity
 * nu of the fluid and nu_boundary against walls and bodies, CG to |b - A v|_M <= tol |b|_M or max_iter iterations; nu = 0 = off
 * (the default).  No reference counterpart: returns 1 on the reference build, for nu or nu_boundary < 0 or not finite,
 * tol <= 0 or NaN, max_iter < 1 or > 1000 (SPHK_IMPLICIT_VISCOSITY_MAX_ITER), and for nu_boundary > 0 in a system with dynamic
 * bodies (the setting is then kept). */
int   sph_app_set_implicit_viscosity(sph_app* app, float nu, float nu_boundary, float tol, int max_iter);
/* iterations and relative residual |r|_M / |b|_M of the last implicit viscosity solve (0, 0 before the first); synchronises;
 * 1 on the reference build */
int   sph_app_viscosity_stats(sph_app* app, int* iterations, float* rel_residual);
/* Non-Newtonian viscosity in every following step (BasicSPHSolver::setRheology; DESIGN.md section 2.9), replacing the
 * constant-nu implicit solve: model 1 = Cross, params {nu0, nu_inf, lambda, m}; 2 = Herschel-Bulkley, params {K, n, tau_y, m_reg}
 * (6 floats, the unused ones 0); nu clamped to [nu_min, nu_max]; walls and bodies act with boundary_factor * nu_i.  model 0 = off.
 * Returns 1 on the reference build and for a setting the class layer refuses (the setting is then kept). */
int   sph_app_set_rheology(sph_app* app, int model, const float* params, float nu_min, float nu_max, float boundary_factor,
                           float tol, int max_iter);
/* of the last non-Newtonian solve (zeros before the first): iterations, |r|_M / |b|_M, max shear rate, min / max nu, particles at
 * the nu_max clamp (any pointer may be NULL); synchronises; 1 on the reference build */
int   sph_app_rheology_stats(sph_app* app, int* iterations, float* rel_residual, float* gamma_max, float* nu_min, float* nu_max,
                             int* n_at_max);
/* nu_i of the last non-Newtonian solve (float[fluid size]; zeros before the first); 1 on the reference build */
int   sph_app_download_viscosity(sph_app* app, float* nu_host);
/* Heat transfer in every following step (BasicSPHSolver::setThermal; DESIGN.md section 2.10): diffusivity alpha, buoyancy
 * dv = -beta (T - t_ref) G dt, the static walls at wall_t with conductance wall_h (0: adiabatic), body b at body_t_h[2b] with
 * conductance body_t_h[2b+1], emitter k's particles at emitter_t[k] (missing: t_ref).  on = 0: off.  Returns 1 on the reference
 * build and for a setting the class layer refuses (the setting is then kept). */
int   sph_app_set_thermal(sph_app* app, int on, float alpha, float beta, float t_ref, float wall_t, float wall_h, int n_bodies,
                          const float* body_t_h, int n_emitters, const float* emitter_t);
/* nu = clamp(nu_ref exp(-e (T - t_ref)), nu_min, nu_max) solved instead of the constant-nu solve while heat transfer is on
 * (BasicSPHSolver::setThermalViscosity); on = 0: off.  1 on the reference build and for a refused setting. */
int   sph_app_set_thermal_viscosity(sph_app* app, int on, float nu_ref, float e, float nu_min, float nu_max, float wall_factor,
                                    float tol, int max_iter);
/* the fluid's temperatures (float[fluid size], the fluid's current order); 1 on the reference build */
int   sph_app_upload_temperature(sph_app* app, const float* t_host);
int   sph_app_download_temperature(sph_app* app, float* t_host);
/* conduction substeps, largest dt_k sum c_ij and particle-substeps above 1 of the last step; min, max and sum m T of the current
 * temperatures (any pointer may be NULL); synchronises; 1 on the reference build */
int   sph_app_thermal_stats(sph_app* app, int* substeps, float* max_courant, int* violators, float* t_min, float* t_max, double* heat);
/* Fluid-solid adhesion in every following step (BasicSPHSolver::setAdhesion; DESIGN.md section 2.11): beta of the static walls
 * (wall) and of body b (body_beta[b], b < n_bodies; bodies past n_bodies do not adhere).  on = 0: off.  Returns 1 on the
 * reference build and for a setting the class layer refuses (the setting is then kept). */
int   sph_app_set_adhesion(sph_app* app, int on, float wall, int n_bodies, const float* body_beta);
/* wetted particles and the largest |a_i| of the last step's adhesion sweep (either pointer may be NULL); synchronises; 1 on the
 * reference build */
int   sph_app_adhesion_stats(sph_app* app, int* wetted, float* max_accel);
/* Probes and water-level gauges (SPHSystem::setProbes; DESIGN.md section 2.13): from the next step on every step records the
 * records {S, rho, vx, vy, vz, p, T, n} of n_points points (points_xyz: float[3 n_points]) and the levels of n_gauges gauges
 * (gauge_ab: float[6 n_gauges] = {a.xyz, b.xyz}, gauge_samples: int[n_gauges]) into a ring of `capacity` rows.  n_points = n_gauges
 * = 0: off.  Returns 1 on the reference build and for a setting the class layer refuses (the setting is then kept). */
int   sph_app_set_probes(sph_app* app, int n_points, const float* points_xyz, int n_gauges, const float* gauge_ab,
                         const int* gauge_samples, float threshold, int capacity);
/* The recorded rows still in the ring, oldest first (synchronises).  With steps, times, records and levels all NULL: only the counts
 * (*rows, *n_points, *n_gauges, *overwritten); otherwise also steps[rows] (the step index), times[rows] (simulated time after the
 * step), records[rows][n_points][8] and levels[rows][n_gauges] -- arrays sized from a count query made since the last step.  Any
 * count pointer may be NULL.  1 on the reference build. */
int   sph_app_probe_series(sph_app* app, int* rows, int* n_points, int* n_gauges, long long* overwritten, long long* steps,
                           double* times, float* records, float* levels);
/* On demand, between steps (synchronise): records of n points (float[3 n]) into out (float[8 n]); records of the lattice origin +
 * spacing (i, j, k), z fastest, into out (float[8 nx ny nz]).  1 for a refused call and on the reference build. */
int   sph_app_sample_probes(sph_app* app, int n, const float* points_xyz, float* out);
int   sph_app_sample_lattice(sph_app* app, const float* origin, float spacing, const int* dims, float* out);
/* Checkpoints (SPHSystem::checkpoint / waitCheckpoint / restore; DESIGN.md section 2.14).  sph_app_checkpoint enqueues the snapshot
 * of the state and returns; the file (path.tmp, fsync, rename) is written behind the following steps, and sph_app_checkpoint_wait
 * reports it.  A checkpoint taken while a pipelined sph_app_submit step is in flight holds the state after that step (stream order).
 * user: user_bytes opaque bytes stored with the state (NULL / 0: none).  sph_app_restore overwrites the state of a system built with
 * the same configuration; user_out (capacity user_cap, may be NULL) receives the stored user bytes and *user_bytes their count.  1
 * for a refused call (printed; a refused restore changes nothing) and on the reference build. */
int   sph_app_checkpoint(sph_app* app, const char* path, const void* user, int user_bytes);
int   sph_app_checkpoint_wait(sph_app* app);
int   sph_app_restore(sph_app* app, const char* path, void* user_out, int user_cap, int* user_bytes);
/* Tank motion (SPHSystem::setTankMotion; DESIGN.md section 2.15): the system runs in the frame of a tank rolled about `axis` through
 * `pivot` (theta = e roll_amplitude sin(roll_omega t + roll_phase) + spin integrated), shaken (pivot acceleration e (accel + sum_k
 * harmonic_amplitude[k] sin(harmonic_omega[k] t + harmonic_phase[k])), k < n_harmonics <= 4, in the world) and ramped in over
 * `ramp` seconds (e = min(1, t / ramp)), t the simulated time.  The layout is sphk_tank_motion's.  NULL: off.  Returns 1 on the
 * reference build and for a setting the class layer refuses (out-of-range values, heat transfer, a rotation with dynamic bodies;
 * the setting is then kept). */
typedef struct sph_app_tank_motion {
    float axis[3];
    float pivot[3];
    float roll_amplitude, roll_omega, roll_phase;
    float spin;
    float accel[3];
    int   n_harmonics;
    float harmonic_amplitude[4][3];
    float harmonic_omega[4];
    float harmonic_phase[4];
    float ramp;
} sph_app_tank_motion;
int   sph_app_set_tank_motion(sph_app* app, const sph_app_tank_motion* motion);
/* The motion at the simulated time *t (SPHSystem::tankState): state9 = {theta, theta', theta'', a_w.xyz (world), R (G - a_w).xyz
 * (tank axes)}; G and zeros without a motion.  Either pointer may be NULL; 1 on the reference build. */
int   sph_app_tank_state(sph_app* app, double* t, float* state9);
/* Kinematic rigid bodies (SPHSystem's constructor with a vector of sphb200::KinematicBody; DESIGN.md section 2.3).  No
 * reference counterpart: NULL / 1 on the reference build.  Body b is the points body_xyz[body_begin[b] .. body_begin[b+1])
 * (body coordinates; body_begin[0] = 0), pose[7 b ..] = {cx, cy, cz, qx, qy, qz, qw} (quaternion scalar part last),
 * motion[6 b ..] = {Vx, Vy, Vz, Ox, Oy, Oz} in the world frame.  The boundary set of the system is the static boundary_xyz
 * followed by the bodies' particles (sph_app_boundary_size and sph_app_download_boundary include them).  n_bodies = 0 is
 * sph_app_create.  NULL on failure, including bodies the engine refuses (more than 64, non-finite pose or motion). */
sph_app* sph_app_create_with_bodies(const float* fluid_xyz, int n_fluid, const float* boundary_xyz, int n_boundary,
                                    int n_bodies, const int* body_begin, const float* body_xyz, const float* pose,
                                    const float* motion, const sph_app_params* params);
/* new motion of one body from the next step on (SPHSystem::setBodyMotion); 1 for a bad index or non-finite values */
int   sph_app_set_body_motion(sph_app* app, int body, const float* linear_velocity_xyz, const float* angular_velocity_xyz);
/* current pose of one body, float[7] as above (synchronises) */
int   sph_app_body_pose(sph_app* app, int body, float* pose);
/* Two-way coupled rigid bodies (DESIGN.md section 2.4): sph_app_create_with_bodies plus mass_inertia[4 b ..] = {M, Ix, Iy, Iz}
 * per body (sphb200::KinematicBody::mass and ::inertia; principal moments about the centre in the axes of body_xyz).  M > 0
 * makes a body dynamic (the fluid pushes it; gravity and wall contact apply) and needs I > 0; M = 0 keeps it kinematic and
 * its reaction is still reported.  Masses are in the fluid's units: m0 / spacing^3 per unit volume (not rho0).  NULL on the
 * reference build and when the engine refuses the bodies or their dynamics. */
sph_app* sph_app_create_with_dynamic_bodies(const float* fluid_xyz, int n_fluid, const float* boundary_xyz, int n_boundary,
                                            int n_bodies, const int* body_begin, const float* body_xyz, const float* pose,
                                            const float* motion, const float* mass_inertia, const sph_app_params* params);
/* current motion of one body, float[6] = {V, Omega} (the integrated one for a dynamic body); synchronises */
int   sph_app_body_motion(sph_app* app, int body, float* motion);
/* {Jx, Jy, Jz, Hx, Hy, Hz}: the impulse and angular impulse about the centre the fluid gave one body over the last step
 * (zero without dynamic bodies); synchronises */
int   sph_app_body_impulse(sph_app* app, int body, float* impulse);
/* Open boundaries (SPHSystem's constructor with sphb200::OpenBoundaries; DESIGN.md section 2.6): emitters add fluid particles and
 * sinks remove them, so the live count (sph_app_fluid_size, and the count the download / upload calls copy) changes between
 * steps.  An emitter is a rectangular nozzle: `width` x `height` particles `spacing` apart in the plane normal to `direction`,
 * centred on `origin`, moving at speed * normalize(direction); one layer enters every time the stream has advanced by one
 * spacing.  A sink is the box lo <= x < hi, sinks_lo_hi[6 k ..] = {lo.xyz, hi.xyz}.  max_fluid (>= n_fluid) is the capacity of
 * the fluid set: a layer that does not fit is refused.  No bodies.  NULL on failure, including emitters or sinks the class layer
 * refuses (invalid values, more than 16 of either, a layer outside the clamp box [0, 0.99 space]), and on the reference build.
 * sph_app_submit returns 1 for such a system (its pipelining assumes a fixed count). */
typedef struct sph_app_emitter {
    float origin[3];
    float direction[3];
    float speed;
    float spacing;
    int   width, height;
} sph_app_emitter;
sph_app* sph_app_create_open(const float* fluid_xyz, int n_fluid, int max_fluid, const float* boundary_xyz, int n_boundary,
                             int n_emitters, const sph_app_emitter* emitters, int n_sinks, const float* sinks_lo_hi,
                             const sph_app_params* params);
/* cumulative particle counts {emitted, removed, refused} (zeros for a closed system) and, when check_bits is not NULL, the sticky
 * bits of the per-step count check (0 = fine; 1 = after some step the in-grid particles were not exactly the live ones, e.g. a live
 * particle uploaded outside the grid); synchronises for the bits; 1 on the reference build */
int   sph_app_open_boundary_stats(sph_app* app, long long* stats3, int* check_bits);
/* CFL-adaptive time stepping (SPHSystem::setAdaptiveTimeStep; DESIGN.md section 2.8): from the next step on, every step runs at
 * dt = C R / (v_max + |G| dt_prev) clamped to [dt_min, dt_max] (0 = the defaults: dt_max = params.dt, dt_min = dt_max / 64), v_max
 * the speed bound of fluid, bodies and emitters the previous step left on the device.  C = 0 turns it off again (back to params.dt).
 * Returns 1 on the reference build and for values the class layer refuses (C < 0, non-finite or negative values, dt_min > dt_max,
 * dt_max above params.dt in a system with emitters;
 * the setting is then kept).  An adaptive system never captures a step graph, and sph_app_submit returns 1 for it. */
int   sph_app_set_adaptive_dt(sph_app* app, float C, float dt_min, float dt_max);
/* CFL substeps until frame_seconds (> 0) of simulated time have passed (SPHSystem::advance): their count and smallest dt (either
 * pointer may be NULL).  1 for a system that is not adaptive, a frame that is not finite and > 0, and on the reference build. */
int   sph_app_advance(sph_app* app, double frame_seconds, int* substeps, float* min_dt);
/* speed_dt3 = {the speed bound the last dt was chosen from, the last dt, the smallest dt of the last sph_app_advance}, *source = what
 * set the bound (0 fluid, 1 body, 2 emitter), counts2 = {steps held at dt_min, steps with non-finite velocities or bound},
 * *simulated_time = the double sum of the float dt of every step.  Any pointer may be NULL; 1 on the reference build. */
int   sph_app_adaptive_stats(sph_app* app, float* speed_dt3, int* source, long long* counts2, double* simulated_time);
/* Scenes from triangle meshes (DESIGN.md section 2.12): the class layer's Wavefront OBJ reader (sphb200::loadObj: v, and f with
 * i, i/j, i//k, i/j/k items, negative indices and fan-triangulated polygons), vertices mapped by scale * v + t (sphk_mesh_transform).
 * Host only, no device.  v: float[3 v_cap], tri: int[3 t_cap] (0-based).  0: read, *nv / *nt set; 2: read, but *nv > v_cap or
 * *nt > t_cap -- the counts are set and nothing is written; 1: refused (an unreadable file, a malformed number or index; the
 * message, naming the line, is sph_app_load_obj_error(): valid until the thread's next call) or the reference build. */
int   sph_app_load_obj(const char* path, float scale, const float* t, float* v, int v_cap, int* tri, int t_cap, int* nv, int* nt);
const char* sph_app_load_obj_error(void);
/* Name of the engine underneath: "reference-cuda" or "b200-native". */
const char* sph_app_engine(void);

#ifdef __cplusplus
}
#endif
#endif /* SPH_APP_H_ */
