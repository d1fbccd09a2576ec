// sphk_sweeps.cu -- the per-particle neighbour sweeps of the three solvers + element-wise steps.
//
// One generic sweep driver, instantiated per operator:
//   * k_sweep_cells<Op> : walks the 27 neighbour cells row by row: the three z-neighbours of a (dx,dy) row are consecutive
//     cell indices, hence ONE contiguous particle range per row; rows in the reference's order (dx outermost), inside a
//     row first the fluid range, then the boundary range.  (The reference interleaves fluid and boundary per CELL,
//     SURVEY 2.2: the difference is the position of a few boundary terms inside a sum, ~1e-7 relative.)
//   * k_sweep_list<Op>  : walks a per-step neighbour list (built once per neighbour search by the same row walk, candidates
//     kept in that order) while positions are unchanged -- the ~85% of candidate pairs outside the support are tested once
//     per step instead of once per sweep (DFSPH runs 20 sweeps per step on identical positions).
//   * k_sweep_tile<Op>  : the same over tile lists (neighbour windows staged in shared memory by bulk copies; option).
// Data path (DESIGN.md 4.1): the sweeps are bound by the gather path -- L1 misses on scattered
// 16-byte records -- and, for the 16-byte sweeps, increasingly by FP32 issue; not by HBM.  Hence:
//   - a neighbour is two 16-byte halves in two arrays, A = {x,y,z,s} and B = {vx,vy,vz,m}; operators that need only
//     position + scalar gather A (one LDG.E.128), the others A and B;
//   - list indices arrive four at a time in one coalesced, streaming (evict-first) 16-byte load, the next batch is prefetched;
//   - accumulation is in registers (the reference accumulates density in global memory, BasicSPHSolver.cu:37,48); kernel
//     constants are folded per launch; selects instead of branches; the non-uniform-mass case sits behind one warp-uniform
//     branch per particle.
// Sums are formed row by row in the candidate order above; results agree with the reference kernels to ~1e-6 relative
// (tests/, <= 1e-5 required).  Compiled with -use_fast_math like the reference (Q10).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <algorithm>
#include <cmath>
#include <math_constants.h>
#include <cooperative_groups.h>
#include <cooperative_groups/reduce.h>
#include "sphk_internal.cuh"

// =================================================================================================
// Operators.  Acc = per-particle register accumulator.
//   begin(acc, i, lo_i, hi_i)                     lo = {x,y,z,s}, hi = {vx,vy,vz,m} of particle i
//   pair (acc, i, j, isB, d, r2, mj, lo_j, hi_j)  d = x_i - x_j; mj = mass_j; j unified index (boundary b = capF + b)
//   end  (acc, i, lo_i, hi_i)
// kHi: the operator reads the velocity of its neighbours -> 256-bit gather; else 128-bit (position + scalar).
// Boundary records carry v = 0 and s = 0, so "v_i - v_j", "kappa_i + kappa_j", "p_i/rho_i^2 + p_j/rho_j^2"
// evaluate the reference's boundary terms without a separate code path (x - 0 and x + 0 are exact).
// =================================================================================================

// computeDensity_CUDA, BasicSPHSolver.cu:32-72
struct OpDensity {
    float* density;
    static constexpr bool kFluidOnly = false, kHi = false;
    struct Acc { float rho; template <class F> __device__ void sums(F f) { f(rho); } };
    __device__ void begin(Acc& a, int, float4, float4, const DevScene&) const { a.rho = 0.f; }
    __device__ void pair(Acc& a, int, int, bool, float3, float r2, float mj, float4 lo, float4, const DevScene& s) const {
        a.rho += mj * w_cubic(sqrtf(r2), s.k);
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const { density[i] = a.rho; }
};

// pressureForce_CUDA, BasicSPHSolver.cu:113-165.  rec.s = p / max(eps, rho^2), precomputed per particle
// (identical value to the reference's per-pair expression); the particle's own value comes from its record.
struct OpPressureForce {
    Rec rec; float* vel; float dt;
    static constexpr bool kFluidOnly = false, kHi = false;
    struct Acc { float3 a; float pri; template <class F> __device__ void sums(F f) { f(a.x); f(a.y); f(a.z); } };
    __device__ void begin(Acc& a, int, float4 lo, float4, const DevScene&) const { a.a = f3(0, 0, 0); a.pri = lo.w; }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        // `i != j` of BasicSPHSolver.cu:120 is implied: the self pair has d = 0 and contributes 0
        a.a += -mj * (a.pri + lo.w) * (d * grad_w_factor(sqrtf(r2), s.k));
    }
    __device__ void end(Acc& a, int i, float4, float4 hi, const DevScene&) const {
        float3 acc = a.a;
        const float l2 = dot3(acc, acc);
        if (sqrtf(l2) > SPHK_MAX_A) acc = acc * rsqrtf(l2) * SPHK_MAX_A;      // :160-161
        const float3 v = f3(hi.x + acc.x * dt, hi.y + acc.y * dt, hi.z + acc.z * dt);
        rec_set_vel(rec + i, v); store3(vel, i, v);
    }
};

// viscosity_CUDA + vel += deltaV, BasicSPHSolver.cu:183-225.  Jacobi: new velocities go to a temp.
struct OpViscosity {
    float4* velNew; float* vel; float* deltaV; float rho0, visc, dt;
    static constexpr bool kFluidOnly = true, kHi = true;
    struct Acc { float3 a; float3 vi; template <class F> __device__ void sums(F f) { f(a.x); f(a.y); f(a.z); } };
    __device__ void begin(Acc& a, int, float4, float4 hi, const DevScene&) const { a.a = f3(0, 0, 0); a.vi = xyz(hi); }
    __device__ void pair(Acc& a, int, int, bool, float3, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        a.a += mj * ((xyz(hi) - a.vi) / rho0) * lap_visc(sqrtf(r2), s.k);
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const {
        const float3 dv = visc * a.a * dt;
        store3(deltaV, i, dv);
        const float3 v = a.vi + dv;
        velNew[i] = make_float4(v.x, v.y, v.z, 0.f); store3(vel, i, v);
    }
};

// computeColorGrad_CUDA, BasicSPHSolver.cu:277-318
struct OpColorGrad {
    float* colorGrad; float rho0, rhoB;
    static constexpr bool kFluidOnly = false, kHi = false;
    struct Acc { float3 num; float den; template <class F> __device__ void sums(F f) { f(num.x); f(num.y); f(num.z); f(den); } };
    __device__ void begin(Acc& a, int, float4, float4, const DevScene&) const { a.num = f3(0, 0, 0); a.den = 0.f; }
    __device__ void pair(Acc& a, int, int, bool isB, float3 d, float r2, float mj, float4 lo, float4, const DevScene& s) const {
        const float r = sqrtf(r2);
        const float V = mj / (isB ? rhoB : rho0);
        a.num += V * (d * grad_w_factor(r, s.k));
        a.den += V * w_cubic(r, s.k);
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const { store3(colorGrad, i, a.num / fmaxf(SPHK_EPS, a.den)); }
};

// surfaceTensionAndAirPressure_CUDA, BasicSPHSolver.cu:332-370.  rec.s = dot(c, c) precomputed.
struct OpSurface {
    Rec rec; float* vel; float dt, rho0, kappa, airP;
    static constexpr bool kFluidOnly = true, kHi = false;
    struct Acc { float3 a; float cii, ratio; template <class F> __device__ void sums(F f) { f(a.x); f(a.y); f(a.z); } };
    __device__ void begin(Acc& a, int, float4 lo, float4, const DevScene&) const {
        a.a = f3(0, 0, 0);
        a.cii = lo.w;
        const float lci = sqrtf(lo.w);
        a.ratio = lci / fmaxf(SPHK_EPS, lci);       // "disable inner particles", :349
    }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        const float r = sqrtf(r2);
        const float mr = mj / (rho0 * rho0);
        a.a += 0.25f * mr * kappa * (a.cii + lo.w) * (d * grad_st_factor(r, s.k));
        a.a += airP * mr * (d * grad_w_factor(r, s.k)) * a.ratio;
    }
    __device__ void end(Acc& a, int i, float4, float4 hi, const DevScene&) const {
        const float3 v = f3(hi.x + a.a.x * dt, hi.y + a.a.y * dt, hi.z + a.a.z * dt);
        rec_set_vel(rec + i, v); store3(vel, i, v);
    }
};

// computeDensityAlpha_CUDA, DFSPHSolver.cu:212-249
struct OpDensityAlpha {
    float* density; float* alpha;
    static constexpr bool kFluidOnly = false, kHi = false;
    struct Acc { float den, lam; float3 gs; template <class F> __device__ void sums(F f) { f(den); f(lam); f(gs.x); f(gs.y); f(gs.z); } };
    __device__ void begin(Acc& a, int, float4, float4, const DevScene&) const { a.den = 0.f; a.lam = 0.f; a.gs = f3(0, 0, 0); }
    __device__ void pair(Acc& a, int, int, bool isB, float3 d, float r2, float mj, float4 lo, float4, const DevScene& s) const {
        const float r = sqrtf(r2);
        a.den += mj * w_cubic(r, s.k);
        const float3 mg = mj * (d * grad_w_factor(r, s.k));
        a.gs += mg;
        a.lam += isB ? 0.0f : dot3(mg, mg);         // boundary excluded from the second term, :218
    }
    __device__ static float alpha_of(const Acc& a) { return -1.0f / fmaxf(SPHK_EPS, dot3(a.gs, a.gs) + a.lam); }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const {
        density[i] = a.den;
        alpha[i] = alpha_of(a);
    }
};

// computeDivergenceError_CUDA (DFSPHSolver.cu:261-306, kDensity=false) and computeDensityError_CUDA
// (:74-116, kDensity=true; optionally with the warm-stiffness accumulate of :199-203 fused).
// Writes the stiffness into rec.s as well: the following correct sweep gathers it with the positions.
template <bool kDensity> struct OpDfsphError {
    Rec rec; const float* density; const float* alpha; float* error; float* stiff; float* warm;
    float dt, rho0;
    static constexpr bool kFluidOnly = false, kHi = true;
    struct Acc { float e; float3 vi; bool quiet; template <class F> __device__ void sums(F f) { f(e); } };
    __device__ void begin(Acc& a, int, float4, float4 hi, const DevScene&) const { a.e = 0.f; a.vi = xyz(hi); }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        a.e += mj * dot3(a.vi - xyz(hi), d * grad_w_factor(sqrtf(r2), s.k));
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const { finish(a, i, density[i], alpha[i]); }
    // the epilogue with the particle's density and alpha given (the fused sweep passes the values it has just formed)
    __device__ void finish(Acc& a, int i, float rho_i, float alpha_i) const {
        float e;
        if (kDensity) e = fmaxf(0.0f, dt * a.e + rho_i - rho0);
        else {
            e = fmaxf(0.0f, a.e);
            if (rho_i + dt * e < rho0 && rho_i <= rho0) e = 0.0f;     // :302-303
        }
        error[i] = e;
        const float k = e * alpha_i;
        stiff[i] = k;
        rec_set_s(rec + i, k);
        if (kDensity && warm) warm[i] += k;
        // Quiet (chunk activity): e = +0 and kappa = -0, the state of every particle whose density and divergence errors are
        // clamped to zero.  fmaxf(0, x) compiles to FMNMX.FTZ against RZ: +0 for every x <= 0 and for NaN; alpha = -1 / max(eps, .)
        // is negative and finite, so kappa = (+0) * alpha = -0.  Then:  warm += kappa  leaves warm unchanged bit for bit
        // (x + -0 = x for every x), and the particle adds an exact zero to every correct-sweep pair term it takes part in.
        a.quiet = __float_as_uint(e) == 0u && __float_as_uint(k) == 0x80000000u;
    }
};

// correctDivergenceError_CUDA (DFSPHSolver.cu:308-329) / correctDensityError_CUDA (:118-158);
// computeDeltaPos_CUDA (PBDSolver.cu:170-210) shares the pair term with lambda as the scalar.  Reads rec.s.
template <int kMode /*0: vel += a, 1: vel += a/dt, 2: deltaPos = a/rho0*/> struct OpScalarGradient {
    Rec rec; float* vel; float* deltaPos; float dt_or_rho0;
    static constexpr bool kFluidOnly = false, kHi = false;
    struct Acc { float3 a; float ki; template <class F> __device__ void sums(F f) { f(a.x); f(a.y); f(a.z); } };
    __device__ void begin(Acc& a, int, float4 lo, float4, const DevScene&) const { a.a = f3(0, 0, 0); a.ki = lo.w; }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        a.a += mj * (a.ki + lo.w) * (d * grad_w_factor(sqrtf(r2), s.k));
    }
    __device__ float3 velocity(float3 sum, float4 hi) const {
        const float3 dv = (kMode == 1) ? sum / dt_or_rho0 : sum;
        return f3(hi.x + dv.x, hi.y + dv.y, hi.z + dv.z);
    }
    __device__ void end(Acc& a, int i, float4, float4 hi, const DevScene&) const {
        if (kMode == 2) { store3(deltaPos, i, a.a / dt_or_rho0); return; }
        const float3 v = velocity(a.a, hi);
        rec_set_vel(rec + i, v); store3(vel, i, v);
    }
    // The epilogue on the +0 sum of a skipped walk (chunk activity), storing only what differs in bits from what is stored --
    // a -0 component, a NaN payload, a velocity that differs from its record: the arrays end up as after end(), and afterwards
    // hold a fixed point of it when the +0 sum adds +0 (quiet_adds_zero): x + 0 = x for every x but -0, and a NaN stays one.
    __device__ void end_quiet(int i) const {
        const float4 hi = *(rec + i).b;
        const float3 u = load3(vel, i);
        const float3 v = velocity(f3(0.f, 0.f, 0.f), hi);
        if (!same_bits3(v, xyz(hi))) rec_set_vel(rec + i, v);
        if (!same_bits3(v, u)) store3(vel, i, v);
    }
    bool quiet_adds_zero() const { return kMode == 0 || (std::isnormal(dt_or_rho0) && dt_or_rho0 > 0.f); }   // host: +0 / dt = +0
};

// computeDensityLambda_CUDA, PBDSolver.cu:127-168 (rho0 passed through `bool`, Q4).  Writes lambda to rec.s.
struct OpPbdLambda {
    Rec rec; float* density; float* lambda; float rho0, rho0AsBool, relaxation;
    static constexpr bool kFluidOnly = false, kHi = false;
    struct Acc { float den, lam; float3 gs; template <class F> __device__ void sums(F f) { f(den); f(lam); f(gs.x); f(gs.y); f(gs.z); } };
    __device__ void begin(Acc& a, int, float4, float4, const DevScene&) const { a.den = 0.f; a.lam = 0.f; a.gs = f3(0, 0, 0); }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float r2, float mj, float4 lo, float4, const DevScene& s) const {
        const float r = sqrtf(r2);
        a.den += mj * w_cubic(r, s.k);
        const float3 g = -mj * (d * grad_w_factor(r, s.k)) / rho0AsBool;
        a.gs -= g;
        a.lam += dot3(g, g);
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const {
        density[i] = a.den;
        float l = (a.den > rho0) ? (-(a.den / rho0 - 1.0f) / (dot3(a.gs, a.gs) + a.lam + SPHK_EPS)) : 0.0f;
        l *= relaxation;
        lambda[i] = l;
        rec_set_s(rec + i, l);
    }
};

// XSPHViscosity_CUDA, PBDSolver.cu:89-115, Jacobi: new velocities go to a temp (the reference races, Q5)
struct OpXsph {
    float4* velNew; float c, rho0;
    static constexpr bool kFluidOnly = true, kHi = true;
    struct Acc { float3 a; float3 vi; template <class F> __device__ void sums(F f) { f(a.x); f(a.y); f(a.z); } };
    __device__ void begin(Acc& a, int, float4, float4 hi, const DevScene&) const { a.a = f3(0, 0, 0); a.vi = xyz(hi); }
    __device__ void pair(Acc& a, int, int, bool, float3, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        a.a += mj * (xyz(hi) - a.vi) * w_cubic(sqrtf(r2), s.k);
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const {
        const float3 v = a.vi + c * a.a / rho0;
        velNew[i] = make_float4(v.x, v.y, v.z, 0.f);
    }
};

// neighbour-list builder: keeps every candidate with r^2 <= r2cut in the cell walk's order, self excluded
// (the self pair contributes exactly 0 to every operator: W(0)=0 by Q1, d = 0, v_i - v_i = 0).
struct OpBuildList {
    int* nbr; int* cnt; float4* posBuild;
    static constexpr bool kFluidOnly = false, kHi = false;
    struct Acc { int n; template <class F> __device__ void sums(F) {} };
    __device__ void begin(Acc& a, int, float4, float4, const DevScene&) const { a.n = 0; }
    // layout: entries 4b..4b+3 of particle i form the int4 at nbr4[b * stride + i] (one coalesced LDG.128 per
    // batch of four neighbours in the walk)
    __device__ size_t slot(int n, int i, const DevScene& s) const {
        return (static_cast<size_t>(n >> 2) * s.nbrStride + i) * 4 + (n & 3);
    }
    __device__ void pair(Acc& a, int i, int j, bool, float3, float, float mj, float4, float4, const DevScene& s) const {
        if (j == i) return;
        if (a.n < s.kmax) nbr[slot(a.n, i, s)] = j;
        ++a.n;
    }
    __device__ void end(Acc& a, int i, float4 lo, float4, const DevScene& s) const {
        cnt[i] = a.n;
        // pad the last batch with the particle itself: the self pair contributes exactly 0 to every operator
        for (int n = a.n; (n & 3) && n < s.kmax; ++n) nbr[slot(n, i, s)] = i;
    }
};

// Two operators in one sweep: every neighbour record is gathered once and fed to both.  Each operator keeps its
// own accumulators and sees exactly the pairs it would see alone (a fluid-only operator is not shown boundary
// neighbours), so each quantity is formed by the same operations in the same order as in its own sweep.
template <class A, class B> struct OpPair {
    A a; B b;
    static constexpr bool kFluidOnly = A::kFluidOnly && B::kFluidOnly, kHi = A::kHi || B::kHi;
    struct Acc {
        typename A::Acc a; typename B::Acc b;
        template <class F> __device__ void sums(F f) { a.sums(f); b.sums(f); }
    };
    __device__ void begin(Acc& c, int i, float4 lo, float4 hi, const DevScene& s) const { a.begin(c.a, i, lo, hi, s); b.begin(c.b, i, lo, hi, s); }
    __device__ void pair(Acc& c, int i, int j, bool isB, float3 d, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        if (!(A::kFluidOnly && isB)) a.pair(c.a, i, j, isB, d, r2, mj, lo, hi, s);
        if (!(B::kFluidOnly && isB)) b.pair(c.b, i, j, isB, d, r2, mj, lo, hi, s);
    }
    __device__ void end(Acc& c, int i, float4 lo, float4 hi, const DevScene& s) const { a.end(c.a, i, lo, hi, s); b.end(c.b, i, lo, hi, s); }
};

// density / alpha (+ colour gradient when kColorGrad) and the divergence error in one sweep.  The error's epilogue takes the
// particle's density and alpha from the registers they were formed in.  Reading them back from the arrays the same sweep
// has just written is not safe: nvcc compiled those reads of the cell-walk instantiation as read-only loads issued before
// the stores (LDG.E.CONSTANT), so the stiffness was formed with the alpha of the previous call.
template <bool kColorGrad> struct OpDensityAlphaDivError {
    using DA = typename std::conditional<kColorGrad, OpPair<OpDensityAlpha, OpColorGrad>, OpDensityAlpha>::type;
    using P = OpPair<DA, OpDfsphError<false>>;
    P p;
    static constexpr bool kFluidOnly = P::kFluidOnly, kHi = P::kHi;
    using Acc = typename P::Acc;
    __device__ void begin(Acc& c, int i, float4 lo, float4 hi, const DevScene& s) const { p.begin(c, i, lo, hi, s); }
    __device__ void pair(Acc& c, int i, int j, bool isB, float3 d, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        p.pair(c, i, j, isB, d, r2, mj, lo, hi, s);
    }
    __device__ void end(Acc& c, int i, float4 lo, float4 hi, const DevScene& s) const {
        p.a.end(c.a, i, lo, hi, s);
        const OpDensityAlpha::Acc* da;
        if constexpr (kColorGrad) da = &c.a.a; else da = &c.a;
        p.b.finish(c.b, i, da->den, OpDensityAlpha::alpha_of(*da));
    }
};

// Roles in chunk activity (k_sweep_list): the DFSPH error sweeps produce the record scalar kappa and report whether each
// particle left it quiet; the DFSPH correct sweeps consume it.  PBD's lambda sweeps (OpScalarGradient<2>) take no part.
enum { kActNone = 0, kActError = 1, kActCorrect = 2 };
struct act_never_quiet { template <class Acc> __device__ static bool quiet(const Acc&) { return false; } };
template <class Op> struct act_of : act_never_quiet { static constexpr int role = kActNone; };
template <bool kD> struct act_of<OpDfsphError<kD>> {
    static constexpr int role = kActError;
    __device__ static bool quiet(const typename OpDfsphError<kD>::Acc& a) { return a.quiet; }
};
template <bool kCG> struct act_of<OpDensityAlphaDivError<kCG>> {
    static constexpr int role = kActError;
    __device__ static bool quiet(const typename OpDensityAlphaDivError<kCG>::Acc& a) { return a.b.quiet; }
};
template <> struct act_of<OpScalarGradient<0>> : act_never_quiet { static constexpr int role = kActCorrect; };
template <> struct act_of<OpScalarGradient<1>> : act_never_quiet { static constexpr int role = kActCorrect; };

// viscosity + surface tension / air pressure in one sweep (BasicSPHSolver.cu:183-225 then :332-381): the
// viscosity term reads the neighbours' velocity BEFORE either update (as both reference kernels do), the surface
// term does not read velocities at all, so  v_new = (v + deltaV) + a_surf*dt  is the reference's sequence.
struct OpViscositySurface {
    float4* velNew; float* vel; float* deltaV; float rho0, visc, dt, kappa, airP;
    static constexpr bool kFluidOnly = true, kHi = true;
    struct Acc {
        float3 av, as, vi; float cii, ratio;
        template <class F> __device__ void sums(F f) { f(av.x); f(av.y); f(av.z); f(as.x); f(as.y); f(as.z); }
    };
    __device__ void begin(Acc& a, int, float4 lo, float4 hi, const DevScene&) const {
        a.av = f3(0, 0, 0); a.as = f3(0, 0, 0); a.vi = xyz(hi);
        a.cii = lo.w;
        const float lci = sqrtf(lo.w);
        a.ratio = lci / fmaxf(SPHK_EPS, lci);
    }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        const float r = sqrtf(r2);
        a.av += mj * ((xyz(hi) - a.vi) / rho0) * lap_visc(r, s.k);
        const float mr = mj / (rho0 * rho0);
        a.as += 0.25f * mr * kappa * (a.cii + lo.w) * (d * grad_st_factor(r, s.k));
        a.as += airP * mr * (d * grad_w_factor(r, s.k)) * a.ratio;
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const {
        const float3 dv = visc * a.av * dt;
        store3(deltaV, i, dv);
        float3 v = a.vi + dv;
        v = f3(v.x + a.as.x * dt, v.y + a.as.y * dt, v.z + a.as.z * dt);
        velNew[i] = make_float4(v.x, v.y, v.z, 0.f); store3(vel, i, v);
    }
};

// ---- vorticity confinement (no reference counterpart; Macklin & Mueller 2013, section 5) ----------------------------------
__device__ __forceinline__ float3 cross3(float3 a, float3 b) {
    return f3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// omega_i = sum_j V_j (v_i - v_j) x gradW_ij, V_j = m_j / rho0, fluid neighbours only (a boundary has no velocity field to
// curl).  Rigid rotation v = W x x gives +2 W in the bulk.  |omega_i| goes to omegaNorm only, never to rec.s: a fused sweep
// gathers the neighbours' rec.s = |c|^2 while this runs.  r^2, r and the arithmetic after the kernel gradient are written with
// rounded intrinsics: nvcc contracts a * b - c * d into an FMA either way round depending on the kernel it is inlined into,
// and the fused sweeps must form omega bit for bit as this sweep does.
struct OpVorticity {
    float* omega; float* omegaNorm; float invRho0;
    static constexpr bool kFluidOnly = true, kHi = true;
    struct Acc { float3 w; float3 vi; template <class F> __device__ void sums(F f) { f(w.x); f(w.y); f(w.z); } };
    __device__ void begin(Acc& a, int, float4, float4 hi, const DevScene&) const { a.w = f3(0, 0, 0); a.vi = xyz(hi); }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float, float mj, float4, float4 hi, const DevScene& s) const {
        // (r^2 formed here: the drivers' dot product is contracted differently in different instantiations)
        const float r2 = __fmaf_rn(d.z, d.z, __fmaf_rn(d.y, d.y, __fmul_rn(d.x, d.x)));
        const float gw = grad_w_factor(__fsqrt_rn(r2), s.k);
        const float3 g = f3(__fmul_rn(d.x, gw), __fmul_rn(d.y, gw), __fmul_rn(d.z, gw));
        const float3 u = f3(__fsub_rn(a.vi.x, hi.x), __fsub_rn(a.vi.y, hi.y), __fsub_rn(a.vi.z, hi.z));
        const float V = __fmul_rn(mj, invRho0);
        a.w.x = __fmaf_rn(V, __fsub_rn(__fmul_rn(u.y, g.z), __fmul_rn(u.z, g.y)), a.w.x);
        a.w.y = __fmaf_rn(V, __fsub_rn(__fmul_rn(u.z, g.x), __fmul_rn(u.x, g.z)), a.w.y);
        a.w.z = __fmaf_rn(V, __fsub_rn(__fmul_rn(u.x, g.y), __fmul_rn(u.y, g.x)), a.w.z);
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const {
        store3(omega, i, a.w);
        omegaNorm[i] = __fsqrt_rn(__fmaf_rn(a.w.z, a.w.z, __fmaf_rn(a.w.y, a.w.y, __fmul_rn(a.w.x, a.w.x))));
    }
};

// eta_i = sum_j V_j (|omega_j| - |omega_i|) gradW_ij (difference form: a uniform |omega| gives exactly 0), N = eta / max(|eta|,
// eps), v_i += dt eps (N x omega_i).  rec.s = |omega| (mirrored by the entry).  Reads no neighbour velocity: in place.
struct OpVorticityConfinement {
    Rec rec; float* vel; const float* omega; float invRho0, dtEps;
    static constexpr bool kFluidOnly = true, kHi = false;
    struct Acc { float3 eta; float wi; template <class F> __device__ void sums(F f) { f(eta.x); f(eta.y); f(eta.z); } };
    __device__ void begin(Acc& a, int, float4 lo, float4, const DevScene&) const { a.eta = f3(0, 0, 0); a.wi = lo.w; }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float r2, float mj, float4 lo, float4, const DevScene& s) const {
        a.eta += (mj * invRho0 * (lo.w - a.wi)) * (d * grad_w_factor(sqrtf(r2), s.k));
    }
    __device__ void end(Acc& a, int i, float4, float4 hi, const DevScene&) const {
        const float3 n = a.eta / fmaxf(sqrtf(dot3(a.eta, a.eta)), SPHK_EPS);
        const float3 dv = dtEps * cross3(n, load3(omega, i));
        const float3 v = f3(hi.x + dv.x, hi.y + dv.y, hi.z + dv.z);
        rec_set_vel(rec + i, v); store3(vel, i, v);
    }
};

// ---- implicit viscosity (no reference counterpart; Weiler, Koschier, Brand & Bender 2018; DESIGN.md section 2.5) -------------
// Pair coefficient c_ij = -10 nu V_j g(r) / (r^2 + 0.01 R^2), g = grad_w_factor <= 0 (so c_ij >= 0), V_j = m_j / rho0; a boundary
// pair takes nu_b and m_b / rho_B.  `nuV` = nu V_j.  m_i c_ij = m_j c_ji: the system is self-adjoint in the mass inner product.
__device__ __forceinline__ float visc_coef(float nuV, float r2, const KConst& k) {
    return -10.0f * nuV * grad_w_factor(sqrtf(r2), k) / (r2 + 0.01f * k.R * k.R);
}
// symmetric 3x3 matrices as 6 floats {xx, yy, zz, xy, xz, yz}
__device__ __forceinline__ float3 sym_apply(const float* __restrict__ S, int i, float3 p) {
    const float* a = S + 6 * static_cast<size_t>(i);
    return f3(a[0] * p.x + a[3] * p.y + a[4] * p.z, a[3] * p.x + a[1] * p.y + a[5] * p.z, a[4] * p.x + a[5] * p.y + a[2] * p.z);
}

// D_i = I + dt sum_j c_ij d d^T (fluid and boundary neighbours), b_i = v*_i + dt sum_b c_ib d (d . v_b) (v_b = the boundary
// record's velocity: 0, or a kinematic body's v_k); Dinv (when non-null) = D_i^-1 by cofactors (D_i is symmetric, eigenvalues >= 1)
struct OpViscImplicitSetup {
    float* D; float* Dinv; float* b; float nuRho, nuBRho, dt;     // nu / rho0, nu_b / rho_B
    static constexpr bool kFluidOnly = false, kHi = true;
    struct Acc {
        float s[6]; float3 bb; float3 vi;
        template <class F> __device__ void sums(F f) { for (int k = 0; k < 6; ++k) f(s[k]); f(bb.x); f(bb.y); f(bb.z); }
    };
    __device__ void begin(Acc& a, int, float4, float4 hi, const DevScene&) const {
        for (int k = 0; k < 6; ++k) a.s[k] = 0.f;
        a.bb = f3(0, 0, 0); a.vi = xyz(hi);
    }
    __device__ void pair(Acc& a, int, int, bool isB, float3 d, float r2, float mj, float4, float4 hi, const DevScene& s) const {
        const float c = visc_coef(mj * (isB ? nuBRho : nuRho), r2, s.k);
        const float3 cd = c * d;
        a.s[0] += cd.x * d.x; a.s[1] += cd.y * d.y; a.s[2] += cd.z * d.z;
        a.s[3] += cd.x * d.y; a.s[4] += cd.x * d.z; a.s[5] += cd.y * d.z;
        if (isB) a.bb += dot3(d, xyz(hi)) * cd;
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const {
        float m[6];
        for (int k = 0; k < 6; ++k) m[k] = dt * a.s[k];
        m[0] += 1.0f; m[1] += 1.0f; m[2] += 1.0f;
        float* out = D + 6 * static_cast<size_t>(i);
        for (int k = 0; k < 6; ++k) out[k] = m[k];
        store3(b, i, a.vi + dt * a.bb);
        if (!Dinv) return;
        const float c00 = m[1] * m[2] - m[5] * m[5], c11 = m[0] * m[2] - m[4] * m[4], c22 = m[0] * m[1] - m[3] * m[3];
        const float c01 = m[4] * m[5] - m[3] * m[2], c02 = m[3] * m[5] - m[1] * m[4], c12 = m[3] * m[4] - m[0] * m[5];
        const float inv = 1.0f / (m[0] * c00 + m[3] * c01 + m[4] * c02);
        float* o = Dinv + 6 * static_cast<size_t>(i);
        o[0] = c00 * inv; o[1] = c11 * inv; o[2] = c22 * inv; o[3] = c01 * inv; o[4] = c02 * inv; o[5] = c12 * inv;
    }
};

// (A p)_i = D_i p_i - dt sum_j c_ij d (d . p_j), fluid neighbours only; p = the velocity slots of the fluid records (B.xyz; the
// solve keeps its CG direction there, so every path -- tile staging of B included -- gathers p with the record and B.w stays m)
struct OpViscImplicitMatvec {
    const float* D; float* Ap; float nuRho, dt;
    static constexpr bool kFluidOnly = true, kHi = true;
    struct Acc { float3 a; template <class F> __device__ void sums(F f) { f(a.x); f(a.y); f(a.z); } };
    __device__ void begin(Acc& a, int, float4, float4, const DevScene&) const { a.a = f3(0, 0, 0); }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float r2, float mj, float4, float4 hi, const DevScene& s) const {
        a.a += (visc_coef(mj * nuRho, r2, s.k) * dot3(d, xyz(hi))) * d;
    }
    __device__ void end(Acc& a, int i, float4, float4 hi, const DevScene&) const {
        store3(Ap, i, sym_apply(D, i, xyz(hi)) - dt * a.a);
    }
};

// ---- non-Newtonian viscosity (no reference counterpart; DESIGN.md section 2.9) ----------------------------------------------
// float <-> double without flushing subnormals (-use_fast_math makes the plain conversions flush them to zero)
__device__ __forceinline__ double f2d(float x) { double d; asm("cvt.f64.f32 %0, %1;" : "=d"(d) : "f"(x)); return d; }
__device__ __forceinline__ float d2f_rn(double x) { float f; asm("cvt.rn.f32.f64 %0, %1;" : "=f"(f) : "d"(x)); return f; }

// The viscosity model nu(gamma_dot) in double, clamped to [nu_min, nu_max] (a NaN shear rate lands on nu_max); *atMax: the
// clamp at nu_max bound (the unyielded part of a yield-stress fluid).
__device__ __forceinline__ double rheo_nu(const sphk_rheology& r, double g, bool* atMax) {
    double raw;
    if (r.model == SPHK_RHEOLOGY_CROSS) {
        const double nu0 = r.params[0], nuInf = r.params[1], lam = r.params[2], m = r.params[3];
        raw = nuInf + (nu0 - nuInf) / (1.0 + pow(lam * g, m));
    } else {                                   // Herschel-Bulkley, Papanastasiou-regularised
        const double K = r.params[0], n = r.params[1], tau = r.params[2], mr = r.params[3];
        const double power = K > 0.0 ? K * pow(g, n - 1.0) : 0.0;
        const double yield = g > 0.0 ? tau * (-expm1(-mr * g) / g) : tau * mr;
        raw = power + yield;
    }
    const double hi = r.nu_max, lo = r.nu_min;
    *atMax = !(raw < hi);
    return *atMax ? hi : fmax(raw, lo);
}

// Statistics of one shear sweep in the context's memory, as uint bits of non-negative floats (so atomicMax / atomicMin order them):
// {.., .., max gamma_dot, min nu, max nu, particles at the nu_max clamp}; slots 0 and 1 take the solve's iterations and residual.
#define SPHK_RHEO_STATS 6
__device__ __forceinline__ void rheo_fold_stats(unsigned int* st, float gd, float nu, bool atMax) {
    namespace cg = cooperative_groups;
    const cg::coalesced_group g = cg::coalesced_threads();
    const unsigned int gmax = cg::reduce(g, __float_as_uint(gd), cg::greater<unsigned int>());
    const unsigned int nmin = cg::reduce(g, __float_as_uint(nu), cg::less<unsigned int>());
    const unsigned int nmax = cg::reduce(g, __float_as_uint(nu), cg::greater<unsigned int>());
    const unsigned int cnt = __popc(g.ballot(atMax));
    if (g.thread_rank() == 0) {
        atomicMax(st + 2, gmax); atomicMin(st + 3, nmin); atomicMax(st + 4, nmax);
        if (cnt) atomicAdd(st + 5, cnt);
    }
}

// Shear rate (Monaghan-style corrected gradient): with u = v_j - v_i, gradW = g d, V_j = m_j / rho0 (a boundary neighbour:
// m_b / rho_B and the record's velocity, counted only when beta > 0)
//   G_i = sum_j V_j u (x) gradW        M_i = -sum_j V_j g d d^T  (symmetric, {xx, yy, zz, xy, xz, yz})
//   grad v_i = G_i M_i^-1, or G_i 3 / tr M_i where det M_i < theta (tr M_i / 3)^3 (few neighbours or one-sided support)
//   gamma_dot_i = sqrt(2 E:E),  E = (grad v + grad v^T) / 2
// A linear field v = A x + b gives G = A M, so the corrected gradient is A exactly.  The epilogue works in double, evaluates the
// model, writes gamma_dot and nu_i (+ the 9-float gradient, row-major d v_a / d x_b, and the fallback flag for tests) and folds the
// statistics.
#define SPHK_RHEO_THETA 0.01
struct OpShearRate {
    float* gamma; float* nu; float* grad; int* flag; unsigned int* stats; sphk_rheology rh; float invRho0, invRhoB; bool wall;
    static constexpr bool kFluidOnly = false, kHi = true;
    struct Acc {
        float G[9]; float M[6]; float3 vi;
        template <class F> __device__ void sums(F f) { for (int k = 0; k < 9; ++k) f(G[k]); for (int k = 0; k < 6; ++k) f(M[k]); }
    };
    __device__ void begin(Acc& a, int, float4, float4 hi, const DevScene&) const {
        for (int k = 0; k < 9; ++k) a.G[k] = 0.f;
        for (int k = 0; k < 6; ++k) a.M[k] = 0.f;
        a.vi = xyz(hi);
    }
    __device__ void pair(Acc& a, int, int, bool isB, float3 d, float r2, float mj, float4, float4 hi, const DevScene& s) const {
        if (isB && !wall) return;
        const float Vg = mj * (isB ? invRhoB : invRho0) * grad_w_factor(sqrtf(r2), s.k);
        const float3 u = xyz(hi) - a.vi, w = Vg * d;          // V_j gradW
        a.G[0] += u.x * w.x; a.G[1] += u.x * w.y; a.G[2] += u.x * w.z;
        a.G[3] += u.y * w.x; a.G[4] += u.y * w.y; a.G[5] += u.y * w.z;
        a.G[6] += u.z * w.x; a.G[7] += u.z * w.y; a.G[8] += u.z * w.z;
        a.M[0] -= w.x * d.x; a.M[1] -= w.y * d.y; a.M[2] -= w.z * d.z;
        a.M[3] -= w.x * d.y; a.M[4] -= w.x * d.z; a.M[5] -= w.y * d.z;
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const {
        const double m0 = f2d(a.M[0]), m1 = f2d(a.M[1]), m2 = f2d(a.M[2]), m3 = f2d(a.M[3]), m4 = f2d(a.M[4]), m5 = f2d(a.M[5]);
        const double tr = m0 + m1 + m2;
        const double c00 = m1 * m2 - m5 * m5, c11 = m0 * m2 - m4 * m4, c22 = m0 * m1 - m3 * m3;
        const double c01 = m4 * m5 - m3 * m2, c02 = m3 * m5 - m1 * m4, c12 = m3 * m4 - m0 * m5;
        const double det = m0 * c00 + m3 * c01 + m4 * c02;
        const double t3 = tr / 3.0;
        const bool corrected = tr > 0.0 && det >= SPHK_RHEO_THETA * t3 * t3 * t3;
        double inv[9];
        if (corrected) {
            const double q = 1.0 / det;
            inv[0] = c00 * q; inv[1] = c01 * q; inv[2] = c02 * q;
            inv[3] = c01 * q; inv[4] = c11 * q; inv[5] = c12 * q;
            inv[6] = c02 * q; inv[7] = c12 * q; inv[8] = c22 * q;
        } else {
            const double q = tr > 0.0 ? 1.0 / t3 : 0.0;
            for (int k = 0; k < 9; ++k) inv[k] = (k % 4 == 0) ? q : 0.0;
        }
        double L[9];
        for (int r = 0; r < 3; ++r)
            for (int col = 0; col < 3; ++col)
                L[3 * r + col] = f2d(a.G[3 * r]) * inv[col] + f2d(a.G[3 * r + 1]) * inv[3 + col] + f2d(a.G[3 * r + 2]) * inv[6 + col];
        double ee = 0.0;
        for (int r = 0; r < 3; ++r)
            for (int col = 0; col < 3; ++col) {
                const double e = 0.5 * (L[3 * r + col] + L[3 * col + r]);
                ee += e * e;
            }
        const double gd = sqrt(2.0 * ee);
        bool atMax;
        const float gf = d2f_rn(gd), nf = d2f_rn(rheo_nu(rh, gd, &atMax));
        gamma[i] = gf;
        nu[i] = nf;
        if (grad) for (int k = 0; k < 9; ++k) grad[9 * static_cast<size_t>(i) + k] = d2f_rn(L[k]);
        if (flag) flag[i] = corrected ? 0 : 1;
        rheo_fold_stats(stats, gf, nf, atMax);
    }
};

// The implicit viscosity sweeps with a per-particle viscosity: rec.s = nu_i / rho0 (mirrored by the entry, k_rheo_mirror), a
// fluid pair takes the mean nu_ij V_j = (s_i + s_j) / 2 m_j (so m_i c_ij = m_j c_ji: A stays self-adjoint in the mass inner
// product), a boundary pair beta nu_i m_b / rho_B.  With nu_i = nu everywhere and beta = 1 every coefficient is the one the
// constant-nu sweeps form (the same float operations on the same values).
struct OpViscImplicitSetupField {
    OpViscImplicitSetup base; const float* nuField; float beta, rhoB;
    static constexpr bool kFluidOnly = false, kHi = true;
    struct Acc : OpViscImplicitSetup::Acc { float si, sb; };
    __device__ void begin(Acc& a, int i, float4 lo, float4 hi, const DevScene& s) const {
        base.begin(a, i, lo, hi, s);
        a.si = lo.w;
        a.sb = __fdiv_rn(beta * nuField[i], rhoB);
    }
    __device__ void pair(Acc& a, int, int, bool isB, float3 d, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        const float c = visc_coef(mj * (isB ? a.sb : 0.5f * (a.si + lo.w)), r2, s.k);
        const float3 cd = c * d;
        a.s[0] += cd.x * d.x; a.s[1] += cd.y * d.y; a.s[2] += cd.z * d.z;
        a.s[3] += cd.x * d.y; a.s[4] += cd.x * d.z; a.s[5] += cd.y * d.z;
        if (isB) a.bb += dot3(d, xyz(hi)) * cd;
    }
    __device__ void end(Acc& a, int i, float4 lo, float4 hi, const DevScene& s) const { base.end(a, i, lo, hi, s); }
};

struct OpViscImplicitMatvecField {
    const float* D; float* Ap; float dt;
    static constexpr bool kFluidOnly = true, kHi = true;
    struct Acc : OpViscImplicitMatvec::Acc { float si; };
    __device__ void begin(Acc& a, int, float4 lo, float4, const DevScene&) const { a.a = f3(0, 0, 0); a.si = lo.w; }
    __device__ void pair(Acc& a, int, int, bool, float3 d, float r2, float mj, float4 lo, float4 hi, const DevScene& s) const {
        a.a += (visc_coef(mj * (0.5f * (a.si + lo.w)), r2, s.k) * dot3(d, xyz(hi))) * d;
    }
    __device__ void end(Acc& a, int i, float4, float4 hi, const DevScene&) const {
        store3(Ap, i, sym_apply(D, i, xyz(hi)) - dt * a.a);
    }
};

// ---- heat transfer (no reference counterpart; DESIGN.md section 2.10) -------------------------------------------------------
// Brookshaw / Cleary-Monaghan conduction, rec.s = T (ensure_scalar): c_ij = -2 alpha V_j f r^2 / (r^2 + eta^2), eta^2 = 0.0025 R^2,
// V_j = m_j / rho0; a boundary neighbour of group g takes V_b = m_b / rho_B, h_g alpha and T_g.  Without bodies every boundary
// particle is in group 0, whose {T, h} the operator carries (no extra load); with bodies the group is local[b].w and {T_g, h_g}
// come from the context's table.  The epilogue writes dT/dt and folds max dt_k sum_j c_ij and the count above 1.
__device__ __forceinline__ float heat_coef(float aV, float r2, const KConst& k) {
    return -2.0f * aV * grad_w_factor(sqrtf(r2), k) * __fdividef(r2, r2 + 0.0025f * k.R * k.R);
}
struct OpHeatConduction {
    float* dTdt; unsigned int* stats; const float4* local; const float2* groups;
    float alphaRho0, alphaRhoB, t0, h0, dtSub; int nB;
    static constexpr bool kFluidOnly = false, kHi = false, kIndex = true;
    struct Acc { float q, c, ti; template <class F> __device__ void sums(F f) { f(q); f(c); } };
    __device__ void begin(Acc& a, int, float4 lo, float4, const DevScene&) const { a.q = 0.f; a.c = 0.f; a.ti = lo.w; }
    __device__ void pair(Acc& a, int, int j, bool isB, float3, float r2, float mj, float4 lo, float4, const DevScene& s) const {
        float tj = lo.w, h = 1.0f;
        if (isB) {
            tj = t0; h = h0;
            if (local) {
                const int b = j - s.bOff;
                if (b >= 0 && b < nB) {
                    const float2 g = groups[static_cast<int>(body_group(local[b]))];
                    tj = g.x; h = g.y;
                }
            }
        }
        const float c = heat_coef(mj * (isB ? h * alphaRhoB : alphaRho0), r2, s.k);
        a.q += c * (tj - a.ti);
        a.c += c;
    }
    __device__ void end(Acc& a, int i, float4, float4, const DevScene&) const {
        dTdt[i] = a.q;
        namespace cg = cooperative_groups;
        const float cour = dtSub * a.c > 0.f ? dtSub * a.c : 0.f;      // (no -0: its bits would top the unsigned max)
        const cg::coalesced_group g = cg::coalesced_threads();
        const unsigned int cmax = cg::reduce(g, __float_as_uint(cour), cg::greater<unsigned int>());
        const unsigned int cnt = __popc(g.ballot(cour > 1.0f));
        if (g.thread_rank() == 0) {
            atomicMax(stats, cmax);
            if (cnt) atomicAdd(stats + 1, cnt);
        }
    }
};

// =================================================================================================
// Sweep drivers
// =================================================================================================
template <class Op>
__device__ __forceinline__ void fetch(const DevScene& s, int j, float4& lo, float4& hi) {
    lo = rec_lo(s.rec + j);
    if (Op::kHi) hi = rec_hi(s.rec + j);
    else hi = make_float4(0.f, 0.f, 0.f, 0.f);
}
// One candidate pair (i, j) with j's gathered halves.  Mass of the neighbour: the B half when it was gathered; else
// the A half's fourth slot for a boundary neighbour (boundary records keep their mass there, their scalar is 0), the
// uniform fluid mass for a fluid neighbour (one extra load when the fluid masses differ).
// kUniform: the caller has established that all fluid masses equal m0 (the list walk branches on that ONCE per particle, so
// the per-pair code of the common case carries no trace of the extra load).
template <class Op, bool kUniform = false>
__device__ __forceinline__ void feed_pair(const DevScene& s, const Op& op, typename Op::Acc& acc, int i, float3 xi, int j, bool isB,
                                          float4 lo, float4 hi, float m0, float3 d, float r2) {
    float mj;
    if (Op::kHi) mj = hi.w;
    else if (kUniform) mj = isB ? lo.w : m0;
    else mj = isB ? lo.w : (m0 < 0.f ? rec_m(s.rec + j) : m0);
    lo.w = isB ? 0.0f : lo.w;
    op.pair(acc, i, j, isB, d, r2, mj, lo, hi, s);
}
// uniform fluid mass of the last search, or -1 when the masses differ
__device__ __forceinline__ float uniform_mass(const DevScene& s) {
    const float lo = s.massRange[0], hi = s.massRange[1];
    return (lo == hi) ? lo : -1.0f;
}

// The 27-cell walk, row-merged: the three z-neighbours (x+dx, y+dy, z-1..z+1) are consecutive cell indices,
// hence ONE contiguous particle range per (dx,dy) row (CUDAFunctions.cuh:68: z is the fastest dimension).
// Rows are visited in the reference's order (dx outermost); inside a row the fluid range comes first, then
// the boundary range (the reference interleaves fluid/boundary per cell: the difference is the order of a few
// boundary terms in the sum, ~1e-7 relative).  The centre cell is recomputed from the LIVE position while the
// ranges stay those of the last search -- the reference's PBD semantics (Q7).
template <class Op>
__device__ __forceinline__ void walk_cells(const DevScene& s, const Op& op, typename Op::Acc& acc, int i, float4 pi, float m0) {
    const int cx = cell_coord(pi.x, s.cellLength) - s.org.x, cy = cell_coord(pi.y, s.cellLength) - s.org.y,
              cz = cell_coord(pi.z, s.cellLength) - s.org.z;
    const float3 xi = xyz(pi);
    if (cz < -1 || cz > s.cs.z) return;
    const int zlo = max(cz - 1, 0), zhi = min(cz + 1, s.cs.z - 1);
    if (zlo > zhi) return;
#pragma unroll 1
    for (int r = 0; r < 9; ++r) {
        const int x = cx + r / 3 - 1, y = cy + r % 3 - 1;
        if (x < 0 || x >= s.cs.x || y < 0 || y >= s.cs.y) continue;
        const int c0 = (x * s.cs.y + y) * s.cs.z;
        {
            const int end = s.csF[c0 + zhi + 1];
            for (int j = s.csF[c0 + zlo]; j < end; ++j) {
                float4 lo, hi;
                fetch<Op>(s, j, lo, hi);
                const float3 d = xi - xyz(lo);
                const float r2 = dot3(d, d);
                if (r2 <= s.r2list) feed_pair(s, op, acc, i, xi, j, false, lo, hi, m0, d, r2);
            }
        }
        if (!Op::kFluidOnly) {
            const int end = s.csB[c0 + zhi + 1];
            for (int jb = s.csB[c0 + zlo]; jb < end; ++jb) {
                const int j = s.bOff + jb;
                float4 lo, hi;
                fetch<Op>(s, j, lo, hi);
                const float3 d = xi - xyz(lo);
                const float r2 = dot3(d, d);
                if (r2 <= s.r2list) feed_pair(s, op, acc, i, xi, j, true, lo, hi, m0, d, r2);
            }
        }
    }
}

template <class Op>
__global__ void __launch_bounds__(SPHK_BLOCK) k_sweep_cells(const DevScene s, const Op op) {
    if (s.pred && *s.pred == 0) return;
    const int i = s.iBegin + blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (!in_range(s, i)) return;
    float4 lo, hi;
    rec_full(s.rec + i, lo, hi);
    typename Op::Acc acc;
    op.begin(acc, i, lo, hi, s);
    walk_cells(s, op, acc, i, lo, uniform_mass(s));
    op.end(acc, i, lo, hi, s);
}

template <class Op, bool kUniform = false>
__device__ __forceinline__ void list_pair(const DevScene& s, const Op& op, typename Op::Acc& acc, int i, float3 xi, int j,
                                          float4 lo, float4 hi, float m0) {
    const bool isB = j >= s.bOff;
    if (Op::kFluidOnly && isB) return;
    const float3 d = xi - xyz(lo);
    feed_pair<Op, kUniform>(s, op, acc, i, xi, j, isB, lo, hi, m0, d, dot3(d, d));
}

template <class Op, bool kUniform>
__device__ __forceinline__ void walk_list(const DevScene& s, const Op& op, typename Op::Acc& acc, int i, float3 xi, int n, float m0) {
    const int nb4 = (n + 3) >> 2;
    const int4* __restrict__ row = reinterpret_cast<const int4*>(s.nbr) + i;
    int4 jn = make_int4(i, i, i, i);
    if (nb4 > 0) jn = __ldcs(row);
    for (int b = 0; b < nb4; ++b) {
        const int4 j4 = jn;
        row += s.nbrStride;
        if (b + 1 < nb4) jn = __ldcs(row);
        float4 l0, h0, l1, h1, l2, h2, l3, h3;
        fetch<Op>(s, j4.x, l0, h0); fetch<Op>(s, j4.y, l1, h1); fetch<Op>(s, j4.z, l2, h2); fetch<Op>(s, j4.w, l3, h3);
        list_pair<Op, kUniform>(s, op, acc, i, xi, j4.x, l0, h0, m0);
        list_pair<Op, kUniform>(s, op, acc, i, xi, j4.y, l1, h1, m0);
        list_pair<Op, kUniform>(s, op, acc, i, xi, j4.z, l2, h2, m0);
        list_pair<Op, kUniform>(s, op, acc, i, xi, j4.w, l3, h3, m0);
    }
}

// one particle's walk of its neighbour list (thread per particle); returns whether an error sweep left the particle quiet
template <class Op>
__device__ __forceinline__ bool sweep_list_particle(const DevScene& s, const Op& op, int i) {
    float4 lo, hi;
    rec_full(s.rec + i, lo, hi);
    const float3 xi = xyz(lo);
    typename Op::Acc acc;
    op.begin(acc, i, lo, hi, s);
    int n = s.cnt[i];
    const float m0 = uniform_mass(s);
    if (s.cellFlag) {                                  // skin list: a fast mover is (or was) within reach of this cell -> exact walk
        const int c = cell_index(cell_coord(lo.x, s.cellLength) - s.org.x, cell_coord(lo.y, s.cellLength) - s.org.y,
                                 cell_coord(lo.z, s.cellLength) - s.org.z, s.cs);
        if (c >= s.cs.x * s.cs.y * s.cs.z || s.cellFlag[c]) n = s.kmax + 1;
    }
    if (n <= s.kmax) {
        // (the warp-uniform branch keeps the common case -- equal fluid masses, SPHSystem.cu:73 -- free of the per-pair mass load)
        if (Op::kHi || m0 >= 0.f) walk_list<Op, true>(s, op, acc, i, xi, n, m0);
        else walk_list<Op, false>(s, op, acc, i, xi, n, m0);
    } else {
        walk_cells(s, op, acc, i, lo, m0);  // more neighbours than the list keeps: exact fallback
    }
    op.end(acc, i, lo, hi, s);
    return act_of<Op>::quiet(acc);
}

// ---- chunk activity: the DFSPH sweeps skip what they would recompute unchanged ----------------------------------------------
// A chunk is the 32 particles [32k, 32k + 32) of the sorted fluid set: warp k of a list sweep launched over all nF (iBegin = 0),
// with the default or the patch mapping alike.  chunkAct[k] is the ballot of the chunk's particles whose record scalar may be
// non-zero: a lane counts as quiet only when it is in the sweep's range and its error sweep left e = +0, kappa = -0
// (OpDfsphError::finish), or k_s_copy wrote exactly -0 -- ghosts of a slab rank and lanes past nF are always active.
// Reach: every list entry of a particle of tile T (and every cell of its exact cell-walk fallback) is a boundary record, whose
// scalar is 0, or lies in one of T's nine fluid windows (tile_window: the cells [cA + off - 1, cB + off + 1] around the tile's
// cells [cA, cB]).  The list builder keeps those windows in tileWin; a tile with a particle outside the grid is unbounded.
// The fluid windows of `tile`, one per lane 0..8, loaded together (one round trip instead of one per window): lane r holds the
// chunk words [a, b] that window r touches (b < a: empty; a count of -1 marks an unbounded tile, b = -2).
__device__ __forceinline__ int2 tile_reach(const DevScene& s, int tile) {
    const int lane = threadIdx.x & 31;
    int2 w = make_int2(0, 0);
    if (lane < 9) w = s.tileWin[static_cast<size_t>(tile) * SPHK_TILE_WINS + lane];
    if (w.y < 0) return make_int2(0, -2);
    return make_int2(w.x >> 5, w.y > 0 ? (w.x + w.y - 1) >> 5 : (w.x >> 5) - 1);
}
template <bool kStamp> __device__ __forceinline__ bool chunk_quiet(const DevScene& s, int k) {
    return kStamp ? s.stamp[k] <= s.seq : s.act[k] == 0u;
}
// true when every chunk the fluid windows touch has chunkAct == 0 (kStamp false) / a stamp <= s.seq (kStamp true).  Lane l
// checks chunk a + l of every window, so the nine chunk-word loads of the common case (no window spans more than 32 chunks)
// are independent and issued together; longer windows finish in a loop.
template <bool kStamp>
__device__ __forceinline__ bool reach_quiet(const DevScene& s, int2 t) {
    const unsigned int full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    if (__any_sync(full, t.y == -2)) return false;    // unbounded tile
    const bool more = __any_sync(full, t.y - t.x >= 32);
    bool ok = true;
#pragma unroll
    for (int r = 0; r < 9; ++r) {
        const int a = __shfl_sync(full, t.x, r), b = __shfl_sync(full, t.y, r);
        if (a + lane <= b) ok &= chunk_quiet<kStamp>(s, a + lane);
    }
    if (more) {
#pragma unroll 1
        for (int r = 0; r < 9; ++r) {
            const int a = __shfl_sync(full, t.x, r), b = __shfl_sync(full, t.y, r);
            for (int k = a + 32 + lane; k <= b; k += 32) ok &= chunk_quiet<kStamp>(s, k);
        }
    }
    return __all_sync(full, ok);
}

// ---- velocity epochs: a quiet chunk's epilogue runs once per stretch of correct sweeps ----------------------------------------
// The quiet epilogue adds +0 to every velocity (OpScalarGradient::quiet_adds_zero): after one pass through it a chunk's vel and
// rec.b hold a fixed point, and every later pass is a no-op -- until anything else writes velocities.  The host counts in
// velCredited the launches known to write neither vel nor rec.b (error sweeps, the scalar copy, loop control, reductions) and
// the correct sweeps that keep the marks; an epoch is a run of marked correct sweeps over one vel array with only those in
// between (vel_mark() unchanged).  Every marked sweep writes the mark of every chunk of its grid: a warp that walks clears it,
// a quiet warp sets it after its pass -- also when the loop predicate skips the sweep (cleared, nothing is known of what came
// before).  The first sweep of an epoch (trust 0) ignores the marks it finds and takes every quiet chunk through end_quiet;
// later ones skip a quiet chunk whose mark is set.  So a mark is only trusted after the same epoch has written it: marks left
// by an earlier epoch -- or by an earlier replay of a captured step, which repeats the same trust flags -- are never read.

// one warp = one chunk of a DFSPH error or correct sweep that keeps chunk activity
template <class Op>
__device__ __forceinline__ void sweep_list_warp(const DevScene& s, const Op& op, int i) {
    const int lane = threadIdx.x & 31, chunk = i >> 5;
    if (i - lane >= s.nF) return;                     // a whole warp past the set (patch mapping rounds the grid up)
    const bool in = in_range(s, i);
    if constexpr (act_of<Op>::role == kActError) {
        // Reuse (s.reuse: the host's token -- the previous error sweep was of this kind with the same arrays, dt and rho0, and
        // since then no launch changed positions, densities, alpha, rec.s or these outputs, only correct sweeps moved velocities).
        // The outputs of this chunk's particles depend on their own velocity and those of their reach, nothing else that moved:
        // when no chunk of the reach was stamped since that sweep, they are what it wrote.  Own kappa quiet is required as well:
        // the density error's warm accumulate (warm += kappa) must be a no-op for a skip to be exact -- a particle with
        // kappa != 0 whose velocities did not change still accumulates.
        if (s.reuse) {
            const int2 t = tile_reach(s, i / SPHK_BLOCK);    // (issued with the chunk word: one round trip for both)
            if (s.act[chunk] == 0u && reach_quiet<true>(s, t)) return;
        }
        bool quiet = false;
        if (in) quiet = sweep_list_particle(s, op, i);
        const unsigned int act = __ballot_sync(0xffffffffu, !quiet);
        if ((threadIdx.x & 31) == 0) s.act[i >> 5] = act;
    } else {
        // Every kappa in reach is -0 (boundary records: +0 after feed_pair), so every pair term is mj * (+-0) * (d * f) with a
        // finite d * f (listed pairs have r^2 <= r2list at unchanged positions): +-0, and the accumulator, starting at +0, stays
        // +0.  The walk is skipped; the epilogue runs on the +0 sum (end_quiet), so vel and rec.b hold exactly what the walk
        // would write (v + 0: -0 components become +0), or -- a marked chunk of a trusted sweep -- already hold it.  Neither
        // is stamped: an error sweep cannot tell a +0 velocity component from a -0 one (its sum starts at +0 and only ever adds
        // terms; a zero term of either sign leaves it unchanged).
        if (s.act) {
            const int2 t = tile_reach(s, i / SPHK_BLOCK);
            const bool marked = s.mark && s.trust && s.mark[chunk] != 0;
            if (s.act[chunk] == 0u && reach_quiet<false>(s, t)) {
                if (marked) return;
                if (in) op.end_quiet(i);
                if (lane == 0 && s.mark) s.mark[chunk] = 1;
                return;
            }
        }
        if (lane == 0) {                               // (before the walk: nothing of this stays live across it)
            s.stamp[chunk] = s.seq;
            if (s.mark) s.mark[chunk] = 0;
        }
        if (in) sweep_list_particle(s, op, i);
    }
}

// the particle (default mapping) or the chunk (patch mapping) of thread t of a list sweep
__device__ __forceinline__ int list_thread(const DevScene& s) {
    int t = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (s.patch > 0) {               // groups of 4 runs of `patch` chunks; block bb of a group: chunk bb of each run, one per warp
        static_assert(SPHK_BLOCK == 128, "four warps per block");
        const int chunk = t >> 5, per = 4 * s.patch, g = chunk / per, r = chunk - g * per;
        t = ((g * per + (r & 3) * s.patch + (r >> 2)) << 5) | (t & 31);
    }
    return s.iBegin + t;
}

template <class Op>
__global__ void __launch_bounds__(SPHK_BLOCK) k_sweep_list(const DevScene s, const Op op) {
    if (s.pred && *s.pred == 0) return;
    const int i = list_thread(s);
    if (!in_range(s, i)) return;
    sweep_list_particle(s, op, i);
}
// the DFSPH error and correct sweeps when they keep chunk activity (a kernel of its own: the plain walk keeps its registers)
template <class Op>
__global__ void __launch_bounds__(SPHK_BLOCK) k_sweep_list_act(const DevScene s, const Op op) {
    const int i = list_thread(s);
    if (s.pred && *s.pred == 0) {
        // a skipped correct sweep still writes its marks (velocity epochs): cleared
        if (act_of<Op>::role == kActCorrect && s.mark && (threadIdx.x & 31) == 0 && i < s.nF) s.mark[i >> 5] = 0;
        return;
    }
    sweep_list_warp(s, op, i);
}

// =================================================================================================
// Tile lists: neighbour windows staged in shared memory (TMA bulk copies), 16-bit tile-local lists
// =================================================================================================
// A tile = SPHK_BLOCK consecutive particles of the sorted fluid set = one thread block.  Let [cA, cB] be the range of
// cell indices its particles occupy.  z is the fastest cell dimension (CUDAFunctions.cuh:68), so for each of the nine
// (dx,dy) rows every neighbour cell of every particle of the tile lies in the ONE contiguous cell range
// [cA + off - 1, cB + off + 1], off = (dx*cs.y + dy)*cs.z, i.e. in one contiguous range of sorted records -- per set:
// 9 fluid + 9 boundary windows, ~1300 records for a tile at the lattice density.  The list builder computes the windows
// once per step (tileWin), every sweep copies them from the A (and, for velocity sweeps, B) record arrays into shared
// memory with cp.async.bulk (one elected thread, completion on an mbarrier) while the threads load their own records,
// and then walks per-particle lists of 16-bit slots of the staged arrays.  What this buys over gathering from global
// memory: no L1 misses on the ~31 gathers per particle (each window record is fetched once per
// tile as part of a full line instead of ~3.3 times as a lone 32-byte sector), and half the list traffic.
// A tile whose windows exceed SPHK_TILE_CAP records, and particles outside the grid, fall back to the exact cell walk
// (their count is stored as kmax + 1).
__device__ __forceinline__ void build_particle_global(const DevScene& s, int i, float4 lo, int* __restrict__ nbr, int* __restrict__ cnt,
                                                      float4* __restrict__ posBuild);
__device__ __forceinline__ unsigned int smem_u32(const void* p) { return static_cast<unsigned int>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned int bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned int bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned int parity) {
    unsigned int ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}

// thread 0: prefix sums of the window lengths; stages the windows when they fit.  Returns nothing; sPre[18] = total.
__device__ __forceinline__ void tile_stage(const DevScene& s, const int2* sWin, int* sPre, float4* smA, float4* smB, bool wantB,
                                           unsigned long long* bar, int cap = SPHK_TILE_CAP) {
    int t = 0;
    for (int w = 0; w < SPHK_TILE_WINS; ++w) { sPre[w] = t; t += sWin[w].y; }
    sPre[SPHK_TILE_WINS] = t;
    if (t > cap) return;
    smA[t] = make_float4(1.0e6f, 1.0e6f, 1.0e6f, 0.f);           // the dummy slot: list padding, contributes exactly 0
    if (wantB) smB[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t == 0) return;
    mbar_init(bar, 1);
    mbar_expect_tx(bar, static_cast<unsigned int>(t) * 16u * (wantB ? 2u : 1u));
    for (int w = 0; w < SPHK_TILE_WINS; ++w) {
        const int len = sWin[w].y;
        if (len <= 0) continue;
        bulk_g2s(smA + sPre[w], s.rec.a + sWin[w].x, static_cast<unsigned int>(len) * 16u, bar);
        if (wantB) bulk_g2s(smB + sPre[w], s.rec.b + sWin[w].x, static_cast<unsigned int>(len) * 16u, bar);
    }
}

// ---- builder -----------------------------------------------------------------------------------------------------------
// candidates [slot0, slot0 + count) of the staged A records against x; hits appended as 16-bit slots (two-phase, like
// build_range: branch-free tests -> bit mask -> walk the set bits)
__device__ __forceinline__ void build_range_tile(const float4* smA, int slot0, int count, float3 xi, float r2list, int selfSlot, int kmax,
                                                 int& n, unsigned short*& wp, long long jump) {
    for (int k0 = 0; k0 < count; k0 += 32) {
        const int len = min(32, count - k0);
        const float4* base = smA + slot0 + k0;
        unsigned int mask = 0u;
#pragma unroll 4
        for (int k = 0; k < len; ++k) {
            const float3 d = xi - xyz(base[k]);
            mask |= (dot3(d, d) <= r2list ? 1u : 0u) << k;
        }
        const int self = selfSlot - (slot0 + k0);
        if (self >= 0 && self < 32) mask &= ~(1u << self);
        while (mask) {
            const int k = __ffs(mask) - 1;
            mask &= mask - 1;
            if (n < kmax) *wp = static_cast<unsigned short>(slot0 + k0 + k);
            wp += ((n & 7) == 7) ? jump : 1;
            ++n;
        }
    }
}

// the 18 windows of the tile whose particles occupy cells [cA, cB] (thread w < 18 computes window w)
__device__ __forceinline__ int2 tile_window(const DevScene& s, int w, int cA, int cB, int ncells) {
    if (cB < 0) return make_int2(0, 0);
    const int r = w % 9;
    const bool isB = w >= 9;
    const long long off = (static_cast<long long>(r / 3 - 1) * s.cs.y + (r % 3 - 1)) * s.cs.z;
    long long cl = cA + off - 1, ch = cB + off + 1;
    if (cl < 0) cl = 0;
    if (ch > ncells - 1) ch = ncells - 1;
    if (cl > ch) return make_int2(0, 0);
    const int* cs = isB ? s.csB : s.csF;
    const int a = cs[cl], b = cs[ch + 1];
    return make_int2(a + (isB ? s.bOff : 0), b - a);
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_build_tile(const DevScene s, unsigned short* __restrict__ nbr16, int* __restrict__ cnt, float4* __restrict__ posBuild,
             int2* __restrict__ tileWin) {
    extern __shared__ float4 smA[];                 // [SPHK_TILE_CAP + 1]
    __shared__ unsigned long long bar;
    __shared__ int sMin, sMax;
    __shared__ int2 sWin[SPHK_TILE_WINS];
    __shared__ int sPre[SPHK_TILE_WINS + 1];
    const int tile = s.iBegin / SPHK_BLOCK + blockIdx.x;
    const int i = tile * SPHK_BLOCK + threadIdx.x;
    const bool have = i < s.nF;
    const int ncells = s.cs.x * s.cs.y * s.cs.z;
    if (threadIdx.x == 0) { sMin = 0x7fffffff; sMax = -1; }
    __syncthreads();
    float4 lo = make_float4(0.f, 0.f, 0.f, 0.f);
    int cx = 0, cy = 0, cz = 0, c = ncells;
    if (have) {
        lo = rec_lo(s.rec + i);
        cx = cell_coord(lo.x, s.cellLength) - s.org.x; cy = cell_coord(lo.y, s.cellLength) - s.org.y; cz = cell_coord(lo.z, s.cellLength) - s.org.z;
        c = cell_index(cx, cy, cz, s.cs);
        if (c < ncells) { atomicMin(&sMin, c); atomicMax(&sMax, c); }
    }
    __syncthreads();
    if (threadIdx.x < SPHK_TILE_WINS) {
        const int2 w = tile_window(s, threadIdx.x, sMin, sMax, ncells);
        sWin[threadIdx.x] = w;
        tileWin[static_cast<size_t>(tile) * SPHK_TILE_WINS + threadIdx.x] = w;
    }
    __syncthreads();
    if (threadIdx.x == 0) tile_stage(s, sWin, sPre, smA, nullptr, false, &bar);
    __syncthreads();
    const int T = sPre[SPHK_TILE_WINS];
    const bool staged = T <= SPHK_TILE_CAP;
    if (staged && T > 0) mbar_wait(&bar, 0);        // every thread: the block must not retire with bulk copies in flight
    if (!have || !in_range(s, i)) return;
    if (!staged || c >= ncells) { cnt[i] = s.kmax + 1; return; }      // this particle walks the cells (exact fallback)
    const float3 xi = xyz(lo);
    const int zlo = max(cz - 1, 0), zhi = min(cz + 1, s.cs.z - 1);
    const int selfSlot = sPre[4] + (i - sWin[4].x);
    int n = 0;
    unsigned short* wp = nbr16 + static_cast<size_t>(i) * 8;                  // entry 0 of particle i
    const long long jump = static_cast<long long>(s.nbrStride) * 8 - 7;        // from entry 7 of batch b to entry 0 of batch b+1
#pragma unroll 1
    for (int r = 0; r < 9; ++r) {
        const int x = cx + r / 3 - 1, y = cy + r % 3 - 1;
        if (x < 0 || x >= s.cs.x || y < 0 || y >= s.cs.y) continue;
        const int c0 = (x * s.cs.y + y) * s.cs.z;
        {
            const int a = s.csF[c0 + zlo], b = s.csF[c0 + zhi + 1];
            build_range_tile(smA, sPre[r] + (a - sWin[r].x), b - a, xi, s.r2list, selfSlot, s.kmax, n, wp, jump);
        }
        {
            const int a = s.csB[c0 + zlo], b = s.csB[c0 + zhi + 1];
            if (b > a) build_range_tile(smA, sPre[r + 9] + (a + s.bOff - sWin[r + 9].x), b - a, xi, s.r2list, -1, s.kmax, n, wp, jump);
        }
    }
    cnt[i] = n;
    // pad the open batch to its end with the dummy slot: the sweep reads whole batches of 8, also when kmax = 4 (mod 8).
    // The buffer holds kmax/4 planes of 16 bytes per particle (the int32 lists' layout), at least the ceil(kmax/8) needed here.
    if (n <= s.kmax)
        for (int m = n; m & 7; ++m) { *wp = static_cast<unsigned short>(T); ++wp; }
}

// The default list builder: the tile's candidate windows are staged in shared memory exactly as above (cp.async.bulk +
// mbarrier), the candidate tests read the staged records (lanes of one cell read the same slot: a broadcast), and the
// list it writes is the int32 per-particle list of k_build_list (global record indices, int4 batches, padded with the
// particle itself) -- entry for entry, so the list sweeps and the list tests do not care which builder ran.
// A tile whose windows exceed the staging capacity, and particles outside the grid, take the global-memory path.
// Each lane collects its hits four at a time in registers and writes one int4 per completed batch (not one 4-byte store
// per entry); the candidate tests of a chunk are built into the hit mask four at a time, with constant shifts.
#define SPHK_BUILD_CAP 2047
#define SPHK_BUILD_OVERREAD 3                       // records the 4-candidate groups may read past a range (masked out)
struct ListBatch {
    int4 e;                                         // the open batch; its newest entry in .w
    int n;                                          // entries appended so far (the true count, may exceed kmax)
    int4* wp;                                       // where the open batch goes: nbr4[(n / 4) * stride + i]
    __device__ __forceinline__ void push(int v, int stride, int kmax) {
        e = make_int4(e.y, e.z, e.w, v);
        if ((n & 3) == 3) {
            if (n < kmax) *wp = e;
            wp += stride;
        }
        ++n;
    }
};

// candidates [a, b) (record indices; slot = index + slotOff) against xi, hits except `self` appended in ascending order
__device__ __forceinline__ void build_range_staged(const float4* smA, int slotOff, int a, int b, float3 xi, float r2list, int self,
                                                   ListBatch& lb, int stride, int kmax) {
    for (int g0 = a; g0 < b; g0 += 32) {
        const int len = min(32, b - g0);
        const float4* base = smA + slotOff + g0;
        unsigned int mask = 0u;
        for (int k = 0; k < len; k += 4) {         // a group may run past len: those bits are cleared below
            const float3 d0 = xi - xyz(base[k]), d1 = xi - xyz(base[k + 1]);
            const float3 d2 = xi - xyz(base[k + 2]), d3 = xi - xyz(base[k + 3]);
            const unsigned int m4 = (dot3(d0, d0) <= r2list ? 1u : 0u) | (dot3(d1, d1) <= r2list ? 2u : 0u) |
                                    (dot3(d2, d2) <= r2list ? 4u : 0u) | (dot3(d3, d3) <= r2list ? 8u : 0u);
            mask |= m4 << k;
        }
        mask &= 0xffffffffu >> (32 - len);
        const int sf = self - g0;
        if (sf >= 0 && sf < 32) mask &= ~(1u << sf);
        while (mask) {
            const int k = __ffs(mask) - 1;
            mask &= mask - 1;
            lb.push(g0 + k, stride, kmax);
        }
    }
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_build_list_staged(const DevScene s, int* __restrict__ nbr, int* __restrict__ cnt, float4* __restrict__ posBuild, int2* __restrict__ tileWin) {
    extern __shared__ float4 smA[];                 // [SPHK_BUILD_CAP + 1 + SPHK_BUILD_OVERREAD]
    __shared__ unsigned long long bar;
    __shared__ int sMin, sMax, sOut;
    __shared__ int2 sWin[SPHK_TILE_WINS];
    __shared__ int sPre[SPHK_TILE_WINS + 1];
    const int tile = s.iBegin / SPHK_BLOCK + blockIdx.x;
    const int i = tile * SPHK_BLOCK + threadIdx.x;
    const bool have = i < s.nF;
    const int ncells = s.cs.x * s.cs.y * s.cs.z;
    if (threadIdx.x == 0) { sMin = 0x7fffffff; sMax = -1; sOut = 0; }
    __syncthreads();
    float4 lo = make_float4(0.f, 0.f, 0.f, 0.f);
    int cx = 0, cy = 0, cz = 0, c = ncells;
    if (have) {
        lo = rec_lo(s.rec + i);
        cx = cell_coord(lo.x, s.cellLength) - s.org.x; cy = cell_coord(lo.y, s.cellLength) - s.org.y; cz = cell_coord(lo.z, s.cellLength) - s.org.z;
        c = cell_index(cx, cy, cz, s.cs);
        if (c < ncells) { atomicMin(&sMin, c); atomicMax(&sMax, c); }
        else sOut = 1;
    }
    __syncthreads();
    if (threadIdx.x < SPHK_TILE_WINS) {
        const int2 w = tile_window(s, threadIdx.x, sMin, sMax, ncells);
        sWin[threadIdx.x] = w;
        // the fluid windows are the reach of the tile's sweeps (chunk activity, sweep_list_warp); a particle outside the grid
        // may reach past them: count -1 marks such a tile as unbounded
        if (threadIdx.x < 9) tileWin[static_cast<size_t>(tile) * SPHK_TILE_WINS + threadIdx.x] = (sOut && threadIdx.x == 0) ? make_int2(0, -1) : w;
    }
    __syncthreads();
    if (threadIdx.x == 0) tile_stage(s, sWin, sPre, smA, nullptr, false, &bar, SPHK_BUILD_CAP);
    __syncthreads();
    const int T = sPre[SPHK_TILE_WINS];
    const bool staged = T <= SPHK_BUILD_CAP;
    if (staged && T > 0) mbar_wait(&bar, 0);        // every thread: the block must not retire with bulk copies in flight
    if (!have || !in_range(s, i)) return;
    if (!staged || c >= ncells) { build_particle_global(s, i, lo, nbr, cnt, posBuild); return; }
    const float3 xi = xyz(lo);
    const int zlo = max(cz - 1, 0), zhi = min(cz + 1, s.cs.z - 1);
    ListBatch lb{make_int4(i, i, i, i), 0, reinterpret_cast<int4*>(nbr) + i};
#pragma unroll 1
    for (int r = 0; r < 9; ++r) {
        const int x = cx + r / 3 - 1, y = cy + r % 3 - 1;
        if (x < 0 || x >= s.cs.x || y < 0 || y >= s.cs.y) continue;
        const int c0 = (x * s.cs.y + y) * s.cs.z;
        build_range_staged(smA, sPre[r] - sWin[r].x, s.csF[c0 + zlo], s.csF[c0 + zhi + 1], xi, s.r2list, i, lb, s.nbrStride, s.kmax);
        const int a = s.csB[c0 + zlo], b = s.csB[c0 + zhi + 1];
        if (b > a) build_range_staged(smA, sPre[r + 9] - sWin[r + 9].x, a + s.bOff, b + s.bOff, xi, s.r2list, -1, lb, s.nbrStride, s.kmax);
    }
    cnt[i] = lb.n;
    if (lb.n < s.kmax)                              // pad the open batch with the particle itself
        while (lb.n & 3) lb.push(i, s.nbrStride, s.kmax);
}

// ---- sweep ----------------------------------------------------------------------------------------------------------------
// Operators that read a boundary neighbour's own data (heat transfer: its group) declare kIndex = true; the tile walk then
// recovers the record index of a boundary slot from the staged windows (the other operators get j = -1 there).
template <class Op, class = void> struct op_index : std::false_type {};
template <class Op> struct op_index<Op, std::void_t<decltype(Op::kIndex)>> : std::bool_constant<Op::kIndex> {};

template <class Op>
__device__ __forceinline__ void tile_pair(const DevScene& s, const Op& op, typename Op::Acc& acc, int i, float3 xi, int slot, int preB,
                                          const float4* smA, const float4* smB, float m0, const int2* sWin, const int* sPre) {
    const bool isB = slot >= preB;
    if (Op::kFluidOnly && isB) return;
    const float4 lo = smA[slot];
    float4 hi = make_float4(0.f, 0.f, 0.f, 0.f);
    if (Op::kHi) hi = smB[slot];
    const float3 d = xi - xyz(lo);
    int j = -1;
    if constexpr (op_index<Op>::value) {
        if (isB && slot < sPre[SPHK_TILE_WINS]) {   // (the dummy slot past the windows keeps -1)
            int w = SPHK_TILE_WINS - 1;
            while (w > 9 && sPre[w] > slot) --w;
            j = sWin[w].x + (slot - sPre[w]);
        }
    }
    feed_pair(s, op, acc, i, xi, j, isB, lo, hi, m0, d, dot3(d, d));
}

template <class Op>
__global__ void __launch_bounds__(SPHK_BLOCK) k_sweep_tile(const DevScene s, const Op op) {
    extern __shared__ float4 sm[];                  // A[SPHK_TILE_CAP + 1], then B[SPHK_TILE_CAP + 1] for velocity sweeps
    if (s.pred && *s.pred == 0) return;
    float4* smA = sm;
    float4* smB = sm + (SPHK_TILE_CAP + 1);
    __shared__ unsigned long long bar;
    __shared__ int2 sWin[SPHK_TILE_WINS];
    __shared__ int sPre[SPHK_TILE_WINS + 1];
    const int tile = s.iBegin / SPHK_BLOCK + blockIdx.x;
    const int i = tile * SPHK_BLOCK + threadIdx.x;
    const bool on = in_range(s, i);
    if (threadIdx.x < SPHK_TILE_WINS) sWin[threadIdx.x] = s.tileWin[static_cast<size_t>(tile) * SPHK_TILE_WINS + threadIdx.x];
    __syncthreads();
    if (threadIdx.x == 0) tile_stage(s, sWin, sPre, smA, smB, Op::kHi, &bar);
    __syncthreads();
    const int T = sPre[SPHK_TILE_WINS];
    if (!on) {                                      // (the block must not retire with bulk copies in flight)
        if (T > 0 && T <= SPHK_TILE_CAP) mbar_wait(&bar, 0);
        return;
    }
    // own data and the first list batch travel while the bulk copies are in flight
    float4 lo, hi;
    rec_full(s.rec + i, lo, hi);
    const float3 xi = xyz(lo);
    typename Op::Acc acc;
    op.begin(acc, i, lo, hi, s);
    int n = s.cnt[i];
    const float m0 = uniform_mass(s);
    if (s.cellFlag) {                                  // skin list: a fast mover is (or was) within reach of this cell -> exact walk
        const int c = cell_index(cell_coord(lo.x, s.cellLength) - s.org.x, cell_coord(lo.y, s.cellLength) - s.org.y,
                                 cell_coord(lo.z, s.cellLength) - s.org.z, s.cs);
        if (c >= s.cs.x * s.cs.y * s.cs.z || s.cellFlag[c]) n = s.kmax + 1;
    }
    if (!Op::kHi && m0 < 0.f) n = s.kmax + 1;                      // non-uniform fluid masses: a sweep that stages A only has no neighbour mass
    if (n <= s.kmax && T <= SPHK_TILE_CAP) {
        const int nb8 = (n + 7) >> 3;
        const uint4* __restrict__ row = reinterpret_cast<const uint4*>(s.nbr) + i;
        uint4 jn = make_uint4(0u, 0u, 0u, 0u);
        if (nb8 > 0) jn = __ldcs(row);
        if (T > 0) mbar_wait(&bar, 0);
        const int preB = sPre[9];
        for (int b = 0; b < nb8; ++b) {
            const uint4 j8 = jn;
            row += s.nbrStride;
            if (b + 1 < nb8) jn = __ldcs(row);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.x & 0xffffu), preB, smA, smB, m0, sWin, sPre);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.x >> 16), preB, smA, smB, m0, sWin, sPre);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.y & 0xffffu), preB, smA, smB, m0, sWin, sPre);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.y >> 16), preB, smA, smB, m0, sWin, sPre);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.z & 0xffffu), preB, smA, smB, m0, sWin, sPre);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.z >> 16), preB, smA, smB, m0, sWin, sPre);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.w & 0xffffu), preB, smA, smB, m0, sWin, sPre);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.w >> 16), preB, smA, smB, m0, sWin, sPre);
        }
    } else {
        if (T > 0 && T <= SPHK_TILE_CAP) mbar_wait(&bar, 0);
        walk_cells(s, op, acc, i, lo, m0);          // exact fallback (global gathers)
    }
    op.end(acc, i, lo, hi, s);
}

// Dedicated neighbour-list builder (the generic k_sweep_cells<OpBuildList> is kept as the simple reference of
// what it computes; tests compare the two lists entry by entry).  Same candidate order as walk_cells.
// The generic walk is issue-bound by SIMT divergence: ~15% of the candidates are hits, so with 32 lanes the
// "append" path runs on almost every iteration at ~5/32 lane utilisation (ncu: 27 warp instructions per
// candidate).  Here each chunk of <= 32 candidates is processed in two convergent phases:
//   1. distance tests only, hits recorded as bits of a per-thread mask (no branches);
//   2. the set bits are walked (find-first-set) and appended through a running pointer -- the trip count is
//      the warp's maximum hit count (~7), not the candidate count.
__device__ __forceinline__ void build_range(const DevScene& s, float3 xi, int i, int a, int b, int off, int& n, int*& wp,
                                            long long jump) {
    for (int j0 = a; j0 < b; j0 += 32) {
        const int len = min(32, b - j0);
        const Rec base = s.rec + off + j0;
        unsigned int mask = 0u;
#pragma unroll 4
        for (int k = 0; k < len; ++k) {
            const float3 d = xi - xyz(rec_lo(base + k));
            mask |= (dot3(d, d) <= s.r2list ? 1u : 0u) << k;
        }
        const int self = i - (off + j0);
        if (self >= 0 && self < 32) mask &= ~(1u << self);
        while (mask) {
            const int k = __ffs(mask) - 1;
            mask &= mask - 1;
            if (n < s.kmax) *wp = off + j0 + k;
            wp += ((n & 3) == 3) ? jump : 1;
            ++n;
        }
    }
}

__device__ __forceinline__ void build_particle_global(const DevScene& s, int i, float4 lo, int* __restrict__ nbr, int* __restrict__ cnt,
                                                      float4* __restrict__ posBuild) {
    const float3 xi = xyz(lo);
    const int cx = cell_coord(lo.x, s.cellLength) - s.org.x, cy = cell_coord(lo.y, s.cellLength) - s.org.y,
              cz = cell_coord(lo.z, s.cellLength) - s.org.z;
    const int zlo = max(cz - 1, 0), zhi = min(cz + 1, s.cs.z - 1);
    int n = 0;
    int* wp = nbr + static_cast<size_t>(i) * 4;                       // slot of entry 0: nbr4[0 * stride + i].x
    const long long jump = static_cast<long long>(s.nbrStride) * 4 - 3;  // from .w of batch b to .x of batch b+1
    if (zlo <= zhi) {
#pragma unroll 1
        for (int r = 0; r < 9; ++r) {
            const int x = cx + r / 3 - 1, y = cy + r % 3 - 1;
            if (x < 0 || x >= s.cs.x || y < 0 || y >= s.cs.y) continue;
            const int c0 = (x * s.cs.y + y) * s.cs.z;
            build_range(s, xi, i, s.csF[c0 + zlo], s.csF[c0 + zhi + 1], 0, n, wp, jump);
            build_range(s, xi, i, s.csB[c0 + zlo], s.csB[c0 + zhi + 1], s.bOff, n, wp, jump);
        }
    }
    cnt[i] = n;
    // pad the open batch with the particle itself: the self pair contributes exactly 0 to every operator
    for (int m = n; (m & 3) && m < s.kmax; ++m) { *wp = i; ++wp; }
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_build_list(const DevScene s, int* __restrict__ nbr, int* __restrict__ cnt, float4* __restrict__ posBuild) {
    const int i = s.iBegin + blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (!in_range(s, i)) return;
    build_particle_global(s, i, rec_lo(s.rec + i), nbr, cnt, posBuild);
}

// computeBoundaryMass_CUDA, SPHSystem.cu:79-105: boundary particles against the boundary set only
__global__ void __launch_bounds__(SPHK_BLOCK)
k_boundary_mass(Rec recB, float* __restrict__ mass, int n, const int* __restrict__ csB, int3 cs, int3 org,
                float cellLength, float rhoB, KConst k, const float4* __restrict__ bodyLocal) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float4 pi = rec_lo(recB + i);
    // with kinematic bodies the sum runs over the particle's own group (the static set, or its body): per-group Akinci
    const float gi = bodyLocal ? body_group(bodyLocal[i]) : 0.f;
    const int cx = cell_coord(pi.x, cellLength) - org.x, cy = cell_coord(pi.y, cellLength) - org.y,
              cz = cell_coord(pi.z, cellLength) - org.z;
    float sum = 0.f;
    for (int m = 0; m < 27; ++m) {
        const int c = cell_index(cx + m / 9 - 1, cy + (m % 9) / 3 - 1, cz + m % 3 - 1, cs);
        if (c == cs.x * cs.y * cs.z) continue;
        const int end = csB[c + 1];
        for (int j = csB[c]; j < end; ++j) {
            if (bodyLocal && body_group(bodyLocal[j]) != gi) continue;
            const float3 d = xyz(pi) - xyz(rec_lo(recB + j));
            sum += w_cubic(sqrtf(dot3(d, d)), k);
        }
    }
    mass[i] = rhoB / fmaxf(SPHK_EPS, sum);
}
// boundary records: the mass lives in both halves (A.w for sweeps that gather A only, B.w for the others)
__global__ void __launch_bounds__(SPHK_BLOCK) k_set_mass(Rec rec, const float* __restrict__ mass, int n) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i < n) { const float m = mass[i]; rec.a[i].w = m; rec.b[i].w = m; }
}

// ---- element-wise kernels -------------------------------------------------------------------------
__global__ void __launch_bounds__(SPHK_BLOCK) k_gravity(Rec rec, float* __restrict__ vel, int n, float3 dv) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float4 hi = rec_hi(rec + i);
    const float3 v = f3(hi.x + dv.x, hi.y + dv.y, hi.z + dv.z);
    rec_set_vel(rec + i, v); store3(vel, i, v);
}

// computePressure_CUDA, BasicSPHSolver.cu:103-111
__global__ void __launch_bounds__(SPHK_BLOCK)
k_pressure(const float* __restrict__ density, float* __restrict__ pressure, int n, float rho0, float stiff) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    float p = stiff * (powf((density[i] / rho0), 7) - 1.0f);
    if (p < 0.0f) p = 0.0f;
    pressure[i] = p;
}
// rec.s producers for the sweeps whose neighbour scalar is not written by the preceding sweep
__global__ void __launch_bounds__(SPHK_BLOCK)
k_s_prho(const float* __restrict__ density, const float* __restrict__ pressure, Rec rec, int n) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i < n) rec_set_s(rec + i, pressure[i] / fmaxf(SPHK_EPS, density[i] * density[i]));
}
__global__ void __launch_bounds__(SPHK_BLOCK) k_s_cg2(const float* __restrict__ cg, Rec rec, int n) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float3 c = load3(cg, i);
    rec_set_s(rec + i, dot3(c, c));
}
// (+ the chunk activity of the copied scalar: -0 is quiet, sweep_list_warp)
__global__ void __launch_bounds__(SPHK_BLOCK) k_s_copy(const float* __restrict__ a, Rec rec, int n, unsigned int* __restrict__ act) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    float v = 0.f;
    if (i < n) { v = a[i]; rec_set_s(rec + i, v); }
    const unsigned int b = __ballot_sync(0xffffffffu, !(i < n && __float_as_uint(v) == 0x80000000u));
    if ((threadIdx.x & 31) == 0 && i < n) act[i >> 5] = b;
}

// Particles::advect (Particles.cu:28-36) + enforceBoundary_CUDA(pos, vel) (BasicSPHSolver.cu:85-96)
__device__ __forceinline__ void clamp_axis(float& p, float* v, float L) {
    if (p <= L * .00f) { p = L * .00f; if (v) *v = fmaxf(*v, 0.0f); }
    if (p >= L * .99f) { p = L * .99f; if (v) *v = fminf(*v, 0.0f); }
}
__global__ void __launch_bounds__(SPHK_BLOCK)
k_advect(Rec rec, float* __restrict__ pos, float* __restrict__ vel, int n, float dt, float3 space) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    float4 p, v;
    rec_full(rec + i, p, v);
    p.x = p.x + dt * v.x; p.y = p.y + dt * v.y; p.z = p.z + dt * v.z;
    clamp_axis(p.x, &v.x, space.x); clamp_axis(p.y, &v.y, space.y); clamp_axis(p.z, &v.z, space.z);
    rec_store(rec + i, p, v);
    store3(pos, i, xyz(p)); store3(vel, i, xyz(v));
}
// thrust::transform(pos += dpos) + enforceBoundary_CUDA(pos), PBDSolver.cu:212-223,247-253
__global__ void __launch_bounds__(SPHK_BLOCK)
k_apply_delta_pos(Rec rec, float* __restrict__ pos, const float* __restrict__ dpos, int n, float3 space, const SkinTrack track) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    float d2 = 0.f;
    if (i < n) {
        float4 p = rec_lo(rec + i);
        const float3 d = load3(dpos, i);
        p.x += d.x; p.y += d.y; p.z += d.z;
        clamp_axis(p.x, nullptr, space.x); clamp_axis(p.y, nullptr, space.y); clamp_axis(p.z, nullptr, space.z);
        rec_set_pos(rec + i, xyz(p)); store3(pos, i, xyz(p));
        if (track.posBuild) d2 = skin_track(track, i, xyz(p));
    }
    if (track.posBuild) skin_track_max(track, d2);
}
// vel = (pos - posLast) / dt, PBDSolver.cu:55-60
__global__ void __launch_bounds__(SPHK_BLOCK)
k_vel_from_pos(Rec rec, const float* __restrict__ posLast, float* __restrict__ vel, int n, float dt) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float3 v = (xyz(rec_lo(rec + i)) - load3(posLast, i)) / dt;
    rec_set_vel(rec + i, v); store3(vel, i, v);
}
__global__ void __launch_bounds__(SPHK_BLOCK)
k_commit_vel(const float4* __restrict__ src, Rec rec, float* __restrict__ vel, int begin, int end, const int* __restrict__ rangeDev) {
    const int i = begin + blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= end) return;
    if (rangeDev && (i < rangeDev[0] || i >= rangeDev[0] + rangeDev[1])) return;
    const float3 v = xyz(src[i]);
    rec_set_vel(rec + i, v);
    if (vel) store3(vel, i, v);
}
__global__ void __launch_bounds__(256) k_list_stats(const int* __restrict__ cnt, int n, int kmax, unsigned long long* out) {
    unsigned long long mx = 0, ov = 0, tot = 0;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
        const int c = cnt[i];
        if (c > mx) mx = c;
        ov += c > kmax; tot += c;
    }
    atomicMax(out, mx); atomicAdd(out + 1, ov); atomicAdd(out + 2, tot);
}

// =================================================================================================
// Host side
// =================================================================================================
static int check_scene(const sphk_ctx* c, const sphk_scene* s) {
    if (!c || !s) return SPHK_ERR_INVALID;
    if (!c->fluidSearched || !c->boundarySearched) return SPHK_ERR_STATE;
    if (s->fluid.n != c->nF || s->boundary.n != c->nB) return SPHK_ERR_STATE;
    if (!s->cell_start_fluid || !s->cell_start_boundary || !s->fluid.pos || !s->fluid.vel) return SPHK_ERR_INVALID;
    if (!(s->radius > 0.f)) return SPHK_ERR_INVALID;
    c->countSettable = false;           // the first sweep after a search closes sphk_fluid_set_count's window
    return SPHK_OK;
}

static KConst kernel_constants(float R) {
    const double pi = 3.14159265358979323846, r = R;
    KConst k;
    k.R = R;
    k.hInv = static_cast<float>(2.0 / r);
    k.cW = static_cast<float>(0.25 / (pi * r * r * r));
    k.cG = static_cast<float>(1.0 / (pi * r * r * r * r * r));
    k.cLap = static_cast<float>(45.0 / (pi * r * r * r * r * r * r));
    k.cST = static_cast<float>(136.0241 / (pi * r * r * r * r * r * r * r * r * r));
    k.stOff = static_cast<float>(0.0156 * r * r * r * r * r * r);
    // candidates beyond the support contribute exactly 0 to every operator; the margin only covers the
    // approximate sqrt of the support tests (q > 2, r <= R)
    k.r2cut = R * R * (1.0f + 1e-5f);
    return k;
}

static DevScene dev_scene(const sphk_ctx* c, const sphk_scene* s) {
    DevScene d;
    d.rec = c->rec; d.csF = s->cell_start_fluid; d.csB = s->cell_start_boundary;
    d.nbr = c->nbr; d.cnt = c->cnt; d.massRange = c->massRange;
    d.nF = c->nF; d.bOff = c->capF;
    d.nbrStride = c->capF; d.kmax = c->kmax;
    d.dummy = c->capF + c->capB;
    d.tileWin = c->tileWin;
    d.pred = c->pred;
    d.cs = c->cs; d.org = c->org; d.cellLength = c->cellLength;
    d.iBegin = c->actCount < 0 ? 0 : c->actBegin;
    d.iEnd = c->actCount < 0 ? c->nF : c->actBegin + c->actCount;
    d.rangeDev = c->rangeDev;
    d.patch = c->patch;
    if (c->rangeDev) { d.iBegin = 0; d.iEnd = c->nF; }      // launched over everything, cut on the device
    d.k = kernel_constants(s->radius);
    d.r2list = d.k.r2cut;
    d.cellFlag = nullptr;
    d.act = nullptr; d.stamp = nullptr; d.seq = 0; d.reuse = 0;
    d.mark = nullptr; d.trust = 0;
    return d;
}

// Chunk activity on the host (sweep_list_warp).  Every launch counts in c->launches; the launches known to leave rec.s and all
// an error sweep reads alone -- except velocities moved under chunk stamps by the correct sweeps -- also count in c->credited
// (correct sweeps, loop control, reductions).  So act_mark() stays put across exactly those: the chunk bits stay valid, and the
// last error sweep's outputs stay reusable, until anything else is launched.  Host-side only: a captured step repeats the order
// of its calls and with it these decisions; what depends on data (which chunks are quiet) is decided on the device.
static long long act_mark(const sphk_ctx* c) { return c->launches - c->credited; }
// Velocity epochs (sweep_list_warp) in the same pattern: vel_mark() stays put across the launches that leave vel and rec.b alone
// and across the correct sweeps that keep the marks; anything else -- a launch, or a copy over the velocities -- ends the epoch.
static long long vel_mark(const sphk_ctx* c) { return c->launches - c->velCredited; }
static bool same_bits(float a, float b) { unsigned int x, y; std::memcpy(&x, &a, 4); std::memcpy(&y, &b, 4); return x == y; }

SkinTrack sphk_skin_track(const sphk_ctx* c, float radius, bool on) {
    SkinTrack t;
    const float half = 0.5f * c->skin * radius;
    t.posBuild = on ? c->snapA : nullptr;
    t.dispMax = c->dispMax; t.cellFlag = c->cellFlag; t.limit2 = half * half;
    t.cs = c->cs; t.org = c->org; t.cellLength = c->cellLength;
    return t;
}

static int ensure_list(sphk_ctx* c, const DevScene& d) {
    // lists are built for the particles the sweeps will compute (the active range: ghosts of a slab rank need none).  A
    // device-resident range is not known to the host, and its contents may change between sweeps: the lists are then built for
    // all nF particles (d.iBegin = 0, d.iEnd = nF), so any range the device later holds finds its lists.
    if (c->listEpoch == c->searchEpoch && d.iBegin >= c->listBegin && d.iEnd <= c->listEnd) return SPHK_OK;
    if (!c->nbr) {
        const size_t bytes = sizeof(int) * static_cast<size_t>(c->kmax) * (static_cast<size_t>(c->capF) + 2);
        if (cudaMalloc(reinterpret_cast<void**>(&c->nbr), bytes) != cudaSuccess) { cudaGetLastError(); return SPHK_ERR_ALLOC; }
    }
    DevScene b = d;
    b.nbr = c->nbr;
    b.rangeDev = nullptr;
    c->listBegin = d.iBegin; c->listEnd = d.iEnd;
    c->listSpans = false;
    c->listHasSkin = c->skin > 0.f;
    if (c->listHasSkin) {
        const float rs = d.k.R * (1.0f + c->skin);
        b.r2list = rs * rs * (1.0f + 1e-5f);
        if (cudaMemsetAsync(c->dispMax, 0, sizeof(unsigned int), c->stream) != cudaSuccess) return SPHK_ERR_STATE;
        if (cudaMemsetAsync(c->cellFlag, 0, static_cast<size_t>(c->ncells) + 1, c->stream) != cudaSuccess) return SPHK_ERR_STATE;
        // positions at build time of EVERY local particle (ghosts of a slab rank included: their owners move them)
        if (cudaMemcpyAsync(c->snapA, c->rec.a, sizeof(float4) * static_cast<size_t>(c->nF), cudaMemcpyDeviceToDevice, c->stream) != cudaSuccess)
            return SPHK_ERR_STATE;
    }
    if (c->tile) {
        static bool attr = false;
        const int smem = (SPHK_TILE_CAP + 1) * 16;
        if (!attr) { cudaFuncSetAttribute(k_build_tile, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); attr = true; }
        const int tiles = (b.iEnd + SPHK_BLOCK - 1) / SPHK_BLOCK - b.iBegin / SPHK_BLOCK;
        k_build_tile<<<tiles, SPHK_BLOCK, smem, c->stream>>>(b, reinterpret_cast<unsigned short*>(c->nbr), c->cnt,
                                                              nullptr, c->tileWin);
    } else if (c->simpleBuild) {
        OpBuildList op{c->nbr, c->cnt, nullptr};
        k_sweep_cells<OpBuildList><<<sphk_blocks(b.iEnd - b.iBegin), SPHK_BLOCK, 0, c->stream>>>(b, op);
    } else if (c->stagedBuild) {
        static bool attr = false;
        const int smem = (SPHK_BUILD_CAP + 1 + SPHK_BUILD_OVERREAD) * 16;
        if (!attr) { cudaFuncSetAttribute(k_build_list_staged, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); attr = true; }
        const int tiles = (b.iEnd + SPHK_BLOCK - 1) / SPHK_BLOCK - b.iBegin / SPHK_BLOCK;
        k_build_list_staged<<<tiles, SPHK_BLOCK, smem, c->stream>>>(b, c->nbr, c->cnt, nullptr, c->tileWin);
        c->listSpans = b.iBegin == 0 && b.iEnd == c->nF;
    } else {
        k_build_list<<<sphk_blocks(b.iEnd - b.iBegin), SPHK_BLOCK, 0, c->stream>>>(b, c->nbr, c->cnt, nullptr);
    }
    c->launches++;
    c->listEpoch = c->searchEpoch;
    return SPHK_OK;
}

// kept (DFSPH error and correct sweeps): the launch kept chunk activity -- a list sweep over every chunk whose list builder recorded
// the tiles' windows.  reuse (error sweeps): the token matches, chunks quiet since it may keep their outputs.
template <class Op> static int run_sweep(sphk_ctx* c, const sphk_scene* s, const Op& op, bool* kept = nullptr, bool reuse = false) {
    constexpr int role = act_of<Op>::role;
    DevScene d = dev_scene(c, s);
    if (kept) *kept = false;
    if (d.iEnd <= d.iBegin) return SPHK_OK;
    // the list is usable while positions are those of the search, or -- skin lists -- while the particles have
    // only been moved by sphk_pbd_delta_pos_apply (displacement tracked on the device against skin/2)
    const bool list = c->useList && (!c->posDirty || (c->skin > 0.f && !c->advected));
    if (list) {
        const int rc = ensure_list(c, d);
        if (rc != SPHK_OK) return rc;
        d.nbr = c->nbr;
        if (c->listHasSkin) d.cellFlag = c->cellFlag;
        if (c->tile) {
            static bool attr = false;
            const int smem = (SPHK_TILE_CAP + 1) * 16 * (Op::kHi ? 2 : 1);
            if (!attr) { cudaFuncSetAttribute(k_sweep_tile<Op>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); attr = true; }
            const int tiles = (d.iEnd + SPHK_BLOCK - 1) / SPHK_BLOCK - d.iBegin / SPHK_BLOCK;
            k_sweep_tile<Op><<<tiles, SPHK_BLOCK, smem, c->stream>>>(d, op);
        }
        else {
            if (role != kActNone && c->listSpans && d.iBegin == 0 && d.iEnd == c->nF) {
                if (kept) *kept = true;
                if (role == kActError) {
                    d.act = c->chunkAct;
                    if (reuse) { d.reuse = 1; d.stamp = c->chunkStamp; d.seq = c->tok.seq; }
                } else {
                    d.stamp = c->chunkStamp;
                    d.seq = ++c->corrSeq;
                    if (c->actMark == act_mark(c)) d.act = c->chunkAct;
                    if constexpr (role == kActCorrect) {
                        if (op.quiet_adds_zero()) {   // else: a quiet pass is no fixed point of the others -- no marks, the epoch ends
                            d.mark = c->chunkMark;
                            d.trust = c->velMark == vel_mark(c) && c->velArr == s->fluid.vel;
                        }
                    }
                }
            }
            int blocks = sphk_blocks(d.iEnd - d.iBegin);
            if (d.patch > 0) blocks = (blocks + d.patch - 1) / d.patch * d.patch;      // whole groups (4 * patch chunks = patch blocks)
            if (d.act || d.stamp) {
                if constexpr (role != kActNone) k_sweep_list_act<Op><<<blocks, SPHK_BLOCK, 0, c->stream>>>(d, op);
            } else {
                k_sweep_list<Op><<<blocks, SPHK_BLOCK, 0, c->stream>>>(d, op);
            }
        }
    } else {
        k_sweep_cells<Op><<<sphk_blocks(d.iEnd - d.iBegin), SPHK_BLOCK, 0, c->stream>>>(d, op);
    }
    c->launches++;
    if (role == kActCorrect) c->credited++;           // velocities only; stamped, or the caller drops the token
    if (role == kActError || d.mark) c->velCredited++;   // the error sweeps write no velocity; a marked correct sweep keeps its marks
    if (d.mark) { c->velMark = vel_mark(c); c->velArr = s->fluid.vel; }
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// after a DFSPH error sweep (kind 1 divergence -- also the fused sweep --, 2 density): its chunk bits and reuse token
static void error_swept(sphk_ctx* c, bool kept, int kind, const sphk_scene* s, const float* alpha, const float* error, const float* stiff,
                        float dt, float rho0) {
    c->actMark = kept ? act_mark(c) : -1;
    c->tok.kind = kept ? kind : 0;
    c->tok.density = s->fluid.density; c->tok.alpha = alpha; c->tok.error = error; c->tok.stiff = stiff;
    c->tok.dt = dt; c->tok.rho0 = rho0;
    c->tok.mark = act_mark(c);
    c->tok.seq = c->corrSeq;
}
static bool error_reusable(const sphk_ctx* c, int kind, const sphk_scene* s, const float* alpha, const float* error, const float* stiff,
                           float dt, float rho0) {
    const auto& k = c->tok;
    return k.kind == kind && k.mark == act_mark(c) && c->actMark == k.mark && c->sTag == stiff && k.density == s->fluid.density &&
           k.alpha == alpha && k.error == error && k.stiff == stiff && same_bits(k.dt, dt) && same_bits(k.rho0, rho0);
}

// rec.s must mirror `array` before a sweep that gathers it; skipped when the previous sweep wrote both
static void ensure_scalar(sphk_ctx* c, const float* array) {
    if (c->sTag == array) return;
    k_s_copy<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(array, c->rec, c->nF, c->chunkAct);
    c->launches++; c->velCredited++;
    c->actMark = act_mark(c);
    c->sTag = array;
}

#define SPHK_CHECK_SCENE(c, s) do { const int rc_ = check_scene((c), (s)); if (rc_ != SPHK_OK) return rc_; } while (0)

extern "C" int sphk_boundary_mass(sphk_ctx* c, const sphk_particles* b, const int* csB, float rhoB, float R) {
    if (!c || !b || !csB || !b->mass) return SPHK_ERR_INVALID;
    if (!c->boundarySearched || b->n != c->nB) return SPHK_ERR_STATE;
    const Rec recB = c->rec + c->capF;
    k_boundary_mass<<<sphk_blocks(c->nB), SPHK_BLOCK, 0, c->stream>>>(recB, b->mass, c->nB, csB, c->cs, c->org, c->cellLength, rhoB,
                                                                     kernel_constants(R), c->bodies ? c->bodies->local : nullptr);
    k_set_mass<<<sphk_blocks(c->nB), SPHK_BLOCK, 0, c->stream>>>(recB, b->mass, c->nB);
    c->launches += 2;
    c->listEpoch = ~0ull;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_gravity(sphk_ctx* c, const sphk_scene* s, float dt, const float G[3]) {
    SPHK_CHECK_SCENE(c, s);
    if (!G) return SPHK_ERR_INVALID;
    const float3 dv = make_float3(dt * G[0], dt * G[1], dt * G[2]);   // const auto dv = dt * G, BasicSPHSolver.cu:229
    k_gravity<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(c->rec, s->fluid.vel, c->nF, dv);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_viscosity(sphk_ctx* c, const sphk_scene* s, float* delta_v, float rho0, float visc, float dt) {
    SPHK_CHECK_SCENE(c, s);
    if (!delta_v) return SPHK_ERR_INVALID;
    // Jacobi: every thread reads neighbours' OLD velocity (the reference writes deltaV to a buffer and adds
    // afterwards); new velocities go to a temp and are committed to the records by a second pass.
    float4* tmp = c->snapB;
    OpViscosity op{tmp, s->fluid.vel, delta_v, rho0, visc, dt};
    const int rc = run_sweep(c, s, op);
    if (rc != SPHK_OK) return rc;
    const int b = (c->actCount < 0 || c->rangeDev) ? 0 : c->actBegin, e = (c->actCount < 0 || c->rangeDev) ? c->nF : c->actBegin + c->actCount;
    if (e > b) k_commit_vel<<<sphk_blocks(e - b), SPHK_BLOCK, 0, c->stream>>>(tmp, c->rec, nullptr, b, e, c->rangeDev);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_color_grad(sphk_ctx* c, const sphk_scene* s, float* color_grad, float rho0, float rhoB) {
    SPHK_CHECK_SCENE(c, s);
    if (!color_grad) return SPHK_ERR_INVALID;
    OpColorGrad op{color_grad, rho0, rhoB};
    return run_sweep(c, s, op);
}

extern "C" int sphk_surface(sphk_ctx* c, const sphk_scene* s, const float* color_grad, float dt, float rho0,
                            float kappa, float airP) {
    SPHK_CHECK_SCENE(c, s);
    if (!color_grad) return SPHK_ERR_INVALID;
    k_s_cg2<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(color_grad, c->rec, c->nF);
    c->launches++;
    c->sTag = nullptr;
    OpSurface op{c->rec, s->fluid.vel, dt, rho0, kappa, airP};
    return run_sweep(c, s, op);
}

extern "C" int sphk_density(sphk_ctx* c, const sphk_scene* s) {
    SPHK_CHECK_SCENE(c, s);
    if (!s->fluid.density) return SPHK_ERR_INVALID;
    OpDensity op{s->fluid.density};
    return run_sweep(c, s, op);
}

extern "C" int sphk_pressure(sphk_ctx* c, const sphk_scene* s, float rho0, float stiff) {
    SPHK_CHECK_SCENE(c, s);
    if (!s->fluid.density || !s->fluid.pressure) return SPHK_ERR_INVALID;
    k_pressure<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(s->fluid.density, s->fluid.pressure, c->nF, rho0, stiff);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_pressure_force(sphk_ctx* c, const sphk_scene* s, float dt) {
    SPHK_CHECK_SCENE(c, s);
    if (!s->fluid.density || !s->fluid.pressure) return SPHK_ERR_INVALID;
    k_s_prho<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(s->fluid.density, s->fluid.pressure, c->rec, c->nF);
    c->launches++;
    c->sTag = nullptr;
    OpPressureForce op{c->rec, s->fluid.vel, dt};
    return run_sweep(c, s, op);
}

extern "C" int sphk_advect(sphk_ctx* c, const sphk_scene* s, float dt, const float space[3]) {
    SPHK_CHECK_SCENE(c, s);
    if (!space) return SPHK_ERR_INVALID;
    k_advect<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(c->rec, s->fluid.pos, s->fluid.vel, c->nF, dt,
                                                              make_float3(space[0], space[1], space[2]));
    c->launches++;
    c->posDirty = true;
    c->advected = true;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_dfsph_density_alpha(sphk_ctx* c, const sphk_scene* s, float* alpha) {
    SPHK_CHECK_SCENE(c, s);
    if (!alpha || !s->fluid.density) return SPHK_ERR_INVALID;
    OpDensityAlpha op{s->fluid.density, alpha};
    return run_sweep(c, s, op);
}

extern "C" int sphk_dfsph_div_error(sphk_ctx* c, const sphk_scene* s, const float* alpha, float* error, float* stiff,
                                    float dt, float rho0) {
    SPHK_CHECK_SCENE(c, s);
    if (!alpha || !error || !stiff || !s->fluid.density) return SPHK_ERR_INVALID;
    OpDfsphError<false> op{c->rec, s->fluid.density, alpha, error, stiff, nullptr, dt, rho0};
    bool kept;
    const int rc = run_sweep(c, s, op, &kept, error_reusable(c, 1, s, alpha, error, stiff, dt, rho0));
    error_swept(c, kept, 1, s, alpha, error, stiff, dt, rho0);
    c->sTag = stiff;
    return rc;
}

extern "C" int sphk_dfsph_den_error(sphk_ctx* c, const sphk_scene* s, const float* alpha, float* error, float* stiff,
                                    float dt, float rho0, float* warm) {
    SPHK_CHECK_SCENE(c, s);
    if (!alpha || !error || !stiff || !s->fluid.density) return SPHK_ERR_INVALID;
    if (warm == c->sTag) c->sTag = nullptr;
    OpDfsphError<true> op{c->rec, s->fluid.density, alpha, error, stiff, warm, dt, rho0};
    bool kept;
    const int rc = run_sweep(c, s, op, &kept, error_reusable(c, 2, s, alpha, error, stiff, dt, rho0));
    error_swept(c, kept, 2, s, alpha, error, stiff, dt, rho0);
    c->sTag = stiff;
    return rc;
}

extern "C" int sphk_dfsph_div_correct(sphk_ctx* c, const sphk_scene* s, const float* stiff) {
    SPHK_CHECK_SCENE(c, s);
    if (!stiff) return SPHK_ERR_INVALID;
    ensure_scalar(c, stiff);
    OpScalarGradient<0> op{c->rec, s->fluid.vel, nullptr, 1.0f};
    bool kept;
    const int rc = run_sweep(c, s, op, &kept);
    if (!kept) c->tok.kind = 0;                       // velocities moved without stamps
    return rc;
}

extern "C" int sphk_dfsph_den_correct(sphk_ctx* c, const sphk_scene* s, const float* stiff, float dt) {
    SPHK_CHECK_SCENE(c, s);
    if (!stiff) return SPHK_ERR_INVALID;
    ensure_scalar(c, stiff);
    OpScalarGradient<1> op{c->rec, s->fluid.vel, nullptr, dt};
    bool kept;
    const int rc = run_sweep(c, s, op, &kept);
    if (!kept) c->tok.kind = 0;                       // velocities moved without stamps
    return rc;
}

extern "C" int sphk_pbd_density_lambda(sphk_ctx* c, const sphk_scene* s, float* lambda, float rho0, float relaxation) {
    SPHK_CHECK_SCENE(c, s);
    if (!lambda || !s->fluid.density) return SPHK_ERR_INVALID;
    OpPbdLambda op{c->rec, s->fluid.density, lambda, rho0, (rho0 != 0.0f) ? 1.0f : 0.0f, relaxation};
    const int rc = run_sweep(c, s, op);
    c->sTag = lambda;
    return rc;
}

extern "C" int sphk_pbd_delta_pos_apply(sphk_ctx* c, const sphk_scene* s, const float* lambda, float* delta_pos,
                                        float rho0, const float space[3]) {
    SPHK_CHECK_SCENE(c, s);
    if (!lambda || !delta_pos || !space) return SPHK_ERR_INVALID;
    ensure_scalar(c, lambda);
    OpScalarGradient<2> op{c->rec, nullptr, delta_pos, rho0};
    const int rc = run_sweep(c, s, op);
    if (rc != SPHK_OK) return rc;
    const bool track = c->listHasSkin && c->listEpoch == c->searchEpoch;
    k_apply_delta_pos<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(c->rec, s->fluid.pos, delta_pos, c->nF,
                                                                       make_float3(space[0], space[1], space[2]),
                                                                       sphk_skin_track(c, s->radius, track));
    c->launches++;
    c->posDirty = true;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// ---- two-way coupled bodies: the fluid's reaction on them (DESIGN.md section 2.4) ---------------------------------------------
// One thread per boundary slot; body particles only.  Walks the fluid cells within `reach` cells of the particle with the
// fluid cell ranges of the search and forms each pair term as the fluid sweep forms it.  The body particle gathers the pair's
// reaction and its moment about the body's centre into its own declaration slot of acc, in double (no atomics: every slot has
// one writer, sums are in walk order).  The pair term is a template:
//   ReactGradW     g = (m_k s_i) (d gradWfactor), d = x_i - x_k; the fluid particle received c m_i g, the body gathers -c m_i g
//   ReactAdhesion  the fluid particle received dt beta_g Psi_k A(r) (-d / r) per unit mass (section 2.11), the body gathers
//                  +dt beta_g Psi_k m_i A(r) d / r; bodies whose beta is 0 are skipped
struct ReactGradW {
    float coef;
    static constexpr bool kByGroup = false;
    __device__ double body_coef(int) const { return coef; }
    __device__ bool term(float3 d, float r2, float mk, float4 lo, const KConst& k, float3& t) const {
        t = (mk * lo.w) * (d * grad_w_factor(sqrtf(r2), k));
        return true;
    }
    __device__ double gather(double cc, float mi) const { return -cc * static_cast<double>(mi); }
};
// A(r) of section 2.11 with cA = 0.007 / R^3.25: -4 r^2 / R + 6 r - 2 R = 2 (2 r - R)(R - r) / R, >= 0 in the band
__device__ __forceinline__ float adhesion_w(float r, float R, float cA) {
    const float t = 2.0f * (2.0f * r - R) * (R - r) / R;
    return (2.0f * r > R && r <= R) ? cA * sqrtf(sqrtf(t)) : 0.0f;
}
struct ReactAdhesion {
    const float* beta;                // the group table of sphk_adhesion
    double dtPsi;                     // dt rho0 / rho_B
    float cA;
    static constexpr bool kByGroup = true;
    __device__ double body_coef(int g) const { return dtPsi * static_cast<double>(beta[g]); }
    __device__ bool term(float3 d, float r2, float mk, float4, const KConst& k, float3& t) const {
        const float r = sqrtf(r2);
        const float a = adhesion_w(r, k.R, cA);
        if (a == 0.0f) return false;
        t = (mk * __fdividef(a, r)) * d;
        return true;
    }
    __device__ double gather(double cc, float mi) const { return cc * static_cast<double>(mi); }
};
template <class Pair>
__global__ void __launch_bounds__(SPHK_BLOCK)
k_bodies_react(const DevScene s, const float* __restrict__ massF, const float4* __restrict__ local, const int* __restrict__ decl,
               const float* __restrict__ pose, int nB, int nStatic, int reach, const Pair pair, double* __restrict__ acc) {
    if (s.pred && *s.pred == 0) return;     // a device-controlled loop has ended: its sweeps did not run
    const int kb = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (kb >= nB) return;
    const int g = static_cast<int>(body_group(local[kb]));
    if (g == 0) return;
    const float4 pk = rec_lo(s.rec + s.bOff + kb);          // {x_k, m_k}
    const float3 xk = xyz(pk);
    const float mk = pk.w;
    const int cx = cell_coord(pk.x, s.cellLength) - s.org.x, cy = cell_coord(pk.y, s.cellLength) - s.org.y,
              cz = cell_coord(pk.z, s.cellLength) - s.org.z;
    if (cx < 0 || cx >= s.cs.x || cy < 0 || cy >= s.cs.y || cz < 0 || cz >= s.cs.z) return;   // off the grid: no interaction
    const int zlo = max(cz - reach, 0), zhi = min(cz + reach, s.cs.z - 1);
    const double cc = pair.body_coef(g);
    if (Pair::kByGroup && !(cc > 0.0)) return;
    double F[3] = {0.0, 0.0, 0.0};
#pragma unroll 1
    for (int x = max(cx - reach, 0); x <= min(cx + reach, s.cs.x - 1); ++x)
#pragma unroll 1
        for (int y = max(cy - reach, 0); y <= min(cy + reach, s.cs.y - 1); ++y) {
            const int c0 = (x * s.cs.y + y) * s.cs.z;
            const int end = s.csF[c0 + zhi + 1];
            for (int j = s.csF[c0 + zlo]; j < end; ++j) {
                const float4 lo = rec_lo(s.rec + j);
                const float3 d = xyz(lo) - xk;
                const float r2 = dot3(d, d);
                if (r2 > s.k.r2cut) continue;
                float3 t;
                if (!pair.term(d, r2, mk, lo, s.k, t)) continue;
                const double f = pair.gather(cc, massF[j]);
                F[0] += f * t.x; F[1] += f * t.y; F[2] += f * t.z;
            }
        }
    const float* P = pose + 7 * (g - 1);
    const double rx = static_cast<double>(xk.x) - P[0], ry = static_cast<double>(xk.y) - P[1], rz = static_cast<double>(xk.z) - P[2];
    double* A = acc + 6 * static_cast<size_t>(decl[kb] - nStatic);
    A[0] += F[0]; A[1] += F[1]; A[2] += F[2];
    A[3] += ry * F[2] - rz * F[1]; A[4] += rz * F[0] - rx * F[2]; A[5] += rx * F[1] - ry * F[0];
}

extern "C" int sphk_bodies_react(sphk_ctx* c, const sphk_scene* s, float coef) {
    SPHK_CHECK_SCENE(c, s);
    if (!s->fluid.mass || !(coef - coef == 0.f)) return SPHK_ERR_INVALID;
    if (!c->bodies || !c->bodies->acc || !c->boundarySearched || s->boundary.n != c->nB) return SPHK_ERR_STATE;
    if (c->actCount >= 0 || c->rangeDev) return SPHK_ERR_STATE;    // slab ranks: bodies are single-context only
    const BodyState* B = c->bodies;
    // positions moved since the search (PBD corrections): a fluid particle within R of x_k may be listed two cells away
    const int reach = c->posDirty ? 2 : 1;
    k_bodies_react<<<sphk_blocks(c->nB), SPHK_BLOCK, 0, c->stream>>>(dev_scene(c, s), s->fluid.mass, B->local, B->decl, B->pose,
                                                                    c->nB, B->nStatic, reach, ReactGradW{coef}, B->acc);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_pbd_velocity_from_positions(sphk_ctx* c, const sphk_scene* s, const float* pos_last, float dt) {
    SPHK_CHECK_SCENE(c, s);
    if (!pos_last) return SPHK_ERR_INVALID;
    k_vel_from_pos<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(c->rec, pos_last, s->fluid.vel, c->nF, dt);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_pbd_xsph(sphk_ctx* c, const sphk_scene* s, float xc, float rho0) {
    SPHK_CHECK_SCENE(c, s);
    float4* tmp = c->snapB;
    OpXsph op{tmp, xc, rho0};
    const int rc = run_sweep(c, s, op);
    if (rc != SPHK_OK) return rc;
    const int b = (c->actCount < 0 || c->rangeDev) ? 0 : c->actBegin, e = (c->actCount < 0 || c->rangeDev) ? c->nF : c->actBegin + c->actCount;
    if (e > b) k_commit_vel<<<sphk_blocks(e - b), SPHK_BLOCK, 0, c->stream>>>(tmp, c->rec, s->fluid.vel, b, e, c->rangeDev);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// XSPHViscosity_CUDA (PBDSolver.cu:89-125) + computeColorGrad_CUDA (BasicSPHSolver.cu:277-330) in one pass: the colour
// gradient depends on positions and masses only, which PBD no longer changes after its projection (PBDSolver.cu:62-66).
extern "C" int sphk_fused_pbd_xsph_color_grad(sphk_ctx* c, const sphk_scene* s, float xc, float rho0, float* color_grad, float rhoB) {
    SPHK_CHECK_SCENE(c, s);
    if (!color_grad) return SPHK_ERR_INVALID;
    float4* tmp = c->snapB;
    OpPair<OpXsph, OpColorGrad> op{OpXsph{tmp, xc, rho0}, OpColorGrad{color_grad, rho0, rhoB}};
    const int rc = run_sweep(c, s, op);
    if (rc != SPHK_OK) return rc;
    const int b = (c->actCount < 0 || c->rangeDev) ? 0 : c->actBegin, e = (c->actCount < 0 || c->rangeDev) ? c->nF : c->actBegin + c->actCount;
    if (e > b) k_commit_vel<<<sphk_blocks(e - b), SPHK_BLOCK, 0, c->stream>>>(tmp, c->rec, s->fluid.vel, b, e, c->rangeDev);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_push_range(Rec rec, const float* __restrict__ vel, const float* __restrict__ scalar, const float* __restrict__ pos,
             const SkinTrack track, int begin, int count) {
    const int t = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    float d2 = 0.f;
    if (t < count) {
        const int i = begin + t;
        if (vel) rec_set_vel(rec + i, load3(vel, i));
        if (scalar) rec_set_s(rec + i, scalar[i]);
        if (pos) {
            const float3 p = load3(pos, i);
            rec_set_pos(rec + i, p);
            if (track.posBuild) d2 = skin_track(track, i, p);     // ghosts moved by their owner count like local moves do
        }
    }
    if (pos && track.posBuild) skin_track_max(track, d2);
}

extern "C" int sphk_set_active_range(sphk_ctx* c, int begin, int count) {
    if (!c) return SPHK_ERR_INVALID;
    if (count >= 0 && (begin < 0 || begin + count > c->nF)) return SPHK_ERR_INVALID;
    c->actBegin = begin; c->actCount = count;
    c->rangeDev = nullptr;
    return SPHK_OK;
}

extern "C" int sphk_set_active_range_device(sphk_ctx* c, const int* device_begin_count) {
    if (!c) return SPHK_ERR_INVALID;
    c->rangeDev = device_begin_count;
    if (device_begin_count) { c->actBegin = 0; c->actCount = -1; }
    return SPHK_OK;
}

extern "C" int sphk_push_range(sphk_ctx* c, const sphk_scene* s, int what, const float* array, int begin, int count) {
    SPHK_CHECK_SCENE(c, s);
    if (begin < 0 || count < 0 || begin + count > c->nF || what < 1 || what > 7) return SPHK_ERR_INVALID;
    if ((what & 2) && !array) return SPHK_ERR_INVALID;
    if (count == 0) return SPHK_OK;
    const bool track = (what & 4) && c->listHasSkin && c->listEpoch == c->searchEpoch;
    k_push_range<<<sphk_blocks(count), SPHK_BLOCK, 0, c->stream>>>(c->rec, (what & 1) ? s->fluid.vel : nullptr,
                                                                  (what & 2) ? array : nullptr, (what & 4) ? s->fluid.pos : nullptr,
                                                                  sphk_skin_track(c, s->radius, track), begin, count);
    c->launches++;
    if (what & 4) c->posDirty = true;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// ---- fused sweeps (same quantities, fewer passes over the neighbour lists) ------------------------------------
extern "C" int sphk_fused_density_color_grad(sphk_ctx* c, const sphk_scene* s, float* color_grad, float rho0, float rhoB) {
    SPHK_CHECK_SCENE(c, s);
    if (!color_grad || !s->fluid.density) return SPHK_ERR_INVALID;
    OpPair<OpDensity, OpColorGrad> op{OpDensity{s->fluid.density}, OpColorGrad{color_grad, rho0, rhoB}};
    return run_sweep(c, s, op);
}

extern "C" int sphk_fused_dfsph_density_alpha_color_grad(sphk_ctx* c, const sphk_scene* s, float* alpha, float* color_grad,
                                                        float rho0, float rhoB) {
    SPHK_CHECK_SCENE(c, s);
    if (!alpha || !color_grad || !s->fluid.density) return SPHK_ERR_INVALID;
    OpPair<OpDensityAlpha, OpColorGrad> op{OpDensityAlpha{s->fluid.density, alpha}, OpColorGrad{color_grad, rho0, rhoB}};
    return run_sweep(c, s, op);
}

// computeDensityAlpha_CUDA (+ computeColorGrad_CUDA) + the FIRST computeDivergenceError_CUDA of correctDivergenceError
// (DFSPHSolver.cu:341): the error sum needs the neighbours' positions and velocities only, and its epilogue needs the
// particle's own density and alpha, which the same thread has just formed -- one pass over the neighbour list less.
extern "C" int sphk_fused_dfsph_density_alpha_div_error(sphk_ctx* c, const sphk_scene* s, float* alpha, float* color_grad_or_null,
                                                       float rho0, float rhoB, float* error, float* stiff, float dt) {
    SPHK_CHECK_SCENE(c, s);
    if (!alpha || !error || !stiff || !s->fluid.density) return SPHK_ERR_INVALID;
    const OpDfsphError<false> err{c->rec, s->fluid.density, alpha, error, stiff, nullptr, dt, rho0};
    int rc;
    bool kept;
    if (color_grad_or_null) {
        OpDensityAlphaDivError<true> op{{OpPair<OpDensityAlpha, OpColorGrad>{OpDensityAlpha{s->fluid.density, alpha},
                                                                             OpColorGrad{color_grad_or_null, rho0, rhoB}}, err}};
        rc = run_sweep(c, s, op, &kept);
    } else {
        OpDensityAlphaDivError<false> op{{OpDensityAlpha{s->fluid.density, alpha}, err}};
        rc = run_sweep(c, s, op, &kept);
    }
    // never reused (it forms density and alpha), but a divergence error for the sweeps after it: the same pair terms in the same
    // order, and the epilogue takes the density and alpha it stores
    error_swept(c, kept, 1, s, alpha, error, stiff, dt, rho0);
    c->sTag = stiff;
    return rc;
}

extern "C" int sphk_fused_viscosity_surface(sphk_ctx* c, const sphk_scene* s, float* delta_v, const float* color_grad,
                                            float rho0, float visc, float dt, float kappa, float airP) {
    SPHK_CHECK_SCENE(c, s);
    if (!delta_v || !color_grad || delta_v == color_grad) return SPHK_ERR_INVALID;
    // rec.s <- |colour gradient|^2 (tagged with the array address | 1 so that repeated calls on sub-ranges of one
    // sweep -- the slab driver computes the boundary planes first -- do not redo the pre-pass)
    const void* tag = reinterpret_cast<const void*>(reinterpret_cast<uintptr_t>(color_grad) | 1u);
    if (c->sTag != tag) {
        k_s_cg2<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(color_grad, c->rec, c->nF);
        c->launches++;
        c->sTag = tag;
    }
    float4* tmp = c->snapB;
    OpViscositySurface op{tmp, s->fluid.vel, delta_v, rho0, visc, dt, kappa, airP};
    const int rc = run_sweep(c, s, op);
    if (rc != SPHK_OK) return rc;
    const int b = (c->actCount < 0 || c->rangeDev) ? 0 : c->actBegin, e = (c->actCount < 0 || c->rangeDev) ? c->nF : c->actBegin + c->actCount;
    if (e > b) k_commit_vel<<<sphk_blocks(e - b), SPHK_BLOCK, 0, c->stream>>>(tmp, c->rec, nullptr, b, e, c->rangeDev);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// ---- vorticity confinement (no reference counterpart) ---------------------------------------------------------------------
// The entries that form omega never write |omega| into rec.s (the fused viscosity + surface sweep gathers rec.s = |c|^2);
// they leave omega_norm, which sphk_vorticity_confinement mirrors into the records before it gathers it.
static int check_vorticity(const float* omega, const float* omega_norm, float rho0) {
    if (!omega || !omega_norm || omega == omega_norm || !(rho0 > 0.f)) return SPHK_ERR_INVALID;
    return SPHK_OK;
}

extern "C" int sphk_vorticity(sphk_ctx* c, const sphk_scene* s, float* omega, float* omega_norm, float rho0) {
    SPHK_CHECK_SCENE(c, s);
    if (check_vorticity(omega, omega_norm, rho0) != SPHK_OK) return SPHK_ERR_INVALID;
    if (c->sTag == omega_norm) c->sTag = nullptr;
    OpVorticity op{omega, omega_norm, 1.0f / rho0};
    return run_sweep(c, s, op);
}

extern "C" int sphk_vorticity_confinement(sphk_ctx* c, const sphk_scene* s, const float* omega, const float* omega_norm, float eps,
                                          float dt, float rho0) {
    SPHK_CHECK_SCENE(c, s);
    if (check_vorticity(omega, omega_norm, rho0) != SPHK_OK || !(eps >= 0.f) || !(dt == dt)) return SPHK_ERR_INVALID;
    ensure_scalar(c, omega_norm);
    OpVorticityConfinement op{c->rec, s->fluid.vel, omega, 1.0f / rho0, dt * eps};
    return run_sweep(c, s, op);
}

// viscosity + surface tension / air pressure + vorticity in one sweep: omega is formed from the velocities the viscosity
// term reads (the records before the commit of the new velocities)
extern "C" int sphk_fused_viscosity_surface_vorticity(sphk_ctx* c, const sphk_scene* s, float* delta_v, const float* color_grad,
                                                      float rho0, float visc, float dt, float kappa, float airP, float* omega,
                                                      float* omega_norm) {
    SPHK_CHECK_SCENE(c, s);
    if (!delta_v || !color_grad || delta_v == color_grad) return SPHK_ERR_INVALID;
    if (check_vorticity(omega, omega_norm, rho0) != SPHK_OK) return SPHK_ERR_INVALID;
    if (c->sTag == omega_norm) c->sTag = nullptr;
    const void* tag = reinterpret_cast<const void*>(reinterpret_cast<uintptr_t>(color_grad) | 1u);
    if (c->sTag != tag) {
        k_s_cg2<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(color_grad, c->rec, c->nF);
        c->launches++;
        c->sTag = tag;
    }
    float4* tmp = c->snapB;
    OpPair<OpViscositySurface, OpVorticity> op{OpViscositySurface{tmp, s->fluid.vel, delta_v, rho0, visc, dt, kappa, airP},
                                               OpVorticity{omega, omega_norm, 1.0f / rho0}};
    const int rc = run_sweep(c, s, op);
    if (rc != SPHK_OK) return rc;
    const int b = (c->actCount < 0 || c->rangeDev) ? 0 : c->actBegin, e = (c->actCount < 0 || c->rangeDev) ? c->nF : c->actBegin + c->actCount;
    if (e > b) k_commit_vel<<<sphk_blocks(e - b), SPHK_BLOCK, 0, c->stream>>>(tmp, c->rec, nullptr, b, e, c->rangeDev);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// XSPH (+ colour gradient when color_grad_or_null != NULL) + vorticity in one sweep: omega is formed from the velocities XSPH
// reads
extern "C" int sphk_fused_pbd_xsph_vorticity(sphk_ctx* c, const sphk_scene* s, float xc, float rho0, float* color_grad_or_null,
                                             float rhoB, float* omega, float* omega_norm) {
    SPHK_CHECK_SCENE(c, s);
    if (check_vorticity(omega, omega_norm, rho0) != SPHK_OK) return SPHK_ERR_INVALID;
    if (c->sTag == omega_norm) c->sTag = nullptr;
    float4* tmp = c->snapB;
    const OpVorticity vort{omega, omega_norm, 1.0f / rho0};
    int rc;
    if (color_grad_or_null) {
        OpPair<OpPair<OpXsph, OpColorGrad>, OpVorticity> op{{OpXsph{tmp, xc, rho0}, OpColorGrad{color_grad_or_null, rho0, rhoB}}, vort};
        rc = run_sweep(c, s, op);
    } else {
        OpPair<OpXsph, OpVorticity> op{OpXsph{tmp, xc, rho0}, vort};
        rc = run_sweep(c, s, op);
    }
    if (rc != SPHK_OK) return rc;
    const int b = (c->actCount < 0 || c->rangeDev) ? 0 : c->actBegin, e = (c->actCount < 0 || c->rangeDev) ? c->nF : c->actBegin + c->actCount;
    if (e > b) k_commit_vel<<<sphk_blocks(e - b), SPHK_BLOCK, 0, c->stream>>>(tmp, c->rec, s->fluid.vel, b, e, c->rangeDev);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// ---- implicit viscosity: preconditioned CG in the mass inner product, loop control on the device ------------------------------
// Workspace (caller-owned floats): ViscCg | 3 x SPHK_VISC_PARTS double partials | D[6n] | Dinv[6n] | r[3n] | z[3n] | Ap[3n].
// The iterate x lives in the API velocity array, the direction p in the velocity slots of the fluid records.  Every kernel of
// the loop returns at once when the loop has ended, so max_iter iterations are enqueued as a fixed launch sequence (a captured
// step graph replays it).  Dot products are m_i-weighted, accumulated in double, in a fixed shape (bit-reproducible).
struct ViscCg {
    int active, iters, maxIter, pad;
    double tol2, bb, rz, rr, alpha, beta;
};
#define SPHK_VISC_HEAD 64                    // floats reserved for ViscCg
#define SPHK_VISC_PARTS 1024                 // blocks of the element-wise reductions, at most
#define SPHK_VISC_RED 256                    // threads of the element-wise kernels
static_assert(sizeof(ViscCg) <= SPHK_VISC_HEAD * sizeof(float), "ViscCg exceeds its head");

// fixed-shape sum of K doubles over a block of SPHK_VISC_RED threads; thread 0 receives the totals
template <int K> __device__ __forceinline__ void visc_block_sum(double (&v)[K]) {
    __shared__ double sm[K][SPHK_VISC_RED / 32];
    for (int k = 0; k < K; ++k) {
        double t = v[k];
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if ((threadIdx.x & 31) == 0) sm[k][threadIdx.x >> 5] = t;
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int k = 0; k < K; ++k) {
            double t = 0.0;
            for (int w = 0; w < SPHK_VISC_RED / 32; ++w) t += sm[k][w];
            v[k] = t;
        }
}
template <int K> __device__ __forceinline__ void visc_store_partials(double (&v)[K], double* __restrict__ part) {
    visc_block_sum(v);
    if (threadIdx.x == 0)
        for (int k = 0; k < K; ++k) part[k * SPHK_VISC_PARTS + blockIdx.x] = v[k];
}
// one block: the K totals of m partials
template <int K> __device__ __forceinline__ void visc_sum_partials(const double* __restrict__ part, int m, double (&v)[K]) {
    for (int k = 0; k < K; ++k) {
        v[k] = 0.0;
        for (int b = threadIdx.x; b < m; b += SPHK_VISC_RED) v[k] += part[k * SPHK_VISC_PARTS + b];
    }
    visc_block_sum(v);
}
__device__ __forceinline__ double mdot(float m, float3 a, float3 b) {
    return static_cast<double>(m) * (static_cast<double>(a.x) * b.x + static_cast<double>(a.y) * b.y + static_cast<double>(a.z) * b.z);
}

// r = b - A x0 (b arrives in r, A x0 in Ap; x0 = v* = the records' velocity, copied to the API array), z = Dinv r, p = z;
// partials {<b,b>, <r,z>, <r,r>}
__global__ void __launch_bounds__(SPHK_VISC_RED)
k_visc_init(Rec rec, float* __restrict__ vel, float* __restrict__ r, const float* __restrict__ Ap, const float* __restrict__ Dinv,
            float* __restrict__ z, int n, double* __restrict__ part) {
    double acc[3] = {0.0, 0.0, 0.0};
    for (int i = blockIdx.x * SPHK_VISC_RED + threadIdx.x; i < n; i += gridDim.x * SPHK_VISC_RED) {
        const float4 hi = rec_hi(rec + i);
        store3(vel, i, xyz(hi));
        const float3 b = load3(r, i), ri = b - load3(Ap, i), zi = sym_apply(Dinv, i, ri);
        store3(r, i, ri); store3(z, i, zi);
        rec_set_vel(rec + i, zi);
        acc[0] += mdot(hi.w, b, b); acc[1] += mdot(hi.w, ri, zi); acc[2] += mdot(hi.w, ri, ri);
    }
    visc_store_partials(acc, part);
}
// the loop test before the first iteration: converged (|r|_M <= tol |b|_M, a fluid at rest included) or <r,z>_M = 0
__global__ void __launch_bounds__(SPHK_VISC_RED) k_visc_init_finish(ViscCg* st, const double* __restrict__ part, int m, double tol2,
                                                                     int maxIter) {
    double v[3];
    visc_sum_partials(part, m, v);
    if (threadIdx.x != 0) return;
    st->tol2 = tol2; st->maxIter = maxIter; st->iters = 0;
    st->bb = v[0]; st->rz = v[1]; st->rr = v[2]; st->alpha = 0.0; st->beta = 0.0;
    st->active = (v[2] <= tol2 * v[0] || v[1] == 0.0) ? 0 : 1;
}
// partials of <p, Ap>
__global__ void __launch_bounds__(SPHK_VISC_RED)
k_visc_alpha_partial(const ViscCg* st, Rec rec, const float* __restrict__ Ap, int n, double* __restrict__ part) {
    if (!st->active) return;
    double acc[1] = {0.0};
    for (int i = blockIdx.x * SPHK_VISC_RED + threadIdx.x; i < n; i += gridDim.x * SPHK_VISC_RED) {
        const float4 hi = rec_hi(rec + i);
        acc[0] += mdot(hi.w, xyz(hi), load3(Ap, i));
    }
    visc_store_partials(acc, part);
}
// alpha = <r,z> / <p,Ap> (a non-positive <p,Ap> -- breakdown -- ends the loop)
__global__ void __launch_bounds__(SPHK_VISC_RED) k_visc_alpha_finish(ViscCg* st, const double* __restrict__ part, int m) {
    if (!st->active) return;
    double v[1];
    visc_sum_partials(part, m, v);
    if (threadIdx.x != 0) return;
    if (!(v[0] > 0.0)) { st->active = 0; return; }
    st->alpha = st->rz / v[0];
}
// x += alpha p, r -= alpha Ap, z = Dinv r; partials {<r,z>, <r,r>}
__global__ void __launch_bounds__(SPHK_VISC_RED)
k_visc_update(const ViscCg* st, Rec rec, float* __restrict__ vel, float* __restrict__ r, const float* __restrict__ Ap,
              const float* __restrict__ Dinv, float* __restrict__ z, int n, double* __restrict__ part) {
    if (!st->active) return;
    const float a = static_cast<float>(st->alpha);
    double acc[2] = {0.0, 0.0};
    for (int i = blockIdx.x * SPHK_VISC_RED + threadIdx.x; i < n; i += gridDim.x * SPHK_VISC_RED) {
        const float4 hi = rec_hi(rec + i);
        store3(vel, i, load3(vel, i) + a * xyz(hi));
        const float3 ri = load3(r, i) - a * load3(Ap, i), zi = sym_apply(Dinv, i, ri);
        store3(r, i, ri); store3(z, i, zi);
        acc[0] += mdot(hi.w, ri, zi); acc[1] += mdot(hi.w, ri, ri);
    }
    visc_store_partials(acc, part);
}
// ++iters; the loop ends when |r|_M <= tol |b|_M, <r,z>_M = 0 or iters = max_iter; else beta = <r,z>_new / <r,z>
__global__ void __launch_bounds__(SPHK_VISC_RED) k_visc_beta_finish(ViscCg* st, const double* __restrict__ part, int m) {
    if (!st->active) return;
    double v[2];
    visc_sum_partials(part, m, v);
    if (threadIdx.x != 0) return;
    const int it = st->iters + 1;
    st->iters = it;
    st->rr = v[1];
    if (v[1] <= st->tol2 * st->bb || v[0] == 0.0 || it >= st->maxIter) { st->active = 0; return; }
    st->beta = v[0] / st->rz;
    st->rz = v[0];
}
// p = z + beta p
__global__ void __launch_bounds__(SPHK_VISC_RED) k_visc_direction(const ViscCg* st, Rec rec, const float* __restrict__ z, int n) {
    if (!st->active) return;
    const float beta = static_cast<float>(st->beta);
    for (int i = blockIdx.x * SPHK_VISC_RED + threadIdx.x; i < n; i += gridDim.x * SPHK_VISC_RED)
        rec_set_vel(rec + i, load3(z, i) + beta * xyz(rec_hi(rec + i)));
}
// the solve's outcome into the context's own memory (the workspace is the caller's and may be gone when the stats are read)
__global__ void k_visc_report(const ViscCg* st, float* out) {
    out[0] = __int_as_float(st->iters);
    out[1] = st->bb > 0.0 ? static_cast<float>(sqrt(st->rr / st->bb)) : 0.0f;
}
// the records' velocity slots <- a float3 array (a test's direction p; the solution at the end of the solve)
__global__ void __launch_bounds__(SPHK_BLOCK) k_visc_set_rec_vel(Rec rec, const float* __restrict__ v, int n) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i < n) rec_set_vel(rec + i, load3(v, i));
}

static int visc_blocks(int n) {
    const int b = (n + SPHK_VISC_RED * 8 - 1) / (SPHK_VISC_RED * 8);
    return b < 1 ? 1 : (b > SPHK_VISC_PARTS ? SPHK_VISC_PARTS : b);
}
static bool finite_nonneg(float x) { return x >= 0.f && x - x == 0.f; }
static int check_visc(const sphk_ctx* c, float nu, float dt, float rho0) {
    if (!finite_nonneg(nu) || !finite_nonneg(dt) || !(rho0 > 0.f)) return SPHK_ERR_INVALID;
    if (c->actCount >= 0 || c->rangeDev) return SPHK_ERR_STATE;      // slab ranks: the solve needs global dot products
    return SPHK_OK;
}
static bool aliases(const void* a, const sphk_scene* s) {
    return a == s->fluid.pos || a == s->fluid.vel || a == s->fluid.mass || a == s->fluid.density || a == s->fluid.pressure;
}

extern "C" long long sphk_implicit_viscosity_work_floats(int n) {
    if (n < 0) return -1;
    return SPHK_VISC_HEAD + 2LL * 3 * SPHK_VISC_PARTS + 21LL * n;
}

struct ViscWork {
    ViscCg* st; double* part; float *D, *Dinv, *r, *z, *Ap;
};
static ViscWork visc_work(float* work, int n) {
    ViscWork w;
    w.st = reinterpret_cast<ViscCg*>(work);
    w.part = reinterpret_cast<double*>(work + SPHK_VISC_HEAD);
    w.D = work + SPHK_VISC_HEAD + 2 * 3 * SPHK_VISC_PARTS;
    w.Dinv = w.D + 6LL * n; w.r = w.Dinv + 6LL * n; w.z = w.r + 3LL * n; w.Ap = w.z + 3LL * n;
    return w;
}

// The solve after its setup sweep (b in r, D and Dinv formed) with the matvec sweep `mv`: r = b - A v*, then max_iter PCG
// iterations under the device-side loop test; the outcome {iterations, |r|_M / |b|_M} goes to `report` (context memory).
template <class Mv>
static int visc_pcg(sphk_ctx* c, const sphk_scene* s, const ViscWork& w, const Mv& mv, float tol, int max_iter, float* report) {
    const int n = c->nF;
    float* vel = s->fluid.vel;
    int rc = run_sweep(c, s, mv);                                                                // A v*
    if (rc != SPHK_OK) return rc;
    const int m = visc_blocks(n);
    k_visc_init<<<m, SPHK_VISC_RED, 0, c->stream>>>(c->rec, vel, w.r, w.Ap, w.Dinv, w.z, n, w.part);
    k_visc_init_finish<<<1, SPHK_VISC_RED, 0, c->stream>>>(w.st, w.part, m, static_cast<double>(tol) * tol, max_iter);
    c->launches += 2;
    const int* outer = c->pred;
    c->pred = &w.st->active;
    for (int k = 0; k < max_iter && rc == SPHK_OK; ++k) {
        rc = run_sweep(c, s, mv);
        k_visc_alpha_partial<<<m, SPHK_VISC_RED, 0, c->stream>>>(w.st, c->rec, w.Ap, n, w.part);
        k_visc_alpha_finish<<<1, SPHK_VISC_RED, 0, c->stream>>>(w.st, w.part, m);
        k_visc_update<<<m, SPHK_VISC_RED, 0, c->stream>>>(w.st, c->rec, vel, w.r, w.Ap, w.Dinv, w.z, n, w.part);
        k_visc_beta_finish<<<1, SPHK_VISC_RED, 0, c->stream>>>(w.st, w.part, m);
        k_visc_direction<<<m, SPHK_VISC_RED, 0, c->stream>>>(w.st, c->rec, w.z, n);
        c->launches += 5;
    }
    c->pred = outer;
    if (n > 0) { k_visc_set_rec_vel<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(c->rec, vel, n); c->launches++; }   // records <- x
    k_visc_report<<<1, 1, 0, c->stream>>>(w.st, report);
    c->launches++;
    if (rc != SPHK_OK) return rc;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_implicit_viscosity(sphk_ctx* c, const sphk_scene* s, float* work, float nu, float nu_boundary, float dt, float rho0,
                                       float rho_boundary, float tol, int max_iter) {
    SPHK_CHECK_SCENE(c, s);
    if (!work || aliases(work, s) || !finite_nonneg(nu_boundary) || !(rho_boundary > 0.f) || !(tol > 0.f) || max_iter < 1 ||
        max_iter > SPHK_IMPLICIT_VISCOSITY_MAX_ITER)
        return SPHK_ERR_INVALID;
    const int rc0 = check_visc(c, nu, dt, rho0);
    if (rc0 != SPHK_OK) return rc0;
    // the viscous force on a dynamic body is not part of its reaction (sphk_bodies_react): the momentum would not balance
    if (nu_boundary > 0.f && c->bodies && c->bodies->acc) return SPHK_ERR_STATE;
    const ViscWork w = visc_work(work, c->nF);
    const float nuRho = nu / rho0, nuBRho = nu_boundary / rho_boundary;
    const int rc = run_sweep(c, s, OpViscImplicitSetup{w.D, w.Dinv, w.r, nuRho, nuBRho, dt});          // b -> r
    if (rc != SPHK_OK) return rc;
    return visc_pcg(c, s, w, OpViscImplicitMatvec{w.D, w.Ap, nuRho, dt}, tol, max_iter, c->viscStats);
}

extern "C" int sphk_implicit_viscosity_stats(sphk_ctx* c, int* iterations, float* rel_residual) {
    if (!c || !iterations) return SPHK_ERR_INVALID;
    float h[2];
    SPHK_CUDA_TRY(cudaMemcpyAsync(h, c->viscStats, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    memcpy(iterations, &h[0], sizeof(int));
    if (rel_residual) *rel_residual = h[1];
    return SPHK_OK;
}

extern "C" int sphk_visc_implicit_setup(sphk_ctx* c, const sphk_scene* s, float* d_out, float* b_out, float nu, float nu_boundary,
                                        float dt, float rho0, float rho_boundary) {
    SPHK_CHECK_SCENE(c, s);
    if (!d_out || !b_out || d_out == b_out || aliases(d_out, s) || aliases(b_out, s) || !finite_nonneg(nu_boundary) ||
        !(rho_boundary > 0.f))
        return SPHK_ERR_INVALID;
    const int rc = check_visc(c, nu, dt, rho0);
    if (rc != SPHK_OK) return rc;
    return run_sweep(c, s, OpViscImplicitSetup{d_out, nullptr, b_out, nu / rho0, nu_boundary / rho_boundary, dt});
}

extern "C" int sphk_visc_implicit_matvec(sphk_ctx* c, const sphk_scene* s, const float* d_in, const float* p_in, float* ap_out,
                                         float nu, float dt, float rho0) {
    SPHK_CHECK_SCENE(c, s);
    if (!d_in || !p_in || !ap_out || d_in == p_in || ap_out == d_in || ap_out == p_in || aliases(ap_out, s)) return SPHK_ERR_INVALID;
    const int rc0 = check_visc(c, nu, dt, rho0);
    if (rc0 != SPHK_OK) return rc0;
    const int n = c->nF;
    if (n > 0) k_visc_set_rec_vel<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(c->rec, p_in, n);
    const int rc = run_sweep(c, s, OpViscImplicitMatvec{d_in, ap_out, nu / rho0, dt});
    if (n > 0) k_visc_set_rec_vel<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(c->rec, s->fluid.vel, n);   // records <- API velocities
    if (n > 0) c->launches += 2;
    if (rc != SPHK_OK) return rc;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// ---- non-Newtonian viscosity (DESIGN.md section 2.9) ------------------------------------------------------------------------
// rec.s <- nu_i / rho0 (correctly rounded: with a uniform nu it is the constant-nu solve's nu / rho0, bit for bit).  rec.s then
// mirrors no caller array: sTag = nullptr, so every later sweep that gathers a scalar re-mirrors or rewrites it first.
__global__ void __launch_bounds__(SPHK_BLOCK) k_rheo_mirror(const float* __restrict__ nu, Rec rec, int n, float rho0) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i < n) rec_set_s(rec + i, __fdiv_rn(nu[i], rho0));
}
__global__ void k_rheo_stats_reset(unsigned int* st) {
    st[2] = 0u; st[3] = 0x7f800000u; st[4] = 0u; st[5] = 0u;      // (min nu starts at +inf)
}
__global__ void __launch_bounds__(SPHK_BLOCK) k_rheo_eval(sphk_rheology rh, const float* __restrict__ g, float* __restrict__ nu, int n) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    bool atMax;
    nu[i] = d2f_rn(rheo_nu(rh, f2d(g[i]), &atMax));
}

static bool finite_f(float x) { return x - x == 0.f; }
static int check_rheology(const sphk_rheology* r) {
    if (!r) return SPHK_ERR_INVALID;
    for (int k = 0; k < 6; ++k) if (!finite_f(r->params[k])) return SPHK_ERR_INVALID;
    if (!finite_nonneg(r->nu_min) || !finite_nonneg(r->nu_max) || r->nu_min > r->nu_max) return SPHK_ERR_INVALID;
    const float* p = r->params;
    if (r->model == SPHK_RHEOLOGY_CROSS) {                  // nu0, nu_inf, lambda >= 0, m > 0
        if (!(p[0] >= 0.f && p[1] >= 0.f && p[2] >= 0.f && p[3] > 0.f)) return SPHK_ERR_INVALID;
    } else if (r->model == SPHK_RHEOLOGY_HERSCHEL_BULKLEY) { // K >= 0, n > 0, tau_y >= 0, m_reg >= 0
        if (!(p[0] >= 0.f && p[1] > 0.f && p[2] >= 0.f && p[3] >= 0.f)) return SPHK_ERR_INVALID;
    } else {
        return SPHK_ERR_INVALID;
    }
    return SPHK_OK;
}
static unsigned int* rheo_stats(sphk_ctx* c) { return reinterpret_cast<unsigned int*>(c->rheoStats); }

// the shear sweep: statistics reset, then gamma_dot and nu (+ gradient and flag) of every particle
static int shear_sweep(sphk_ctx* c, const sphk_scene* s, float* gamma, float* nu, float* grad, int* flag, const sphk_rheology& rh,
                       float beta, float rho0, float rho_boundary) {
    k_rheo_stats_reset<<<1, 1, 0, c->stream>>>(rheo_stats(c));
    c->launches++;
    return run_sweep(c, s, OpShearRate{gamma, nu, grad, flag, rheo_stats(c), rh, 1.0f / rho0, 1.0f / rho_boundary, beta > 0.f});
}
static void rheo_mirror(sphk_ctx* c, const float* nu, float rho0) {
    if (c->nF > 0) { k_rheo_mirror<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(nu, c->rec, c->nF, rho0); c->launches++; }
    c->sTag = nullptr;
}
static int check_field_common(sphk_ctx* c, float beta, float dt, float rho0, float rho_boundary) {
    if (!finite_nonneg(beta) || !(rho_boundary > 0.f)) return SPHK_ERR_INVALID;
    const int rc = check_visc(c, 0.0f, dt, rho0);
    if (rc != SPHK_OK) return rc;
    // the viscous force on a dynamic body is not part of its reaction (sphk_bodies_react): the momentum would not balance
    if (beta > 0.f && c->bodies && c->bodies->acc) return SPHK_ERR_STATE;
    return SPHK_OK;
}

extern "C" long long sphk_rheology_work_floats(int n) {
    if (n < 0) return -1;
    return sphk_implicit_viscosity_work_floats(n) + n;          // + gamma_dot
}

extern "C" int sphk_non_newtonian_viscosity(sphk_ctx* c, const sphk_scene* s, float* work, float* nu_field, const sphk_rheology* rheology,
                                            float beta, float dt, float rho0, float rho_boundary, float tol, int max_iter) {
    SPHK_CHECK_SCENE(c, s);
    if (!work || !nu_field || work == nu_field || aliases(work, s) || aliases(nu_field, s) || !(tol > 0.f) || max_iter < 1 ||
        max_iter > SPHK_IMPLICIT_VISCOSITY_MAX_ITER || check_rheology(rheology) != SPHK_OK)
        return SPHK_ERR_INVALID;
    const int rc0 = check_field_common(c, beta, dt, rho0, rho_boundary);
    if (rc0 != SPHK_OK) return rc0;
    const int n = c->nF;
    const ViscWork w = visc_work(work, n);
    float* gamma = work + sphk_implicit_viscosity_work_floats(n);
    int rc = shear_sweep(c, s, gamma, nu_field, nullptr, nullptr, *rheology, beta, rho0, rho_boundary);   // from v*
    if (rc != SPHK_OK) return rc;
    rheo_mirror(c, nu_field, rho0);
    rc = run_sweep(c, s, OpViscImplicitSetupField{OpViscImplicitSetup{w.D, w.Dinv, w.r, 0.f, 0.f, dt}, nu_field, beta, rho_boundary});
    if (rc != SPHK_OK) return rc;
    return visc_pcg(c, s, w, OpViscImplicitMatvecField{w.D, w.Ap, dt}, tol, max_iter, c->rheoStats);
}

extern "C" int sphk_non_newtonian_stats(sphk_ctx* c, int* iterations, float* rel_residual, float* gamma_max, float* nu_min,
                                        float* nu_max, int* n_at_max) {
    if (!c) return SPHK_ERR_INVALID;
    unsigned int h[SPHK_RHEO_STATS];
    SPHK_CUDA_TRY(cudaMemcpyAsync(h, c->rheoStats, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    float f[SPHK_RHEO_STATS];
    memcpy(f, h, sizeof(h));
    if (iterations) *iterations = static_cast<int>(h[0]);
    if (rel_residual) *rel_residual = f[1];
    if (gamma_max) *gamma_max = f[2];
    if (nu_min) *nu_min = h[3] == 0x7f800000u ? 0.0f : f[3];     // (no fluid particle: 0)
    if (nu_max) *nu_max = f[4];
    if (n_at_max) *n_at_max = static_cast<int>(h[5]);
    return SPHK_OK;
}

extern "C" int sphk_shear_rate(sphk_ctx* c, const sphk_scene* s, float* gamma_out, float* nu_out, float* grad_out_or_null,
                               int* flag_out_or_null, const sphk_rheology* rheology, float beta, float rho0, float rho_boundary) {
    SPHK_CHECK_SCENE(c, s);
    if (!gamma_out || !nu_out || gamma_out == nu_out || aliases(gamma_out, s) || aliases(nu_out, s) ||
        (grad_out_or_null && (aliases(grad_out_or_null, s) || grad_out_or_null == gamma_out || grad_out_or_null == nu_out)) ||
        check_rheology(rheology) != SPHK_OK)
        return SPHK_ERR_INVALID;
    const int rc = check_field_common(c, beta, 0.0f, rho0, rho_boundary);
    if (rc != SPHK_OK) return rc;
    if (c->sTag == nu_out) c->sTag = nullptr;
    return shear_sweep(c, s, gamma_out, nu_out, grad_out_or_null, flag_out_or_null, *rheology, beta, rho0, rho_boundary);
}

extern "C" int sphk_rheology_eval(sphk_ctx* c, const sphk_rheology* rheology, const float* gamma, float* nu_out, int n) {
    if (!c || !gamma || !nu_out || gamma == nu_out || n < 0 || check_rheology(rheology) != SPHK_OK) return SPHK_ERR_INVALID;
    if (n == 0) return SPHK_OK;
    k_rheo_eval<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(*rheology, gamma, nu_out, n);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_visc_field_setup(sphk_ctx* c, const sphk_scene* s, float* d_out, float* b_out, const float* nu, float beta,
                                     float dt, float rho0, float rho_boundary) {
    SPHK_CHECK_SCENE(c, s);
    if (!d_out || !b_out || !nu || d_out == b_out || nu == d_out || nu == b_out || aliases(d_out, s) || aliases(b_out, s))
        return SPHK_ERR_INVALID;
    const int rc = check_field_common(c, beta, dt, rho0, rho_boundary);
    if (rc != SPHK_OK) return rc;
    rheo_mirror(c, nu, rho0);
    return run_sweep(c, s, OpViscImplicitSetupField{OpViscImplicitSetup{d_out, nullptr, b_out, 0.f, 0.f, dt}, nu, beta, rho_boundary});
}

extern "C" int sphk_visc_field_matvec(sphk_ctx* c, const sphk_scene* s, const float* d_in, const float* p_in, float* ap_out,
                                      const float* nu, float dt, float rho0) {
    SPHK_CHECK_SCENE(c, s);
    if (!d_in || !p_in || !ap_out || !nu || d_in == p_in || ap_out == d_in || ap_out == p_in || ap_out == nu || aliases(ap_out, s))
        return SPHK_ERR_INVALID;
    const int rc0 = check_field_common(c, 0.0f, dt, rho0, 1.0f);
    if (rc0 != SPHK_OK) return rc0;
    const int n = c->nF;
    rheo_mirror(c, nu, rho0);
    if (n > 0) k_visc_set_rec_vel<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(c->rec, p_in, n);
    const int rc = run_sweep(c, s, OpViscImplicitMatvecField{d_in, ap_out, dt});
    if (n > 0) k_visc_set_rec_vel<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(c->rec, s->fluid.vel, n);   // records <- API velocities
    if (n > 0) c->launches += 2;
    if (rc != SPHK_OK) return rc;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// ---- heat transfer (DESIGN.md section 2.10) ----------------------------------------------------------------------------------
// the step's group table {T_g, h_g} (groups past n_groups adiabatic) from the setting passed by value, and the statistics reset
__global__ void k_heat_begin(sphk_thermal th, float2* __restrict__ groups, unsigned int* __restrict__ stats) {
    const int g = threadIdx.x;
    if (g < SPHK_THERMAL_GROUPS) groups[g] = g < th.n_groups ? make_float2(th.groups[g].t, th.groups[g].h) : make_float2(0.f, 0.f);
    if (g == 0) { stats[0] = 0u; stats[1] = 0u; }
}
// T += dt_k dT/dt (also into rec.s, which keeps mirroring T); on the last substep v += -beta (T - T_ref) G dt on the API array and the
// records.  A particle at T_ref gets no velocity write at all, so its bits stay those of a step without the stage.
__global__ void __launch_bounds__(SPHK_BLOCK) k_heat_commit(float* __restrict__ T, const float* __restrict__ dTdt, Rec rec,
                                                            float* __restrict__ vel, int n, float dtSub, bool last, float beta,
                                                            float tRef, float3 Gdt) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float t = T[i] + dtSub * dTdt[i];
    T[i] = t;
    rec_set_s(rec + i, t);
    const float dT = t - tRef;
    if (last && dT != 0.f && beta != 0.f) {
        const float3 v = load3(vel, i) - (beta * dT) * Gdt;
        store3(vel, i, v);
        rec_set_vel(rec + i, v);
    }
}
// min T, max T and sum m T (double) in a fixed shape: clamp(ceil(n / 2048), 1, 1024) blocks of 256 threads, each thread's
// grid-stride run, a warp butterfly, the 8 warp values in lane order; then one block over the partials in the same shape.
#define SPHK_HEAT_RED 256
__device__ __forceinline__ void heat_fold(double& lo, double& hi, double& sum) {
    for (int o = 16; o > 0; o >>= 1) {
        lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
    }
}
__device__ __forceinline__ void heat_block(double lo, double hi, double sum, double* out) {
    __shared__ double sh[3][SPHK_HEAT_RED / 32];
    heat_fold(lo, hi, sum);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { sh[0][w] = lo; sh[1][w] = hi; sh[2][w] = sum; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < SPHK_HEAT_RED / 32; ++k) { lo = fmin(lo, sh[0][k]); hi = fmax(hi, sh[1][k]); sum += sh[2][k]; }
        out[0] = lo; out[1] = hi; out[2] = sum;
    }
}
__global__ void __launch_bounds__(SPHK_HEAT_RED) k_heat_partial(const float* __restrict__ T, const float* __restrict__ m, int n,
                                                                double* __restrict__ part) {
    double lo = CUDART_INF, hi = -CUDART_INF, sum = 0.0;
    for (int i = blockIdx.x * SPHK_HEAT_RED + threadIdx.x; i < n; i += gridDim.x * SPHK_HEAT_RED) {
        const double t = f2d(T[i]);
        lo = fmin(lo, t); hi = fmax(hi, t); sum += f2d(m[i]) * t;
    }
    heat_block(lo, hi, sum, part + 3 * blockIdx.x);
}
__global__ void __launch_bounds__(SPHK_HEAT_RED) k_heat_finish(const double* __restrict__ part, int m, double* __restrict__ out) {
    double lo = CUDART_INF, hi = -CUDART_INF, sum = 0.0;
    for (int k = threadIdx.x; k < m; k += SPHK_HEAT_RED) { lo = fmin(lo, part[3 * k]); hi = fmax(hi, part[3 * k + 1]); sum += part[3 * k + 2]; }
    heat_block(lo, hi, sum, out);
}
// nu(T) = clamp(nu_ref exp(-e (T - t_ref)), nu_min, nu_max) in double, rounded once (a NaN lands on nu_max)
__device__ __forceinline__ float thermal_nu(const sphk_viscosity_law& v, float t) {
    const double raw = static_cast<double>(v.nu_ref) * exp(-static_cast<double>(v.e) * (f2d(t) - static_cast<double>(v.t_ref)));
    return d2f_rn(!(raw < static_cast<double>(v.nu_max)) ? static_cast<double>(v.nu_max) : fmax(raw, static_cast<double>(v.nu_min)));
}
__global__ void __launch_bounds__(SPHK_BLOCK) k_thermal_nu(sphk_viscosity_law v, const float* __restrict__ T, float* __restrict__ nu,
                                                           int n) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i < n) nu[i] = thermal_nu(v, T[i]);
}

static int check_thermal(const sphk_ctx* c, const sphk_thermal* th) {
    if (!th || !finite_nonneg(th->alpha) || !finite_f(th->beta) || !finite_f(th->t_ref) || th->n_groups < 0 ||
        th->n_groups > SPHK_THERMAL_GROUPS)
        return SPHK_ERR_INVALID;
    for (int g = 0; g < th->n_groups; ++g)
        if (!finite_f(th->groups[g].t) || !finite_nonneg(th->groups[g].h)) return SPHK_ERR_INVALID;
    if (c && th->n_groups > 1 + (c->bodies ? c->bodies->nBodies : 0)) return SPHK_ERR_STATE;
    return SPHK_OK;
}

extern "C" int sphk_heat_substeps(const sphk_thermal* th, float radius, float dt, int* substeps) {
    if (!substeps || check_thermal(nullptr, th) != SPHK_OK || !(radius > 0.f) || !finite_nonneg(dt) || radius - radius != 0.f)
        return SPHK_ERR_INVALID;
    double hMax = 0.0;
    for (int g = 0; g < th->n_groups; ++g) hMax = std::max(hMax, static_cast<double>(th->groups[g].h));
    const double R = radius;
    const double k = std::ceil(static_cast<double>(dt) * SPHK_HEAT_COP * th->alpha * (1.0 + hMax) / (R * R));
    if (!(k <= 65536.0)) return SPHK_ERR_INVALID;
    *substeps = std::max(1, static_cast<int>(k));
    return SPHK_OK;
}

// table + statistics reset (substep 0 only), mirror, conduction sweep
static int heat_sweep(sphk_ctx* c, const sphk_scene* s, const sphk_thermal& th, const float* T, float* dTdt, float dtSub, float rho0,
                      float rhoB, bool begin) {
    if (begin) { k_heat_begin<<<1, 96, 0, c->stream>>>(th, c->heatGroups, c->heatStats); c->launches++; }
    ensure_scalar(c, T);
    // with bodies every boundary particle's group is read (body b without an entry is adiabatic: the table holds {0, 0} there)
    const float t0 = th.n_groups > 0 ? th.groups[0].t : 0.f, h0 = th.n_groups > 0 ? th.groups[0].h : 0.f;
    return run_sweep(c, s, OpHeatConduction{dTdt, c->heatStats, c->bodies ? c->bodies->local : nullptr, c->heatGroups, th.alpha / rho0,
                                            th.alpha / rhoB, t0, h0, dtSub, c->nB});
}
static int check_heat_call(sphk_ctx* c, const sphk_scene* s, const sphk_thermal* th, const float* T, const float* out, float rho0,
                           float rhoB) {
    if (!T || !out || T == out || aliases(T, s) || aliases(out, s) || !(rho0 > 0.f) || !(rhoB > 0.f)) return SPHK_ERR_INVALID;
    const int rc = check_thermal(c, th);
    if (rc != SPHK_OK) return rc;
    if (c->actCount >= 0 || c->rangeDev) return SPHK_ERR_STATE;      // slab ranks: ghosts would need their temperatures
    return SPHK_OK;
}

extern "C" int sphk_heat_step(sphk_ctx* c, const sphk_scene* s, const sphk_thermal* th, float* T, float* work, float dt, int k,
                              int substeps, float rho0, float rho_boundary, const float* gravity) {
    SPHK_CHECK_SCENE(c, s);
    if (!gravity || !finite_nonneg(dt) || substeps < 1 || k < 0 || k >= substeps) return SPHK_ERR_INVALID;
    const int rc0 = check_heat_call(c, s, th, T, work, rho0, rho_boundary);
    if (rc0 != SPHK_OK) return rc0;
    const float dtSub = dt / static_cast<float>(substeps);
    const int rc = heat_sweep(c, s, *th, T, work, dtSub, rho0, rho_boundary, k == 0);
    if (rc != SPHK_OK) return rc;
    const int n = c->nF;
    if (n > 0) {
        const float3 Gdt = make_float3(gravity[0] * dt, gravity[1] * dt, gravity[2] * dt);
        k_heat_commit<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(T, work, c->rec, s->fluid.vel, n, dtSub, k == substeps - 1, th->beta,
                                                                  th->t_ref, Gdt);
        c->launches++;
    }
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_heat_conduction(sphk_ctx* c, const sphk_scene* s, const sphk_thermal* th, const float* T, float* dtdt_out,
                                    float dt_sub, float rho0, float rho_boundary) {
    SPHK_CHECK_SCENE(c, s);
    if (!finite_nonneg(dt_sub)) return SPHK_ERR_INVALID;
    const int rc = check_heat_call(c, s, th, T, dtdt_out, rho0, rho_boundary);
    if (rc != SPHK_OK) return rc;
    if (c->sTag == dtdt_out) c->sTag = nullptr;
    return heat_sweep(c, s, *th, T, dtdt_out, dt_sub, rho0, rho_boundary, true);
}

extern "C" int sphk_heat_stats(sphk_ctx* c, const float* T, const float* mass, int n, float* max_courant, int* violators, float* t_min,
                               float* t_max, double* heat) {
    if (!c || n < 0 || (n > 0 && (!T || !mass))) return SPHK_ERR_INVALID;
    const bool reduce = T && mass && n > 0;
    if (reduce) {
        const int m = std::min(std::max((n + 2047) / 2048, 1), 1024);
        k_heat_partial<<<m, SPHK_HEAT_RED, 0, c->stream>>>(T, mass, n, c->heatRed);
        k_heat_finish<<<1, SPHK_HEAT_RED, 0, c->stream>>>(c->heatRed, m, c->heatRed + 3 * 1024);
        c->launches += 2;
        SPHK_CUDA_TRY(cudaGetLastError());
    }
    unsigned int st[2];
    double red[3] = {0.0, 0.0, 0.0};
    SPHK_CUDA_TRY(cudaMemcpyAsync(st, c->heatStats, sizeof(st), cudaMemcpyDeviceToHost, c->stream));
    if (reduce) SPHK_CUDA_TRY(cudaMemcpyAsync(red, c->heatRed + 3 * 1024, sizeof(red), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    float cour;
    memcpy(&cour, &st[0], sizeof(cour));
    if (max_courant) *max_courant = cour;
    if (violators) *violators = static_cast<int>(st[1]);
    if (t_min) *t_min = static_cast<float>(red[0]);
    if (t_max) *t_max = static_cast<float>(red[1]);
    if (heat) *heat = red[2];
    return SPHK_OK;
}

static int check_thermal_viscosity(const sphk_viscosity_law* v) {
    if (!v || !finite_nonneg(v->nu_ref) || !finite_f(v->e) || !finite_f(v->t_ref) || !finite_nonneg(v->nu_min) ||
        !finite_nonneg(v->nu_max) || v->nu_min > v->nu_max)
        return SPHK_ERR_INVALID;
    return SPHK_OK;
}

extern "C" int sphk_thermal_viscosity(sphk_ctx* c, const sphk_scene* s, float* work, float* nu_field, const float* T,
                                      const sphk_viscosity_law* law, float beta, float dt, float rho0, float rho_boundary, float tol,
                                      int max_iter) {
    SPHK_CHECK_SCENE(c, s);
    if (!work || !nu_field || !T || work == nu_field || T == nu_field || T == work || aliases(work, s) || aliases(nu_field, s) ||
        !(tol > 0.f) || max_iter < 1 || max_iter > SPHK_IMPLICIT_VISCOSITY_MAX_ITER || check_thermal_viscosity(law) != SPHK_OK)
        return SPHK_ERR_INVALID;
    const int rc0 = check_field_common(c, beta, dt, rho0, rho_boundary);
    if (rc0 != SPHK_OK) return rc0;
    const int n = c->nF;
    if (c->sTag == nu_field) c->sTag = nullptr;
    if (n > 0) { k_thermal_nu<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(*law, T, nu_field, n); c->launches++; }
    const ViscWork w = visc_work(work, n);
    rheo_mirror(c, nu_field, rho0);
    const int rc = run_sweep(c, s, OpViscImplicitSetupField{OpViscImplicitSetup{w.D, w.Dinv, w.r, 0.f, 0.f, dt}, nu_field, beta, rho_boundary});
    if (rc != SPHK_OK) return rc;
    return visc_pcg(c, s, w, OpViscImplicitMatvecField{w.D, w.Ap, dt}, tol, max_iter, c->viscStats);
}

extern "C" int sphk_thermal_viscosity_eval(sphk_ctx* c, const sphk_viscosity_law* law, const float* T, float* nu_out, int n) {
    if (!c || !T || !nu_out || T == nu_out || n < 0 || check_thermal_viscosity(law) != SPHK_OK) return SPHK_ERR_INVALID;
    if (n == 0) return SPHK_OK;
    if (c->sTag == nu_out) c->sTag = nullptr;
    k_thermal_nu<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(*law, T, nu_out, n);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// ---- fluid-solid adhesion (DESIGN.md section 2.11) ------------------------------------------------------------------------------
// the step's group table beta_g (groups past n_groups: 0) from the setting passed by value, and the statistics reset
__global__ void k_adhesion_begin(sphk_adhesion_setting ad, float* __restrict__ groups, unsigned int* __restrict__ stats, const int* pred) {
    if (pred && *pred == 0) return;
    const int g = threadIdx.x;
    if (g < SPHK_ADHESION_GROUPS) groups[g] = g < ad.n_groups ? ad.beta[g] : 0.f;
    if (g == 0) { stats[0] = 0u; stats[1] = 0u; }
}
// One thread per fluid particle: the 9 rows of boundary cell ranges around the particle's current cell (boundary records do not
// move between the boundary search and the velocity stage: sphk_bodies_step searches after it places the bodies).  Without
// bodies every boundary particle is in group 0, whose beta comes by value; with bodies the group is local[b].w and beta_g comes
// from the table (read only for pairs in the band).  accel: a_i per element (tests); else v += dt a_i where some pair acted.
__global__ void __launch_bounds__(SPHK_BLOCK)
k_adhesion(const DevScene s, float* __restrict__ vel, float* __restrict__ accel, const float4* __restrict__ local,
           const float* __restrict__ groups, float beta0, float psi, float cA, float dt, unsigned int* __restrict__ stats) {
    if (s.pred && *s.pred == 0) return;
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= s.nF) return;
    const float3 xi = xyz(rec_lo(s.rec + i));
    const int cx = cell_coord(xi.x, s.cellLength) - s.org.x, cy = cell_coord(xi.y, s.cellLength) - s.org.y,
              cz = cell_coord(xi.z, s.cellLength) - s.org.z;
    float3 a = make_float3(0.f, 0.f, 0.f);
    bool wet = false;
    if (cx >= 0 && cx < s.cs.x && cy >= 0 && cy < s.cs.y && cz >= 0 && cz < s.cs.z) {      // off the grid: no interaction
        const int zlo = max(cz - 1, 0), zhi = min(cz + 1, s.cs.z - 1);
#pragma unroll 1
        for (int x = max(cx - 1, 0); x <= min(cx + 1, s.cs.x - 1); ++x)
#pragma unroll 1
            for (int y = max(cy - 1, 0); y <= min(cy + 1, s.cs.y - 1); ++y) {
                const int c0 = (x * s.cs.y + y) * s.cs.z;
                const int end = s.csB[c0 + zhi + 1];
                for (int b = s.csB[c0 + zlo]; b < end; ++b) {
                    const float4 pb = rec_lo(s.rec + s.bOff + b);          // {x_b, m_b}
                    const float3 d = xi - xyz(pb);
                    const float r = sqrtf(dot3(d, d));
                    const float w = adhesion_w(r, s.k.R, cA);
                    if (w == 0.0f) continue;
                    const float beta = local ? groups[static_cast<int>(body_group(local[b]))] : beta0;
                    if (!(beta > 0.0f)) continue;
                    a -= (beta * psi * pb.w * __fdividef(w, r)) * d;
                    wet = true;
                }
            }
    }
    if (accel) store3(accel, i, a);
    else if (wet) {
        const float3 v = load3(vel, i) + dt * a;
        store3(vel, i, v);
        rec_set_vel(s.rec + i, v);
    }
    namespace cg = cooperative_groups;
    const float am = sqrtf(dot3(a, a));
    const cg::coalesced_group grp = cg::coalesced_threads();
    const unsigned int amax = cg::reduce(grp, __float_as_uint(am), cg::greater<unsigned int>());
    const unsigned int cnt = __popc(grp.ballot(wet));
    if (grp.thread_rank() == 0) {
        if (amax) atomicMax(stats + 1, amax);
        if (cnt) atomicAdd(stats, cnt);
    }
}

static int check_adhesion_call(sphk_ctx* c, const sphk_adhesion_setting* ad, float rho0, float rhoB) {
    if (!ad || ad->n_groups < 1 || ad->n_groups > SPHK_ADHESION_GROUPS || !(rho0 > 0.f) || !(rhoB > 0.f) || !finite_f(rho0) ||
        !finite_f(rhoB))
        return SPHK_ERR_INVALID;
    for (int g = 0; g < ad->n_groups; ++g)
        if (!finite_nonneg(ad->beta[g])) return SPHK_ERR_INVALID;
    if (c->actCount >= 0 || c->rangeDev) return SPHK_ERR_STATE;      // slab ranks: not supported
    if (ad->n_groups > 1 + (c->bodies ? c->bodies->nBodies : 0)) return SPHK_ERR_STATE;
    return SPHK_OK;
}

static double adhesion_scale(float R) { return 0.007 / std::pow(static_cast<double>(R), 3.25); }

// the table + statistics reset, then the sweep (accel: per element, else the velocity update)
static int adhesion_sweep(sphk_ctx* c, const sphk_scene* s, const sphk_adhesion_setting& ad, float* accel, float dt, float rho0, float rhoB) {
    k_adhesion_begin<<<1, 96, 0, c->stream>>>(ad, c->adhGroups, c->adhStats, c->pred);
    c->launches++;
    const DevScene d = dev_scene(c, s);
    if (c->nF > 0) {
        k_adhesion<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(d, s->fluid.vel, accel, c->bodies ? c->bodies->local : nullptr,
                                                                     c->adhGroups, ad.beta[0], rho0 / rhoB,
                                                                     static_cast<float>(adhesion_scale(s->radius)), dt, c->adhStats);
        c->launches++;
    }
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_adhesion(sphk_ctx* c, const sphk_scene* s, const sphk_adhesion_setting* ad, float dt, float rho0, float rho_boundary) {
    SPHK_CHECK_SCENE(c, s);
    if (!finite_nonneg(dt)) return SPHK_ERR_INVALID;
    const int rc0 = check_adhesion_call(c, ad, rho0, rho_boundary);
    if (rc0 != SPHK_OK) return rc0;
    const BodyState* B = c->bodies;
    bool bodyAdheres = false;
    for (int g = 1; g < ad->n_groups; ++g) bodyAdheres = bodyAdheres || ad->beta[g] > 0.f;
    const bool react = B && B->acc && bodyAdheres && c->nB > 0;
    if (react && !s->fluid.mass) return SPHK_ERR_INVALID;         // (before any launch: a refused call changes nothing)
    const int rc = adhesion_sweep(c, s, *ad, nullptr, dt, rho0, rho_boundary);
    if (rc != SPHK_OK) return rc;
    // the reaction on the bodies, into the impulse of the step (sphk_bodies_integrate)
    if (react) {
        // positions moved since the search (PBD corrections): a fluid particle within R of x_k may be listed two cells away
        const int reach = c->posDirty ? 2 : 1;
        const ReactAdhesion pair{c->adhGroups, static_cast<double>(dt) * rho0 / rho_boundary, static_cast<float>(adhesion_scale(s->radius))};
        k_bodies_react<<<sphk_blocks(c->nB), SPHK_BLOCK, 0, c->stream>>>(dev_scene(c, s), s->fluid.mass, B->local, B->decl, B->pose,
                                                                        c->nB, B->nStatic, reach, pair, B->acc);
        c->launches++;
        SPHK_CUDA_TRY(cudaGetLastError());
    }
    return SPHK_OK;
}

extern "C" int sphk_adhesion_accel(sphk_ctx* c, const sphk_scene* s, const sphk_adhesion_setting* ad, float* accel, float rho0,
                                   float rho_boundary) {
    SPHK_CHECK_SCENE(c, s);
    if (!accel || aliases(accel, s)) return SPHK_ERR_INVALID;
    const int rc = check_adhesion_call(c, ad, rho0, rho_boundary);
    if (rc != SPHK_OK) return rc;
    if (c->sTag == accel) c->sTag = nullptr;
    return adhesion_sweep(c, s, *ad, accel, 0.f, rho0, rho_boundary);
}

extern "C" int sphk_adhesion_stats(sphk_ctx* c, int* wetted, float* max_accel) {
    if (!c) return SPHK_ERR_INVALID;
    unsigned int st[2];
    SPHK_CUDA_TRY(cudaMemcpyAsync(st, c->adhStats, sizeof(st), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    float am;
    memcpy(&am, &st[1], sizeof(am));
    if (wetted) *wetted = static_cast<int>(st[0]);
    if (max_accel) *max_accel = am;
    return SPHK_OK;
}

extern "C" int sphk_build_neighbor_list(sphk_ctx* c, const sphk_scene* s) {
    SPHK_CHECK_SCENE(c, s);
    const DevScene d = dev_scene(c, s);
    const int rc = ensure_list(c, d);
    if (rc != SPHK_OK) return rc;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_get_neighbor_list(sphk_ctx* c, const sphk_scene* s, int* counts_out, int* entries_out) {
    SPHK_CHECK_SCENE(c, s);
    if (c->tile) return SPHK_ERR_STATE;     // tile lists hold 16-bit window slots: sphk_get_tile_lists reads them
    const DevScene d = dev_scene(c, s);
    const int rc = ensure_list(c, d);
    if (rc != SPHK_OK) return rc;
    if (counts_out) SPHK_CUDA_TRY(cudaMemcpyAsync(counts_out, c->cnt, sizeof(int) * static_cast<size_t>(c->nF), cudaMemcpyDeviceToDevice, c->stream));
    if (entries_out) SPHK_CUDA_TRY(cudaMemcpyAsync(entries_out, c->nbr, sizeof(int) * static_cast<size_t>(c->kmax) * c->capF,
                                                   cudaMemcpyDeviceToDevice, c->stream));
    return SPHK_OK;
}

extern "C" int sphk_get_tile_lists(sphk_ctx* c, const sphk_scene* s, int* counts_out, unsigned short* slots_out, int* windows_out) {
    SPHK_CHECK_SCENE(c, s);
    if (!c->tile) return SPHK_ERR_STATE;    // int32 lists: sphk_get_neighbor_list
    const DevScene d = dev_scene(c, s);
    const int rc = ensure_list(c, d);
    if (rc != SPHK_OK) return rc;
    const size_t planes = static_cast<size_t>(c->kmax + 7) / 8, tiles = (static_cast<size_t>(c->nF) + SPHK_BLOCK - 1) / SPHK_BLOCK;
    if (counts_out) SPHK_CUDA_TRY(cudaMemcpyAsync(counts_out, c->cnt, sizeof(int) * static_cast<size_t>(c->nF), cudaMemcpyDeviceToDevice, c->stream));
    if (slots_out) SPHK_CUDA_TRY(cudaMemcpyAsync(slots_out, c->nbr, 16 * planes * c->capF, cudaMemcpyDeviceToDevice, c->stream));
    if (windows_out) SPHK_CUDA_TRY(cudaMemcpyAsync(windows_out, c->tileWin, sizeof(int2) * tiles * SPHK_TILE_WINS, cudaMemcpyDeviceToDevice, c->stream));
    return SPHK_OK;
}

extern "C" int sphk_get_skin_displacement(sphk_ctx* c, float* host_out) {
    if (!c || !host_out) return SPHK_ERR_INVALID;
    unsigned int bits = 0;
    SPHK_CUDA_TRY(cudaMemcpyAsync(&bits, c->dispMax, sizeof(bits), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    float d2;
    memcpy(&d2, &bits, sizeof(d2));
    *host_out = sqrtf(d2);
    return SPHK_OK;
}

extern "C" int sphk_list_stats(sphk_ctx* c, const sphk_scene* s, long long out_host[3]) {
    SPHK_CHECK_SCENE(c, s);
    if (!out_host) return SPHK_ERR_INVALID;
    DevScene d = dev_scene(c, s);
    const int rc = ensure_list(c, d);
    if (rc != SPHK_OK) return rc;
    unsigned long long* dev = reinterpret_cast<unsigned long long*>(c->partial);
    SPHK_CUDA_TRY(cudaMemsetAsync(dev, 0, 3 * sizeof(unsigned long long), c->stream));
    k_list_stats<<<256, 256, 0, c->stream>>>(c->cnt + c->listBegin, c->listEnd - c->listBegin, c->kmax, dev);
    c->launches++;
    unsigned long long h[3];
    SPHK_CUDA_TRY(cudaMemcpyAsync(h, dev, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (int k = 0; k < 3; ++k) out_host[k] = static_cast<long long>(h[k]);
    return SPHK_OK;
}

// ---- tank motion (DESIGN.md section 2.15) ---------------------------------------------------------------------------------------
// The schedule of sphk.h in double, host and device alike (k_tank_begin evaluates it at the device-resident frame time).
struct TankEval {
    double th, thd, thdd, g[3], aw[3];
};
__host__ __device__ static void tank_schedule(const TankParams& P, double t, TankEval& E) {
    const bool ramping = P.ramp > 0.0 && t < P.ramp;
    const double e = ramping ? t / P.ramp : 1.0, ed = ramping ? 1.0 / P.ramp : 0.0;
    const double s = sin(P.omega * t + P.phi), c = cos(P.omega * t + P.phi);
    const double ths = ramping ? P.spin * t * t / (2.0 * P.ramp) : P.spin * (t - 0.5 * P.ramp);
    E.th = e * P.theta * s + ths;
    E.thd = ed * P.theta * s + e * P.theta * P.omega * c + e * P.spin;
    E.thdd = 2.0 * ed * P.theta * P.omega * c - e * P.theta * P.omega * P.omega * s + ed * P.spin;
    double d[3];
    for (int a = 0; a < 3; ++a) {
        double acc = P.ac[a];
        for (int k = 0; k < P.nh; ++k) acc += P.A[k][a] * sin(P.w[k] * t + P.ph[k]);
        E.aw[a] = e * acc;
        d[a] = P.G[a] - E.aw[a];
    }
    // R = Rot(n, -theta): R d = cos(theta) d - sin(theta) n x d + (1 - cos(theta)) n (n . d)
    const double ct = cos(E.th), st = sin(E.th), nd = P.n[0] * d[0] + P.n[1] * d[1] + P.n[2] * d[2];
    const double nxd[3] = {P.n[1] * d[2] - P.n[2] * d[1], P.n[2] * d[0] - P.n[0] * d[2], P.n[0] * d[1] - P.n[1] * d[0]};
    for (int a = 0; a < 3; ++a) E.g[a] = ct * d[a] - st * nxd[a] + (1.0 - ct) * P.n[a] * nd;
}
__host__ __device__ static void tank_state_out(const TankEval& E, float* out) {
    out[0] = static_cast<float>(E.th); out[1] = static_cast<float>(E.thd); out[2] = static_cast<float>(E.thdd);
    for (int a = 0; a < 3; ++a) { out[3 + a] = static_cast<float>(E.g[a]); out[6 + a] = static_cast<float>(E.aw[a]); }
}

static bool tank_params(const sphk_tank_motion* m, const float G[3], TankParams& P) {
    if (!m || !G) return false;
    const float* f3s[] = {m->axis, m->pivot, m->accel, G};
    for (const float* v : f3s)
        for (int a = 0; a < 3; ++a) if (!finite_f(v[a])) return false;
    const float sc[] = {m->roll_amplitude, m->roll_omega, m->roll_phase, m->spin, m->ramp};
    for (float v : sc) if (!finite_f(v)) return false;
    if (m->roll_omega < 0.f || m->ramp < 0.f || m->n_harmonics < 0 || m->n_harmonics > SPHK_TANK_HARMONICS) return false;
    for (int k = 0; k < m->n_harmonics; ++k) {
        if (!finite_nonneg(m->harmonic_omega[k]) || !finite_f(m->harmonic_phase[k])) return false;
        for (int a = 0; a < 3; ++a) if (!finite_f(m->harmonic_amplitude[k][a])) return false;
    }
    const double n2 = double(m->axis[0]) * m->axis[0] + double(m->axis[1]) * m->axis[1] + double(m->axis[2]) * m->axis[2];
    if (!(n2 > 0.0)) return false;
    P = TankParams{};
    const double nl = std::sqrt(n2);
    for (int a = 0; a < 3; ++a) {
        P.n[a] = m->axis[a] / nl; P.p[a] = m->pivot[a]; P.ac[a] = m->accel[a]; P.G[a] = G[a];
    }
    P.theta = m->roll_amplitude; P.omega = m->roll_omega; P.phi = m->roll_phase; P.spin = m->spin; P.ramp = m->ramp;
    P.nh = m->n_harmonics;
    for (int k = 0; k < P.nh; ++k) {
        P.w[k] = m->harmonic_omega[k]; P.ph[k] = m->harmonic_phase[k];
        for (int a = 0; a < 3; ++a) P.A[k][a] = m->harmonic_amplitude[k][a];
    }
    return true;
}

extern "C" int sphk_tank_eval(const sphk_tank_motion* m, const float G[3], double t, float out[SPHK_TANK_STATE]) {
    TankParams P;
    if (!out || !tank_params(m, G, P) || !(t >= 0.0) || !(t - t == 0.0)) return SPHK_ERR_INVALID;
    TankEval E;
    tank_schedule(P, t, E);
    tank_state_out(E, out);
    return SPHK_OK;
}

extern "C" int sphk_tank_accel_bound(const sphk_tank_motion* m, const float G[3], const float space[3], double* bound_out) {
    TankParams P;
    if (!bound_out || !space || !tank_params(m, G, P)) return SPHK_ERR_INVALID;
    for (int a = 0; a < 3; ++a) if (!finite_f(space[a]) || !(space[a] > 0.f)) return SPHK_ERR_INVALID;
    double r2 = 0.0;
    for (int a = 0; a < 3; ++a) {
        const double hi = 0.99 * space[a], far = std::fmax(std::fabs(P.p[a]), std::fabs(hi - P.p[a]));
        r2 += far * far;
    }
    const double Th = std::fabs(P.theta), W = P.omega, S = std::fabs(P.spin), rinv = P.ramp > 0.0 ? 1.0 / P.ramp : 0.0;
    double lin = std::sqrt(P.G[0] * P.G[0] + P.G[1] * P.G[1] + P.G[2] * P.G[2]);
    lin += std::sqrt(P.ac[0] * P.ac[0] + P.ac[1] * P.ac[1] + P.ac[2] * P.ac[2]);
    for (int k = 0; k < P.nh; ++k) lin += std::sqrt(P.A[k][0] * P.A[k][0] + P.A[k][1] * P.A[k][1] + P.A[k][2] * P.A[k][2]);
    const double thd = Th * W + Th * rinv + S;
    *bound_out = lin + std::sqrt(r2) * (Th * W * W + (2.0 * Th * W + S) * rinv + thd * thd);
    return SPHK_OK;
}

extern "C" int sphk_tank_set(sphk_ctx* c, const sphk_tank_motion* m, const float G[3]) {
    if (!c) return SPHK_ERR_INVALID;
    TankParams P{};
    if (m && !tank_params(m, G, P)) return SPHK_ERR_INVALID;
    if (c->actCount >= 0 || c->rangeDev) return SPHK_ERR_STATE;       // slab ranks: not supported
    const bool rotates = m && (m->roll_amplitude != 0.f || m->spin != 0.f);
    if (rotates && c->bodies && c->bodies->anyDynamic) return SPHK_ERR_STATE;
    if (!m) { if (c->tank) c->tank->on = false; return SPHK_OK; }
    if (!c->tank) {
        TankState* T = new TankState();
        cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&T->dev), sizeof(TankStep));
        if (e == cudaSuccess) e = cudaMemsetAsync(T->dev, 0, sizeof(TankStep), c->stream);
        if (e != cudaSuccess) { cudaFree(T->dev); delete T; cudaGetLastError(); return e == cudaErrorMemoryAllocation ? SPHK_ERR_ALLOC : static_cast<int>(e); }
        c->tank = T;
    }
    c->tank->P = P;
    c->tank->on = true;
    c->tank->rotates = rotates;
    return SPHK_OK;
}

// the step's state at the frame time, then the frame time advanced by (double) dt
__global__ void k_tank_begin(TankParams P, float dt, TankStep* __restrict__ st) {
    const double t = st->t;
    TankEval E;
    tank_schedule(P, t, E);
    const double a = -2.0 * E.thd * static_cast<double>(dt), ca = cos(a), sa = sin(a);
    const double* n = P.n;
    // Rot(n, a) = cos(a) I + sin(a) [n]x + (1 - cos(a)) n n^T
    const double K[9] = {0.0, -n[2], n[1], n[2], 0.0, -n[0], -n[1], n[0], 0.0};
    for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 3; ++q) st->rot[3 * r + q] = (r == q ? ca : 0.0) + sa * K[3 * r + q] + (1.0 - ca) * n[r] * n[q];
    float s[SPHK_TANK_STATE];
    tank_state_out(E, s);
    for (int k = 0; k < SPHK_TANK_STATE; ++k) st->state[k] = s[k];
    for (int k = 0; k < 3; ++k) st->dv[k] = dt * s[3 + k];          // as sphk_gravity forms dt G
    st->thdd_dt = static_cast<float>(E.thdd * dt);
    st->w2_dt = static_cast<float>(E.thd * E.thd * dt);
    st->t = t + static_cast<double>(dt);
}
// v <- Rot(n, -2 thd dt) v + dt (R (G - a_w) - thdd n x r - thd^2 n x (n x r)); k_gravity's arithmetic when thd = thdd = 0
__global__ void __launch_bounds__(SPHK_BLOCK)
k_tank_force(Rec rec, float* __restrict__ vel, int n, const TankStep* __restrict__ st, float3 ax, float3 pivot) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float4 hi = rec_hi(rec + i);
    const float3 dv = f3(st->dv[0], st->dv[1], st->dv[2]);
    const float s0 = st->state[1], s1 = st->state[2];
    float3 v;
    if (s0 == 0.0f && s1 == 0.0f) {
        v = f3(hi.x + dv.x, hi.y + dv.y, hi.z + dv.z);
    } else {
        const float3 r = xyz(rec_lo(rec + i)) - pivot;
        const float3 nr = f3(ax.y * r.z - ax.z * r.y, ax.z * r.x - ax.x * r.z, ax.x * r.y - ax.y * r.x);
        const float3 nnr = f3(ax.y * nr.z - ax.z * nr.y, ax.z * nr.x - ax.x * nr.z, ax.x * nr.y - ax.y * nr.x);
        const double* M = st->rot;
        const double vx = hi.x, vy = hi.y, vz = hi.z;
        const float3 vr = f3(static_cast<float>(M[0] * vx + M[1] * vy + M[2] * vz), static_cast<float>(M[3] * vx + M[4] * vy + M[5] * vz),
                             static_cast<float>(M[6] * vx + M[7] * vy + M[8] * vz));
        const float a = st->thdd_dt, b = st->w2_dt;
        v = vr + (dv - a * nr - b * nnr);
    }
    rec_set_vel(rec + i, v); store3(vel, i, v);
}

extern "C" int sphk_tank_force(sphk_ctx* c, const sphk_scene* s, float dt) {
    SPHK_CHECK_SCENE(c, s);
    if (!finite_nonneg(dt)) return SPHK_ERR_INVALID;
    if (!c->tank || !c->tank->on) return SPHK_ERR_STATE;
    const TankState* T = c->tank;
    k_tank_begin<<<1, 1, 0, c->stream>>>(T->P, dt, T->dev);
    c->launches++;
    if (c->nF > 0) {
        const float3 ax = make_float3(static_cast<float>(T->P.n[0]), static_cast<float>(T->P.n[1]), static_cast<float>(T->P.n[2]));
        const float3 pv = make_float3(static_cast<float>(T->P.p[0]), static_cast<float>(T->P.p[1]), static_cast<float>(T->P.p[2]));
        k_tank_force<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(c->rec, s->fluid.vel, c->nF, T->dev, ax, pv);
        c->launches++;
    }
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

__global__ void k_tank_set_time(TankStep* st, double t) { st->t = t; }

extern "C" int sphk_tank_set_time(sphk_ctx* c, double t) {
    if (!c || !(t >= 0.0) || !(t - t == 0.0)) return SPHK_ERR_INVALID;
    if (!c->tank) return SPHK_ERR_STATE;
    k_tank_set_time<<<1, 1, 0, c->stream>>>(c->tank->dev, t);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_tank_time(sphk_ctx* c, double* t, float* state_or_null) {
    if (!c || !t) return SPHK_ERR_INVALID;
    if (!c->tank) return SPHK_ERR_STATE;
    TankStep h;
    SPHK_CUDA_TRY(cudaMemcpyAsync(&h, c->tank->dev, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    *t = h.t;
    if (state_or_null) memcpy(state_or_null, h.state, sizeof(h.state));
    return SPHK_OK;
}
