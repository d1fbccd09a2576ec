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
    struct Acc { float e; float3 vi; template <class F> __device__ void sums(F f) { f(e); } };
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
    __device__ void end(Acc& a, int i, float4, float4 hi, const DevScene&) const {
        if (kMode == 2) { store3(deltaPos, i, a.a / dt_or_rho0); return; }
        const float3 dv = (kMode == 1) ? a.a / dt_or_rho0 : a.a;
        const float3 v = f3(hi.x + dv.x, hi.y + dv.y, hi.z + dv.z);
        rec_set_vel(rec + i, v); store3(vel, i, v);
    }
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

// one particle's walk of its neighbour list (thread per particle)
template <class Op>
__device__ __forceinline__ void sweep_list_particle(const DevScene& s, const Op& op, int i) {
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
}

template <class Op>
__global__ void __launch_bounds__(SPHK_BLOCK) k_sweep_list(const DevScene s, const Op op) {
    if (s.pred && *s.pred == 0) return;
    int t = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (s.patch > 0) {               // groups of 4 runs of `patch` chunks; block bb of a group: chunk bb of each run, one per warp
        static_assert(SPHK_BLOCK == 128, "four warps per block");
        const int chunk = t >> 5, per = 4 * s.patch, g = chunk / per, r = chunk - g * per;
        t = ((g * per + (r & 3) * s.patch + (r >> 2)) << 5) | (t & 31);
    }
    const int i = s.iBegin + t;
    if (!in_range(s, i)) return;
    sweep_list_particle(s, op, i);
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
#define SPHK_BUILD_CAP 2047
__device__ __forceinline__ void build_range_staged(const float4* smA, int slot0, int j0g, int count, float3 xi, float r2list, int self,
                                                   int kmax, int& n, int*& wp, long long jump) {
    for (int k0 = 0; k0 < count; k0 += 32) {
        const int len = min(32, count - k0);
        const float4* base = smA + slot0 + k0;
        unsigned int mask = 0u;
#pragma unroll 4
        for (int k = 0; k < len; ++k) {
            const float3 d = xi - xyz(base[k]);
            mask |= (dot3(d, d) <= r2list ? 1u : 0u) << k;
        }
        const int sf = self - (j0g + k0);
        if (sf >= 0 && sf < 32) mask &= ~(1u << sf);
        while (mask) {
            const int k = __ffs(mask) - 1;
            mask &= mask - 1;
            if (n < kmax) *wp = j0g + k0 + k;
            wp += ((n & 3) == 3) ? jump : 1;
            ++n;
        }
    }
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_build_list_staged(const DevScene s, int* __restrict__ nbr, int* __restrict__ cnt, float4* __restrict__ posBuild) {
    extern __shared__ float4 smA[];                 // [SPHK_BUILD_CAP + 1]
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
    if (threadIdx.x < SPHK_TILE_WINS) sWin[threadIdx.x] = tile_window(s, threadIdx.x, sMin, sMax, ncells);
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
    int n = 0;
    int* wp = nbr + static_cast<size_t>(i) * 4;
    const long long jump = static_cast<long long>(s.nbrStride) * 4 - 3;
#pragma unroll 1
    for (int r = 0; r < 9; ++r) {
        const int x = cx + r / 3 - 1, y = cy + r % 3 - 1;
        if (x < 0 || x >= s.cs.x || y < 0 || y >= s.cs.y) continue;
        const int c0 = (x * s.cs.y + y) * s.cs.z;
        {
            const int a = s.csF[c0 + zlo], b = s.csF[c0 + zhi + 1];
            build_range_staged(smA, sPre[r] + (a - sWin[r].x), a, b - a, xi, s.r2list, i, s.kmax, n, wp, jump);
        }
        {
            const int a = s.csB[c0 + zlo], b = s.csB[c0 + zhi + 1];
            if (b > a) build_range_staged(smA, sPre[r + 9] + (a + s.bOff - sWin[r + 9].x), a + s.bOff, b - a, xi, s.r2list, -1, s.kmax, n, wp, jump);
        }
    }
    cnt[i] = n;
    for (int m = n; (m & 3) && m < s.kmax; ++m) { *wp = i; ++wp; }            // pad the open batch with the particle itself
}

// ---- sweep ----------------------------------------------------------------------------------------------------------------
template <class Op>
__device__ __forceinline__ void tile_pair(const DevScene& s, const Op& op, typename Op::Acc& acc, int i, float3 xi, int slot, int preB,
                                          const float4* smA, const float4* smB, float m0) {
    const bool isB = slot >= preB;
    if (Op::kFluidOnly && isB) return;
    const float4 lo = smA[slot];
    float4 hi = make_float4(0.f, 0.f, 0.f, 0.f);
    if (Op::kHi) hi = smB[slot];
    const float3 d = xi - xyz(lo);
    feed_pair(s, op, acc, i, xi, -1, isB, lo, hi, m0, d, dot3(d, d));
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
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.x & 0xffffu), preB, smA, smB, m0);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.x >> 16), preB, smA, smB, m0);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.y & 0xffffu), preB, smA, smB, m0);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.y >> 16), preB, smA, smB, m0);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.z & 0xffffu), preB, smA, smB, m0);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.z >> 16), preB, smA, smB, m0);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.w & 0xffffu), preB, smA, smB, m0);
            tile_pair(s, op, acc, i, xi, static_cast<int>(j8.w >> 16), preB, smA, smB, m0);
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
__global__ void __launch_bounds__(SPHK_BLOCK) k_s_copy(const float* __restrict__ a, Rec rec, int n) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i < n) rec_set_s(rec + i, a[i]);
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
    return d;
}

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
        const int smem = (SPHK_BUILD_CAP + 1) * 16;
        if (!attr) { cudaFuncSetAttribute(k_build_list_staged, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); attr = true; }
        const int tiles = (b.iEnd + SPHK_BLOCK - 1) / SPHK_BLOCK - b.iBegin / SPHK_BLOCK;
        k_build_list_staged<<<tiles, SPHK_BLOCK, smem, c->stream>>>(b, c->nbr, c->cnt, nullptr);
    } else {
        k_build_list<<<sphk_blocks(b.iEnd - b.iBegin), SPHK_BLOCK, 0, c->stream>>>(b, c->nbr, c->cnt, nullptr);
    }
    c->launches++;
    c->listEpoch = c->searchEpoch;
    return SPHK_OK;
}

template <class Op> static int run_sweep(sphk_ctx* c, const sphk_scene* s, const Op& op) {
    DevScene d = dev_scene(c, s);
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
            int blocks = sphk_blocks(d.iEnd - d.iBegin);
            if (d.patch > 0) blocks = (blocks + d.patch - 1) / d.patch * d.patch;      // whole groups (4 * patch chunks = patch blocks)
            k_sweep_list<Op><<<blocks, SPHK_BLOCK, 0, c->stream>>>(d, op);
        }
    } else {
        k_sweep_cells<Op><<<sphk_blocks(d.iEnd - d.iBegin), SPHK_BLOCK, 0, c->stream>>>(d, op);
    }
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// rec.s must mirror `array` before a sweep that gathers it; skipped when the previous sweep wrote both
static void ensure_scalar(sphk_ctx* c, const float* array) {
    if (c->sTag == array) return;
    k_s_copy<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(array, c->rec, c->nF);
    c->launches++;
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
    const int rc = run_sweep(c, s, op);
    c->sTag = stiff;
    return rc;
}

extern "C" int sphk_dfsph_den_error(sphk_ctx* c, const sphk_scene* s, const float* alpha, float* error, float* stiff,
                                    float dt, float rho0, float* warm) {
    SPHK_CHECK_SCENE(c, s);
    if (!alpha || !error || !stiff || !s->fluid.density) return SPHK_ERR_INVALID;
    if (warm == c->sTag) c->sTag = nullptr;
    OpDfsphError<true> op{c->rec, s->fluid.density, alpha, error, stiff, warm, dt, rho0};
    const int rc = run_sweep(c, s, op);
    c->sTag = stiff;
    return rc;
}

extern "C" int sphk_dfsph_div_correct(sphk_ctx* c, const sphk_scene* s, const float* stiff) {
    SPHK_CHECK_SCENE(c, s);
    if (!stiff) return SPHK_ERR_INVALID;
    ensure_scalar(c, stiff);
    OpScalarGradient<0> op{c->rec, s->fluid.vel, nullptr, 1.0f};
    return run_sweep(c, s, op);
}

extern "C" int sphk_dfsph_den_correct(sphk_ctx* c, const sphk_scene* s, const float* stiff, float dt) {
    SPHK_CHECK_SCENE(c, s);
    if (!stiff) return SPHK_ERR_INVALID;
    ensure_scalar(c, stiff);
    OpScalarGradient<1> op{c->rec, s->fluid.vel, nullptr, dt};
    return run_sweep(c, s, op);
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
// fluid cell ranges of the search and forms each pair term as the fluid sweep forms it, g = (m_k s_i) (d gradWfactor),
// d = x_i - x_k (the fluid particle received c m_i g).  The body particle gathers -c m_i g and its moment about the body's
// centre into its own declaration slot of acc, in double (no atomics: every slot has one writer, sums are in walk order).
__global__ void __launch_bounds__(SPHK_BLOCK)
k_bodies_react(const DevScene s, const float* __restrict__ massF, const float4* __restrict__ local, const int* __restrict__ decl,
               const float* __restrict__ pose, int nB, int nStatic, int reach, float coef, double* __restrict__ acc) {
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
    const double cc = coef;
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
                const float3 t = (mk * lo.w) * (d * grad_w_factor(sqrtf(r2), s.k));
                const double f = -cc * static_cast<double>(massF[j]);
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
                                                                    c->nB, B->nStatic, reach, coef, B->acc);
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
    if (color_grad_or_null) {
        OpDensityAlphaDivError<true> op{{OpPair<OpDensityAlpha, OpColorGrad>{OpDensityAlpha{s->fluid.density, alpha},
                                                                             OpColorGrad{color_grad_or_null, rho0, rhoB}}, err}};
        rc = run_sweep(c, s, op);
    } else {
        OpDensityAlphaDivError<false> op{{OpDensityAlpha{s->fluid.density, alpha}, err}};
        rc = run_sweep(c, s, op);
    }
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
    const int n = c->nF;
    ViscCg* st = reinterpret_cast<ViscCg*>(work);
    double* part = reinterpret_cast<double*>(work + SPHK_VISC_HEAD);
    float* D = work + SPHK_VISC_HEAD + 2 * 3 * SPHK_VISC_PARTS;
    float *Dinv = D + 6LL * n, *r = Dinv + 6LL * n, *z = r + 3LL * n, *Ap = z + 3LL * n;
    const float nuRho = nu / rho0, nuBRho = nu_boundary / rho_boundary;
    float* vel = s->fluid.vel;
    int rc = run_sweep(c, s, OpViscImplicitSetup{D, Dinv, r, nuRho, nuBRho, dt});          // b -> r
    if (rc != SPHK_OK) return rc;
    const OpViscImplicitMatvec mv{D, Ap, nuRho, dt};
    rc = run_sweep(c, s, mv);                                                                // A v*
    if (rc != SPHK_OK) return rc;
    const int m = visc_blocks(n);
    k_visc_init<<<m, SPHK_VISC_RED, 0, c->stream>>>(c->rec, vel, r, Ap, Dinv, z, n, part);
    k_visc_init_finish<<<1, SPHK_VISC_RED, 0, c->stream>>>(st, part, m, static_cast<double>(tol) * tol, max_iter);
    c->launches += 2;
    const int* outer = c->pred;
    c->pred = &st->active;
    for (int k = 0; k < max_iter && rc == SPHK_OK; ++k) {
        rc = run_sweep(c, s, mv);
        k_visc_alpha_partial<<<m, SPHK_VISC_RED, 0, c->stream>>>(st, c->rec, Ap, n, part);
        k_visc_alpha_finish<<<1, SPHK_VISC_RED, 0, c->stream>>>(st, part, m);
        k_visc_update<<<m, SPHK_VISC_RED, 0, c->stream>>>(st, c->rec, vel, r, Ap, Dinv, z, n, part);
        k_visc_beta_finish<<<1, SPHK_VISC_RED, 0, c->stream>>>(st, part, m);
        k_visc_direction<<<m, SPHK_VISC_RED, 0, c->stream>>>(st, c->rec, z, n);
        c->launches += 5;
    }
    c->pred = outer;
    if (n > 0) { k_visc_set_rec_vel<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(c->rec, vel, n); c->launches++; }   // records <- x
    k_visc_report<<<1, 1, 0, c->stream>>>(st, c->viscStats);
    c->launches++;
    if (rc != SPHK_OK) return rc;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
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
