// Fused batched environment kernel for sm_90a: action clip -> bus injections -> polar
// Newton-Raphson on the (radial) Ybus with a zero-fill 2x2-block elimination -> reward / info ->
// next profile row (+ noise) -> zone-masked observation gather. One launch per env step.
//
// Work decomposition: a group of G threads owns one env instance - a sub-warp slice (G <= 32: 32/G envs
// per warp in lock-step) or 2-4 whole warps (G = 64 / 128, large feeders); the env's
// Newton state lives in shared memory (one 144 B record per PQ bus, 128-bit accesses); the network's
// admittances, the elimination schedule, the element->bus maps and the observation program
// (identical for all envs) are staged once per CTA with a TMA bulk copy. The Newton loop never
// touches HBM and is written branch-light: every "missing child" points at an all-zero slot.
// In MODE_STEP one to four extra (helper) warps per CTA draw the next profile rows + noise of the CTA's
// envs concurrently with the Newton iteration (warp specialisation, two named barriers).
// MODE_DROOP runs the paper's droop-control baseline (a relaxed loop of power flows) inside the same kernel; the host
// path can hand the kernel pinned host memory for actions / results (mapdn_step_host_pinned: no staging copies).
//
// The linear solve works on the forest of PQ buses (the slack bus is not an unknown), each tree
// re-rooted at its centre so that the leaf->root elimination has half the depth of the feeder.
//
// Replaces, per env: reference voltage_control_env.py step :178-211, _take_action :548-566,
// _clip_reactive_power :568-572, pp.runpp (pandapower 2.7.0 newtonpf; SURVEY Appendix A),
// _calc_reward :574-623, voltage_barrier/*.py, _set_demand_and_pv :491-513, get_obs :232-316,
// reset/manual_reset :96-176; traditional_control/pf_droop_matpower_all.m:121-152,196-231 (MODE_DROOP).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "kernel_params.h"
#include "philox.cuh"

namespace mapdn {

// Profile builds (MAPDN_PROFILE_BUILD=1 python -m mapdn_b200.build): clock64 totals per phase of warp 0 of block 0,
// printed by launch_env_kernel (scripts/phase_prof.py). Compiled out otherwise.
#ifdef MAPDN_PROFILE
#define PROF_DECL long long _pt = clock64(); long long _acc[16] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0};
#define PROF(k) { long long _t = clock64(); _acc[k] += _t - _pt; _pt = _t; }
// inside one forward-sweep step (slots 12..15; they overlap slot 5 "elim"): [12] loop top -> children subtracted (load
// wait), [13] -> results stored (arithmetic), [14] step executions, [15] linear solves
#define PROF_STEP_BEGIN long long _s0 = clock64();
#define PROF_STEP_MID long long _s1 = clock64(); _acc[12] += _s1 - _s0;
#define PROF_STEP_END { _acc[13] += clock64() - _s1; _acc[14] += 1; }
#define PROF_COUNT(k) { _acc[k] += 1; }
#else
#define PROF_DECL
#define PROF(k)
#define PROF_STEP_BEGIN
#define PROF_STEP_MID
#define PROF_STEP_END
#define PROF_COUNT(k)
#endif

enum Mode { MODE_SOLVE = 0, MODE_STEP = 1, MODE_RESET = 2, MODE_DROOP = 3 };
constexpr int kMaxResetAttempts = 16;
constexpr unsigned kFull = 0xffffffffu;
constexpr double kRad2Deg = 57.295779513082320876798;

__device__ __forceinline__ double nanmax(double a, double b) { return (b > a || b != b) ? b : a; }

// ---- group primitives. A group = the G threads that own one env: a sub-warp slice (G <= 32, all groups of
//      a warp run in lock-step, synchronised with __syncwarp) or G/32 whole warps (G = 64 / 128, large feeders:
//      synchronised with a named barrier per group; ids 3.. - 0 is __syncthreads, 1-2 the helper warp's) ----
template <int G> __device__ __forceinline__ void grp_sync(int gidx) {
  if constexpr (G <= 32) __syncwarp();
#ifdef MAPDN_HOST_EMU
  else emu::bar_sync(3 + gidx, G);
#else
  else asm volatile("bar.sync %0, %1;" ::"r"(3 + gidx), "r"(G) : "memory");
#endif
}
// true iff `pred` holds on every thread of the group (includes a group barrier when G > 32)
template <int G> __device__ __forceinline__ bool grp_all(int gidx, bool pred) {
  if constexpr (G <= 32) {
    const unsigned ok = __ballot_sync(kFull, pred);
    const unsigned gmask = (G == 32) ? kFull : (((1u << G) - 1u) << ((threadIdx.x & 31) / G * G));
    return (ok & gmask) == gmask;
  } else {
#ifdef MAPDN_HOST_EMU
    return emu::bar_red_and(3 + gidx, G, pred);
#else
    unsigned r;
    asm volatile(
        "{\n\t.reg .pred p, q;\n\t"
        "setp.ne.u32 q, %1, 0;\n\t"
        "bar.red.and.pred p, %2, %3, q;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(r)
        : "r"(static_cast<unsigned>(pred)), "r"(3 + gidx), "r"(G)
        : "memory");
    return r != 0;
#endif
  }
}
// loop-exit test of the lock-step sub-warp groups: every env handled by this warp is done (G <= 32);
// for multi-warp groups the env's own flag decides (it is group-uniform)
template <int G> __device__ __forceinline__ bool grp_exit(bool done) {
  if constexpr (G <= 32) return __all_sync(kFull, done);
  else return done;
}
template <int G> __device__ __forceinline__ double warp_part_sum(double v) {
#pragma unroll
  for (int m = (G < 32 ? G : 32) / 2; m >= 1; m >>= 1) v += __shfl_xor_sync(kFull, v, m);
  return v;
}
template <int G> __device__ __forceinline__ double warp_part_max(double v) {
#pragma unroll
  for (int m = (G < 32 ? G : 32) / 2; m >= 1; m >>= 1) v = fmax(v, __shfl_xor_sync(kFull, v, m));
  return v;
}
// sum / max over the group of NV values at once; `scratch` = >= NV * G/32 doubles of the env's slab (G > 32 only)
template <int G, int NV> __device__ __forceinline__ void grp_reduce(int gidx, int gl, double (&v)[NV], const bool (&is_max)[NV],
                                                                    double* scratch) {
#pragma unroll
  for (int k = 0; k < NV; ++k) v[k] = is_max[k] ? warp_part_max<G>(v[k]) : warp_part_sum<G>(v[k]);
  if constexpr (G > 32) {
    constexpr int W = G / 32;
    grp_sync<G>(gidx);                                   // scratch is free
    if ((gl & 31) == 0) {
#pragma unroll
      for (int k = 0; k < NV; ++k) scratch[(gl >> 5) * NV + k] = v[k];
    }
    grp_sync<G>(gidx);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      double a = scratch[k];
#pragma unroll
      for (int w = 1; w < W; ++w) a = is_max[k] ? fmax(a, scratch[w * NV + k]) : a + scratch[w * NV + k];
      v[k] = a;
    }
  }
}

// Reciprocal without the library's special-case branch: MUFU.RCP64H seed (~2^-23 rel. error) + one
// third-order step r (1 + e + e^2), e = 1 - x r (-> ~2^-69 before rounding: 3 dependent FMAs instead of the 4 of
// two Newton steps). A zero / denormal pivot yields inf/NaN, which the solver reports as
// "not converged" - the same outcome pandapower reaches through a singular-matrix warning.
__device__ __forceinline__ double fast_rcp(double x) {
  double r;
#ifdef MAPDN_HOST_EMU
  r = static_cast<double>(static_cast<float>(1.0 / x));      // a seed of about the same quality as MUFU.RCP64H
#else
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
#endif
  const double e = fma(-x, r, 1.0);
  const double t = fma(e, e, e);
  return fma(r, t, r);
}

// sin/cos for the bus angles: distribution-feeder angles are a few degrees, so the common path is a pair of
// Taylor polynomials on |x| <= pi/4 (truncation < 1e-19, i.e. exact to rounding; two independent FMA chains,
// no range reduction); larger angles fall back to the library routine.
__device__ __forceinline__ void sincos_angle(double x, double* sn, double* cs) {
  if (fabs(x) <= 0.78539816339744830962) {
    const double z = x * x;
    double ps = 1.0 / 355687428096000.0;                 // 1/17!
    ps = fma(ps, z, -1.0 / 1307674368000.0);             // -1/15!
    ps = fma(ps, z, 1.0 / 6227020800.0);                 // 1/13!
    ps = fma(ps, z, -1.0 / 39916800.0);                  // -1/11!
    ps = fma(ps, z, 1.0 / 362880.0);                     // 1/9!
    ps = fma(ps, z, -1.0 / 5040.0);                      // -1/7!
    ps = fma(ps, z, 1.0 / 120.0);                        // 1/5!
    ps = fma(ps, z, -1.0 / 6.0);                         // -1/3!
    double pc = 1.0 / 20922789888000.0;                  // 1/16!
    pc = fma(pc, z, -1.0 / 87178291200.0);               // -1/14!
    pc = fma(pc, z, 1.0 / 479001600.0);                  // 1/12!
    pc = fma(pc, z, -1.0 / 3628800.0);                   // -1/10!
    pc = fma(pc, z, 1.0 / 40320.0);                      // 1/8!
    pc = fma(pc, z, -1.0 / 720.0);                       // -1/6!
    pc = fma(pc, z, 1.0 / 24.0);                         // 1/4!
    pc = fma(pc, z, -0.5);                               // -1/2!
    *sn = fma(ps * z, x, x);
    *cs = fma(pc, z, 1.0);
  } else {
    sincos(x, sn, cs);
  }
}

// exp(x) for x in [-0.125, 0] (the only range the bowl barrier needs): degree-9 Taylor, |err| < 3e-15
__device__ __forceinline__ double exp_small(double x) {
  double r = 1.0 / 362880.0;
  r = fma(r, x, 1.0 / 40320.0); r = fma(r, x, 1.0 / 5040.0); r = fma(r, x, 1.0 / 720.0);
  r = fma(r, x, 1.0 / 120.0); r = fma(r, x, 1.0 / 24.0); r = fma(r, x, 1.0 / 6.0);
  r = fma(r, x, 0.5); r = fma(r, x, 1.0); r = fma(r, x, 1.0);
  return r;
}

// ---- voltage barriers: reference voltage_barrier/{l1,l2,bowl,bump,courant_beltrami}.py ----
__device__ __forceinline__ double barrier_fn(int kind, double v) {
  switch (kind) {
    case 0: return fabs(v - 1.0);                                   // l1.py:5-8
    case 1: { const double d = v - 1.0; return 2.0 * d * d; }       // l2.py:5-8
    case 2: {                                                       // bowl.py:5-13
      const double d = fabs(v - 1.0);
      if (d > 0.05) return 2.0 * d - 0.095;
      const double dv = v - 1.0;
      // normal pdf N(v; 1, 0.1); |dv| <= 0.05 here, so the exponent lies in [-0.125, 0]
      const double pdf = 3.9894228040143267794 * exp_small(-50.0 * (dv * dv));
      return -0.01 * pdf + 0.04;
    }
    case 3: {                                                       // bump.py:5-13
      if (fabs(v) < 1.0) { const double v2 = v * v; return exp(-1.0 / (1.0 - v2 * v2)); }
      if (v > 1.0 && v < 3.0) { const double w = v - 2.0, w2 = w * w; return exp(-1.0 / (1.0 - w2 * w2)); }
      return 0.0;
    }
    default: {                                                      // courant_beltrami.py:5-8
      const double hi = fmax(0.0, v - 1.05), lo = fmax(0.0, 0.95 - v);
      return hi * hi + lo * lo;
    }
  }
}

// ---- TMA bulk copy of the hot static blob into shared memory (one thread issues) ----
__device__ __forceinline__ void stage_hot_issue(unsigned char* smem_dst, const unsigned char* gsrc,
                                                int bytes, uint64_t* bar) {
#ifdef MAPDN_HOST_EMU
  (void)bar;
  if (threadIdx.x == 0) memcpy(smem_dst, gsrc, bytes);      // the bulk copy has landed when the barrier below releases
  __syncthreads();
  return;
#endif
  const uint32_t bar_a = static_cast<uint32_t>(__cvta_generic_to_shared(bar));
  const uint32_t dst_a = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_a),
        "l"(gsrc), "r"(bytes), "r"(bar_a)
        : "memory");
  }
  __syncthreads();      // the barrier is initialised before anybody waits on it
}
__device__ __forceinline__ void stage_hot_wait(uint64_t* bar) {
#ifdef MAPDN_HOST_EMU
  (void)bar;
  return;
#endif
  const uint32_t bar_a = static_cast<uint32_t>(__cvta_generic_to_shared(bar));
  uint32_t done = 0;
  while (!done) {       // every thread waits for phase 0 of the barrier
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar_a)
        : "memory");
  }
}

// Named barriers between the solver warps and the helper warp of a CTA (producer / consumer)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
#ifdef MAPDN_HOST_EMU
  emu::bar_sync(id, nthreads);
#else
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
#endif
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  __threadfence_block();
#ifdef MAPDN_HOST_EMU
  emu::bar_arrive(id, nthreads);
#else
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
#endif
}

// Views of the staged static blob and of one env's shared-memory slab.
struct Hot {
  const double2 *yup, *ydn, *yii;
  const uint64_t *ndesc, *esched, *bsched;
  const uint16_t *lptr, *lidx, *sptr, *sidx, *xptr, *xidx, *node_of_bus;
  // tables read once per env-step: in the staged blob when it fits the launch shape, else straight from global memory
  // (generic pointers; the cold copies are prefetched into L2 at kernel start)
  const double2* ysl;
  bool in_blob;
  const unsigned char* blob;          // the staged blob (typed as shared memory at the use sites)
  const uint16_t *nbr_ptr, *nbr_idx;   // meshed nets (dense solver) only
  const double2* nbr_y;
};
struct Slab {
  double2* nodes;   // (npq + 2) records of kNodeArrays2 double2 (sentinel + trash at the end)
  double* base;     // the slab as a flat double array (obs program offsets index this)
  double* pv;       // sgen.p_mw   [n_sgen]
  double* q;        // sgen.q_mvar [n_sgen]
  double* scratch;  // [n_sgen + 2 n_load]
  __device__ __forceinline__ double2* node(int i) const { return nodes + i * kNodeArrays2; }
};

// ------------------------------------------------------------------------------------------
// Newton-Raphson (pandapower newtonpf, SURVEY A.4) for one env per G-lane group.
// Unknowns (dtheta_i, dV_i/V_i) per PQ bus; J's 2x2 blocks are built from per-edge terms
//   a_ik = ViVk(G_ik sin t_ik - B_ik cos t_ik),  b_ik = ViVk(G_ik cos t_ik + B_ik sin t_ik)
// and eliminated leaf-to-root (no fill on a tree), then back-substituted root-to-leaf.
// Per iteration: ONE pass over the buses (edge terms of (i, parent) + the children's terms recomputed from their
// voltages + mismatch + diagonal blocks), the forward sweep, and a back sweep that also applies the update
// (theta += dtheta, V += V dV/V, V = Vm exp(j theta)) to the bus it has just solved.
// Returns converged; `iters` = number of linear solves (pandapower's iteration count).
// ------------------------------------------------------------------------------------------
template <int G>
__device__ __forceinline__ bool nr_solve(const Params& p, const Hot& h, const Slab& s, int gidx, int gl, bool skip, int& iters
#ifdef MAPDN_PROFILE
    , long long* _acc, long long& _pt
#endif
) {
  const int npq = p.npq;
  // read once: inside the sweep loop the flag was re-fetched from the constant bank every step (ncu: 10 % of the loop's
  // stall samples on the LDCU / compare / branch)
  const bool extra_children = p.has_extra_children != 0;

  // flat start (pandapower init="auto"): |V| = vm_init, angle 0 on every PQ bus; sentinel record (slack voltage,
  // all-zero Jacobian terms: the "no child" / "no parent" slot); trash record (idle lanes: dx = 0 for ever).
  // The FIRST Newton iteration is static up to its right-hand side: at the flat start S_calc and the Jacobian are the same
  // for every env and every step, so mapdn_create factorises J(V0) once (p.first_tab, six double2 per node: S_calc,
  // M = D'^-1 J[i,parent] (two rows), D'^-1 (two rows), J[parent,i]) and this pass seeds the records with it: the mismatch
  // is S_calc - S_spec, the forward sweep only eliminates the right-hand side (sweep1 below: D'^-1 from UP / DN,
  // J[parent,i] from T), the back sweep finds M where a regular elimination would have left it (D01 / D23). pandapower
  // computes the same factors numerically in every runpp; the iterates agree to rounding.
  double nrm = 0.0;
  {
    // the six double2 of the next bus are requested one pass iteration ahead (read-only path; the table sits in L2 / L1)
    struct First { double2 s0, m0, m1, i0, i1, dn; };
    auto load_first = [&](int i) {
      const double2* ft = p.first_tab + 6 * i;
      First f; f.s0 = __ldg(ft); f.m0 = __ldg(ft + 1); f.m1 = __ldg(ft + 2); f.i0 = __ldg(ft + 3); f.i1 = __ldg(ft + 4); f.dn = __ldg(ft + 5);
      return f;
    };
    First nxt = load_first(min(gl, npq - 1));
    for (int i = gl; i <= npq + 1; i += G) {
      const First cur = nxt;
      nxt = load_first(min(i + G, npq - 1));               // clamped: the last lanes re-read bus npq - 1 (unused)
      const bool sl = (i == npq);
      double2* nd = s.node(i);
      nd[A_VV] = sl ? make_double2(p.vm0, p.va0) : make_double2(p.vm_init, 0.0);
      nd[A_EF] = sl ? make_double2(p.e0, p.f0) : make_double2(p.vm_init, 0.0);
      if (i < npq) {
        const double2 sp = nd[A_SP];
        const double Fp = cur.s0.x - sp.x, Fq = cur.s0.y - sp.y;
        nd[A_UP] = cur.i0; nd[A_DN] = cur.i1; nd[A_T] = cur.dn;
        nd[A_D01] = cur.m0; nd[A_D23] = cur.m1;
        nd[A_R] = make_double2(-Fp, -Fq);
        nrm = nanmax(nrm, nanmax(fabs(Fp), fabs(Fq)));
      } else {
        nd[A_UP] = make_double2(0.0, 0.0);
        nd[A_DN] = make_double2(0.0, 0.0);
        nd[A_T] = make_double2(0.0, 0.0);
        nd[A_R] = make_double2(0.0, 0.0);
        nd[A_D01] = make_double2(1.0, 0.0); nd[A_D23] = make_double2(0.0, 1.0);    // idle lanes eliminate an identity block: no NaN / inf arithmetic
      }
    }
  }
  grp_sync<G>(gidx);

  bool done = skip;      // this group's env converged (idle groups never hold the warp back)
  bool first = true;     // the static first iteration (group- and warp-uniform)
  int it = 0;
  iters = 0;
  const double2 v0 = make_double2(p.e0, p.f0);
  while (true) {
    PROF(2)
    if (!first) {
    // --- per-edge terms of (i, parent): row i / col parent and row parent / col i ---
#pragma unroll 4
    for (int i = gl; i < npq; i += G) {
      const int pa = static_cast<int>(static_cast<uint32_t>(h.ndesc[i]) & 0xFFFFu);   // roots: sentinel, Y = 0
      double2* nd = s.node(i);
      const double2 vi = nd[A_EF], vp = s.node(pa)[A_EF];
      const double2 yu = h.yup[i], yd = h.ydn[i];
      const double cc = vi.x * vp.x + vi.y * vp.y;       // ViVp cos(ti - tp)
      const double ss = vi.y * vp.x - vi.x * vp.y;       // ViVp sin(ti - tp)
      nd[A_UP] = make_double2(yu.x * ss - yu.y * cc, yu.x * cc + yu.y * ss);
      nd[A_DN] = make_double2(-yd.x * ss - yd.y * cc, yd.x * cc - yd.y * ss);
    }
    grp_sync<G>(gidx);
    PROF(3)
    // --- mismatch F = S_calc - S_spec and diagonal Jacobian blocks ---
    nrm = 0.0;
    auto mismatch_pass = [&](auto with_extra) {
    constexpr bool kExtra = decltype(with_extra)::value;
#pragma unroll 4
    for (int i = gl; i < npq; i += G) {
      const uint64_t ndc = h.ndesc[i];
      const int c0 = static_cast<int>((ndc >> 16) & 0xFFFFu), c1 = static_cast<int>((ndc >> 32) & 0xFFFFu);
      const int nx = static_cast<int>((ndc >> 48) & 0x7FFFu);
      double2* nd = s.node(i);
      const double2 vi = nd[A_EF];
      const double2 u = nd[A_UP], a0 = s.node(c0)[A_DN], a1 = s.node(c1)[A_DN];  // roots: UP = 0; no child: zero slot
      const double2 sp = nd[A_SP];
      const double2 ys = (ndc >> 63) ? h.ysl[i] : make_double2(0.0, 0.0);   // Y[i, slack]: slack-adjacent buses only
      const double2 yi = h.yii[i];
      const double cs0 = vi.x * v0.x + vi.y * v0.y, sn0 = vi.y * v0.x - vi.x * v0.y;
      double sa = ys.x * sn0 - ys.y * cs0 + u.x + a0.x + a1.x;
      double sb = ys.x * cs0 + ys.y * sn0 + u.y + a0.y + a1.y;
      if (kExtra) {                        // only nets with a bus of degree > 3
#pragma unroll 1
        for (int c = c1 + 1; c <= c1 + nx; ++c) { const double2 d = s.node(c)[A_DN]; sa += d.x; sb += d.y; }
      }
      const double vv = vi.x * vi.x + vi.y * vi.y;
      const double gv = yi.x * vv, bv = yi.y * vv;
      const double P = gv + sb, Q = sa - bv;
      const double Fp = P - sp.x, Fq = Q - sp.y;
      nd[A_D01] = make_double2(-Q - bv, P + gv);     // dP/dtheta, dP/dV * V
      nd[A_D23] = make_double2(P - gv, Q - bv);      // dQ/dtheta, dQ/dV * V
      nd[A_R] = make_double2(-Fp, -Fq);
      nrm = nanmax(nrm, nanmax(fabs(Fp), fabs(Fq)));
    }
    };
    if (extra_children) mismatch_pass(std::true_type{}); else mismatch_pass(std::false_type{});
    }   // !first
    {   // ||F||inf < tol for the whole env <=> every thread of the group is below tol (NaN-safe)
      const bool ok = grp_all<G>(gidx, nrm < p.tol);
      if (!done && ok) { done = true; iters = it; }
    }
    if (grp_exit<G>(done) || it >= p.max_iter) break;
    ++it;
    grp_sync<G>(gidx);
    PROF(4)
    // --- forward elimination, leaves first: a flat schedule of steps (a level of the elimination forest,
    //     split when it is wider than the group), one entry per (step, lane). Lanes follow chains of the
    //     forest: when a bus was eliminated by the same lane in the previous step, its Schur update reaches
    //     the parent in registers (no shared-memory round trip on the critical path); the node's own blocks
    //     are prefetched one step ahead, behind the child loads the step waits for. Idle lanes work on the
    //     trash record: no divergent branches. ---
    {
      struct Own { double2 d01, d23, r, u, d; };
      auto load_own = [&](uint64_t e) {
        const double2* nd = s.node(static_cast<int>(e & 0xFFFFu));
        Own o; o.d01 = nd[A_D01]; o.d23 = nd[A_D23]; o.r = nd[A_R]; o.u = nd[A_UP]; o.d = nd[A_DN];
        return o;
      };
      // two instantiations (nets with / without a bus of degree > 3): tested inside the loop, the flag was re-fetched from the
      // constant bank on every step (ncu: 10 % of the loop's stall samples on LDCU / compare / branch)
      double2 s01 = make_double2(0.0, 0.0), s23 = s01, tt = s01;     // Schur update produced by this lane's last step
      // steps [st0, st1); warp_only: a narrow phase of a multi-warp group - only warp 0 is here, it synchronises with itself
      auto sweep = [&](auto with_extra, auto warp_only, int st0, int st1) {
      constexpr bool kExtra = decltype(with_extra)::value;
      constexpr bool kWarpOnly = decltype(warp_only)::value;
      if (st0 >= st1) return;
      uint64_t ed = h.esched[st0 * G + gl];
      uint64_t ed_next = h.esched[min(st0 + 1, p.n_esteps - 1) * G + gl];
      Own own = load_own(ed);
      for (int st = st0; st < st1; ++st) {
        PROF_STEP_BEGIN
        const uint64_t ed_next2 = h.esched[min(st + 2, p.n_esteps - 1) * G + gl];   // independent of the data
        const int i = static_cast<int>(ed & 0xFFFFu);
        const int c0 = static_cast<int>((ed >> 16) & 0xFFFFu), c1 = static_cast<int>((ed >> 32) & 0xFFFFu);
        const unsigned fl = static_cast<unsigned>(ed >> 48);
        double2* nd = s.node(i);
        double2 d01 = own.d01, d23 = own.d23, r = own.r;
        const double2 u = own.u, d = own.d;   // J[i,p] = [[a,b],[-b,a]](u), J[p,i] likewise (d); zero at roots
        if (kWarpOnly) __syncwarp(); else grp_sync<G>(gidx);  // the previous step's Schur updates are visible
        // child 0: this lane's registers (chain) or shared memory (a leaf reads the all-zero sentinel record)
        double2 p01 = s01, p23 = s23, pt = tt;
        if (fl & kEschedLeaf) { p01 = make_double2(0.0, 0.0); p23 = p01; pt = p01; }     // a lane starting a new chain
        if (fl & kEschedLoad0) { const double2* k0 = s.node(c0); p01 = k0[A_UP]; p23 = k0[A_DN]; pt = k0[A_T]; }
        d01.x -= p01.x; d01.y -= p01.y; d23.x -= p23.x; d23.y -= p23.y; r.x -= pt.x; r.y -= pt.y;
        const Own own_next = load_own(ed_next);          // not touched before its own step: issued behind the child loads
        if (fl & kEschedLoad1) {                          // child 1 (branching buses only): always shared memory
          const double2* k1 = s.node(c1);
          const double2 q01 = k1[A_UP], q23 = k1[A_DN], qt = k1[A_T];
          d01.x -= q01.x; d01.y -= q01.y; d23.x -= q23.x; d23.y -= q23.y; r.x -= qt.x; r.y -= qt.y;
        }
        if (kExtra) {                                    // only nets with a bus of degree > 3
          const int nx = static_cast<int>(fl & 0xFFu);
#pragma unroll 1
          for (int c = c1 + 1; c <= c1 + nx; ++c) {
            const double2* k = s.node(c);
            const double2 x01 = k[A_UP], x23 = k[A_DN], xt = k[A_T];
            d01.x -= x01.x; d01.y -= x01.y; d23.x -= x23.x; d23.y -= x23.y;
            r.x -= xt.x; r.y -= xt.y;
          }
        }
        PROF_STEP_MID
        // adjugate form: everything that does not need 1/det runs beside the reciprocal (shorter chain, +8 flops)
        const double idet = fast_rcp(d01.x * d23.y - d01.y * d23.x);
        const double ca0 = d23.y * r.x - d01.y * r.y, ca1 = d01.x * r.y - d23.x * r.x;   // adj(D) r
        const double ma00 = d23.y * u.x + d01.y * u.y, ma01 = d23.y * u.y - d01.y * u.x; // adj(D) J[i,p]
        const double ma10 = -d23.x * u.x - d01.x * u.y, ma11 = d01.x * u.x - d23.x * u.y;
        const double sa00 = d.x * ma00 + d.y * ma10, sa01 = d.x * ma01 + d.y * ma11;     // J[p,i] adj(D) J[i,p]
        const double sa10 = d.x * ma10 - d.y * ma00, sa11 = d.x * ma11 - d.y * ma01;
        const double ta0 = d.x * ca0 + d.y * ca1, ta1 = d.x * ca1 - d.y * ca0;           // J[p,i] adj(D) r
        const double c0v = ca0 * idet, c1v = ca1 * idet;
        const double m00 = ma00 * idet, m01 = ma01 * idet, m10 = ma10 * idet, m11 = ma11 * idet;
        s01 = make_double2(sa00 * idet, sa01 * idet);
        s23 = make_double2(sa10 * idet, sa11 * idet);
        tt = make_double2(ta0 * idet, ta1 * idet);
        if (fl & kEschedStore) { nd[A_UP] = s01; nd[A_DN] = s23; nd[A_T] = tt; }   // else: it travels in registers
        if (!(fl & kEschedIdle)) {
          nd[A_R] = make_double2(c0v, c1v);                       // D^-1 r  (becomes dx in the back sweep)
          nd[A_D01] = make_double2(m00, m01);                     // D^-1 J[i,p]
          nd[A_D23] = make_double2(m10, m11);
        }
        ed = ed_next; ed_next = ed_next2; own = own_next;
        PROF_STEP_END
      }
      };
      // G > 32: the levels near the roots fit one warp (host schedule: lanes 0..31 from step n_wide_e on) - warp 0 runs them
      // with __syncwarp while the other warps of the group wait at the barrier behind the sweep (case322: 14 of 19 steps)
      auto run_sweep = [&](auto with_extra) {
        if constexpr (G <= 32) {
          sweep(with_extra, std::false_type{}, 0, p.n_esteps);
        } else {
          sweep(with_extra, std::false_type{}, 0, p.n_wide_e);
          if (p.n_wide_e < p.n_esteps) {
            if (p.n_wide_e > 0) grp_sync<G>(gidx);           // the last wide step's updates are visible to warp 0
            if ((gl >> 5) == 0) sweep(with_extra, std::true_type{}, p.n_wide_e, p.n_esteps);
          }
        }
      };
      // The static first iteration: only the right-hand side is eliminated. A step reads r, D'^-1 (two rows) and
      // J[parent,i] from the bus's own record (seeded by the flat-start pass), subtracts the children's rhs updates
      // (registers / shared memory, the same schedule flags as above), and leaves c = D'^-1 r in R and - if the parent
      // fetches it from shared memory - t = J[parent,i] c in T.
      double2 t1 = make_double2(0.0, 0.0);                 // rhs update produced by this lane's last step
      struct Own1 { double2 r, i0, i1, d; };
      auto load_own1 = [&](uint64_t e) {
        const double2* nd = s.node(static_cast<int>(e & 0xFFFFu));
        Own1 o; o.r = nd[A_R]; o.i0 = nd[A_UP]; o.i1 = nd[A_DN]; o.d = nd[A_T];
        return o;
      };
      auto sweep1 = [&](auto with_extra, auto warp_only, int st0, int st1) {
      constexpr bool kExtra = decltype(with_extra)::value;
      constexpr bool kWarpOnly = decltype(warp_only)::value;
      if (st0 >= st1) return;
      uint64_t ed = h.esched[st0 * G + gl];
      uint64_t ed_next = h.esched[min(st0 + 1, p.n_esteps - 1) * G + gl];
      Own1 own = load_own1(ed);
      for (int st = st0; st < st1; ++st) {
        const uint64_t ed_next2 = h.esched[min(st + 2, p.n_esteps - 1) * G + gl];
        const int i = static_cast<int>(ed & 0xFFFFu);
        const int c0 = static_cast<int>((ed >> 16) & 0xFFFFu), c1 = static_cast<int>((ed >> 32) & 0xFFFFu);
        const unsigned fl = static_cast<unsigned>(ed >> 48);
        double2* nd = s.node(i);
        double2 r = own.r;
        const double2 i0 = own.i0, i1 = own.i1, d = own.d;
        if (kWarpOnly) __syncwarp(); else grp_sync<G>(gidx);  // the previous step's rhs updates are visible
        double2 pt = t1;
        if (fl & kEschedLeaf) pt = make_double2(0.0, 0.0);
        if (fl & kEschedLoad0) pt = s.node(c0)[A_T];
        r.x -= pt.x; r.y -= pt.y;
        const Own1 own_next = load_own1(ed_next);        // the next bus's record: nobody writes it before its own step
        if (fl & kEschedLoad1) { const double2 qt = s.node(c1)[A_T]; r.x -= qt.x; r.y -= qt.y; }
        if (kExtra) {
          const int nx = static_cast<int>(fl & 0xFFu);
#pragma unroll 1
          for (int c = c1 + 1; c <= c1 + nx; ++c) { const double2 xt = s.node(c)[A_T]; r.x -= xt.x; r.y -= xt.y; }
        }
        const double c0v = i0.x * r.x + i0.y * r.y, c1v = i1.x * r.x + i1.y * r.y;          // D'^-1 r
        t1 = make_double2(d.x * c0v + d.y * c1v, d.x * c1v - d.y * c0v);                    // J[parent,i] D'^-1 r
        if (fl & kEschedStore) nd[A_T] = t1;
        if (!(fl & kEschedIdle)) nd[A_R] = make_double2(c0v, c1v);
        ed = ed_next; ed_next = ed_next2; own = own_next;
      }
      };
      auto run_sweep1 = [&](auto with_extra) {
        if constexpr (G <= 32) {
          sweep1(with_extra, std::false_type{}, 0, p.n_esteps);
        } else {
          sweep1(with_extra, std::false_type{}, 0, p.n_wide_e);
          if (p.n_wide_e < p.n_esteps) {
            if (p.n_wide_e > 0) grp_sync<G>(gidx);
            if ((gl >> 5) == 0) sweep1(with_extra, std::true_type{}, p.n_wide_e, p.n_esteps);
          }
        }
      };
      if (first) { if (extra_children) run_sweep1(std::true_type{}); else run_sweep1(std::false_type{}); }
      else if (extra_children) run_sweep(std::true_type{}); else run_sweep(std::false_type{});
      PROF_COUNT(15)
      grp_sync<G>(gidx);                                 // the last step's results are visible to the back sweep
    }
    PROF(5)
    // --- back substitution root -> leaves, same flat-schedule form (roots: dx = D^-1 r already); a lane
    //     that solved the parent in the previous step keeps dx_parent in registers ---
    {
      struct OwnB { double2 m01, m23, x; };
      auto load_own = [&](uint64_t e) {
        const double2* nd = s.node(static_cast<int>(e & 0xFFFFu));
        OwnB o; o.m01 = nd[A_D01]; o.m23 = nd[A_D23]; o.x = nd[A_R];
        return o;
      };
      double2 xl = make_double2(0.0, 0.0);               // dx of the node this lane solved in the previous step
      auto bsweep = [&](auto warp_only, int st0, int st1) {
      constexpr bool kWarpOnly = decltype(warp_only)::value;
      if (st0 >= st1) return;
      uint64_t bd = h.bsched[st0 * G + gl];
      uint64_t bd_next = h.bsched[min(st0 + 1, p.n_bsteps - 1) * G + gl];
      OwnB own = load_own(bd);
      for (int st = st0; st < st1; ++st) {
        const uint64_t bd_next2 = h.bsched[max(0, min(st + 2, p.n_bsteps - 1)) * G + gl];
        const unsigned bfl = static_cast<unsigned>(bd >> 32);
        double2* nd = s.node(static_cast<int>(bd & 0xFFFFu));
        if (kWarpOnly) __syncwarp(); else grp_sync<G>(gidx);  // the previous step's dx are visible
        double2 xp = xl;
        if (!(bfl & kBschedRegParent)) xp = s.node(static_cast<int>((bd >> 16) & 0xFFFFu))[A_R];
        const OwnB own_next = load_own(bd_next);         // D^-1 J and D^-1 r are final since the forward sweep
        double2 x = own.x;
        x.x -= own.m01.x * xp.x + own.m01.y * xp.y;
        x.y -= own.m23.x * xp.x + own.m23.y * xp.y;
        if (!(bfl & kBschedIdle)) nd[A_R] = x;           // idle lanes (trash record) store nothing
        xl = x;
        bd = bd_next; bd_next = bd_next2; own = own_next;
      }
      };
      if constexpr (G <= 32) {
        bsweep(std::false_type{}, 0, p.n_bsteps);
      } else {                                             // the levels below the roots fit one warp: warp 0 alone, then everybody
        if ((gl >> 5) == 0) bsweep(std::true_type{}, 0, p.n_narrow_b);
        if (p.n_narrow_b > 0 && p.n_narrow_b < p.n_bsteps) grp_sync<G>(gidx);
        bsweep(std::false_type{}, p.n_narrow_b, p.n_bsteps);
      }
      grp_sync<G>(gidx);
    }
    PROF(6)
    // --- update (theta += dtheta, V += V * dV/V) and V = Vm exp(j theta): a pass of its own - inside the back sweep the
    //     sin/cos chain would sit in front of the next step of the in-order warp ---
#pragma unroll 4
    for (int i = gl; i < npq; i += G) {
      if (!done) {
        double2* nd = s.node(i);
        const double2 x = nd[A_R];
        double2 v = nd[A_VV];
        v.y += x.x;
        v.x += v.x * x.y;
        double sn, cs;
        sincos_angle(v.y, &sn, &cs);
        nd[A_VV] = v;
        nd[A_EF] = make_double2(v.x * cs, v.x * sn);
      }
    }
    grp_sync<G>(gidx);
    first = false;
    PROF(6)
  }
  return done;
}

// ------------------------------------------------------------------------------------------
// Fallback for meshed networks: the same Newton-Raphson (same unknowns, same iterates up to rounding),
// but the Jacobian is assembled dense ([2 npq] x [2 npq], row-major, unknown 2i = dtheta_i, 2i+1 = dV_i/V_i)
// in a global-memory workspace and solved by one warp with partial-pivoting LU (what SuperLU does for
// pandapower). O(npq^3) per solve: meant for small meshed feeders, not for the radial hot path.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ bool nr_solve_dense(const Params& p, const Hot& h, const Slab& s, double* __restrict__ ws,
                                               int lane, bool skip, int& iters) {
  const int npq = p.npq, m = 2 * npq, ld = m + 1;       // column m holds the right-hand side
  for (int i = lane; i <= npq + 1; i += 32) {
    const bool sl = (i == npq);
    double2* nd = s.node(i);
    nd[A_VV] = sl ? make_double2(p.vm0, p.va0) : make_double2(p.vm_init, 0.0);
    nd[A_EF] = sl ? make_double2(p.e0, p.f0) : make_double2(p.vm_init, 0.0);
    nd[A_UP] = make_double2(0.0, 0.0); nd[A_DN] = make_double2(0.0, 0.0); nd[A_T] = make_double2(0.0, 0.0);
    nd[A_R] = make_double2(0.0, 0.0);
  }
  __syncwarp();
  bool done = skip;
  int it = 0;
  iters = 0;
  const double2 v0 = make_double2(p.e0, p.f0);
  while (true) {
    for (int idx = lane; idx < m * ld; idx += 32) ws[idx] = 0.0;
    __syncwarp();
    // mismatch + Jacobian rows of bus i (SURVEY A.4 formulas, unknown dV/V)
    double nrm = 0.0;
    for (int i = lane; i < npq; i += 32) {
      const double2 vi = s.node(i)[A_EF];
      const double2 ys = h.ysl[i], yi = h.yii[i], sp = s.node(i)[A_SP];
      const double cs0 = vi.x * v0.x + vi.y * v0.y, sn0 = vi.y * v0.x - vi.x * v0.y;
      double sa = ys.x * sn0 - ys.y * cs0, sb = ys.x * cs0 + ys.y * sn0;
      double* rp = ws + static_cast<size_t>(2 * i) * ld;
      double* rq = rp + ld;
      for (int t = h.nbr_ptr[i], te = h.nbr_ptr[i + 1]; t < te; ++t) {
        const int j = h.nbr_idx[t];
        const double2 y = h.nbr_y[t], vj = s.node(j)[A_EF];
        const double cc = vi.x * vj.x + vi.y * vj.y, ss = vi.y * vj.x - vi.x * vj.y;
        const double a = y.x * ss - y.y * cc, b = y.x * cc + y.y * ss;
        sa += a; sb += b;
        rp[2 * j] = a; rp[2 * j + 1] = b; rq[2 * j] = -b; rq[2 * j + 1] = a;
      }
      const double vv = vi.x * vi.x + vi.y * vi.y;
      const double gv = yi.x * vv, bv = yi.y * vv;
      const double P = gv + sb, Q = sa - bv;
      const double Fp = P - sp.x, Fq = Q - sp.y;
      rp[2 * i] = -Q - bv; rp[2 * i + 1] = P + gv; rq[2 * i] = P - gv; rq[2 * i + 1] = Q - bv;
      rp[m] = -Fp; rq[m] = -Fq;
      nrm = nanmax(nrm, nanmax(fabs(Fp), fabs(Fq)));
    }
    const bool ok = __all_sync(kFull, nrm < p.tol);
    if (!done && ok) { done = true; iters = it; }
    if (done || it >= p.max_iter) break;
    ++it;
    __syncwarp();
    // LU with partial pivoting, right-looking, rhs carried as column m
    bool singular = false;
    for (int k = 0; k < m; ++k) {
      double best = -1.0; int brow = k;
      for (int r = k + lane; r < m; r += 32) { const double v = fabs(ws[static_cast<size_t>(r) * ld + k]); if (v > best) { best = v; brow = r; } }
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) {
        const double ob = __shfl_xor_sync(kFull, best, o); const int orow = __shfl_xor_sync(kFull, brow, o);
        if (ob > best || (ob == best && orow < brow)) { best = ob; brow = orow; }
      }
      if (!(best > 0.0)) { singular = true; break; }
      if (brow != k)
        for (int c = k + lane; c <= m; c += 32) {
          const double t0 = ws[static_cast<size_t>(k) * ld + c];
          ws[static_cast<size_t>(k) * ld + c] = ws[static_cast<size_t>(brow) * ld + c];
          ws[static_cast<size_t>(brow) * ld + c] = t0;
        }
      __syncwarp();
      const double pinv = 1.0 / ws[static_cast<size_t>(k) * ld + k];
      for (int r = k + 1; r < m; ++r) {
        const double l = ws[static_cast<size_t>(r) * ld + k] * pinv;     // same value in every lane (broadcast load)
        if (l != 0.0)
          for (int c = k + 1 + lane; c <= m; c += 32) ws[static_cast<size_t>(r) * ld + c] -= l * ws[static_cast<size_t>(k) * ld + c];
      }
      __syncwarp();
    }
    if (singular) { done = false; break; }
    // back substitution; dx of bus i goes to its record (R)
    for (int k = m - 1; k >= 0; --k) {
      double acc = 0.0;
      for (int c = k + 1 + lane; c < m; c += 32) acc += ws[static_cast<size_t>(k) * ld + c] * ws[static_cast<size_t>(c) * ld + m];
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
      if (lane == 0) ws[static_cast<size_t>(k) * ld + m] = (ws[static_cast<size_t>(k) * ld + m] - acc) / ws[static_cast<size_t>(k) * ld + k];
      __syncwarp();
    }
    for (int i = lane; i < npq; i += 32) {
      double2* nd = s.node(i);
      double2 v = nd[A_VV];
      v.y += ws[static_cast<size_t>(2 * i) * ld + m];
      v.x += v.x * ws[static_cast<size_t>(2 * i + 1) * ld + m];
      double sn, cs;
      sincos_angle(v.y, &sn, &cs);
      nd[A_VV] = v;
      nd[A_EF] = make_double2(v.x * cs, v.x * sn);
    }
    __syncwarp();
  }
  return done;
}

// Piece-wise linear q(v) of the droop baseline: reference traditional_control/pf_droop_matpower_all.m:196-231
// (saturation at va = 0.95 / vd = 1.05, dead band collapsed at vb = vc = 1.0, q_max = min(sqrt(S^2 - p^2), q_max_manual))
__device__ __forceinline__ double droop_q(double pv, double s_rated, double v, double qmm) {
  const double va = 0.95, vb = 1.0, vc = 1.0, vd = 1.05;
  const double q_max = fmin(sqrt(s_rated * s_rated - pv * pv), qmm);
  if (v <= va) return q_max;
  if (v > vd) return -q_max;
  if (v >= vb && v <= vc) return 0.0;
  if (v < vb) return (q_max - 0.0) / (va - vb) * (v - vb);
  return (0.0 - q_max) / (vc - vd) * (vc - v);
}

// sgen.q_mvar from an action: reference _clip_reactive_power :568-572
__device__ __forceinline__ double clip_q(double a, double pv, double smax) {
  return sqrt(smax * smax - pv * pv) * a;
}

template <int G, int MODE, bool DENSE = false>
__global__ void __launch_bounds__(G > 32 ? 640 : 384) env_kernel(const __grid_constant__ Params p) {
  static_assert(!DENSE || G == 32, "the dense fallback uses one warp per env");
  static_assert(G == 4 || G == 8 || G == 16 || G == 32 || G == 64 || G == 128, "unsupported group size");
#ifdef MAPDN_HOST_EMU
  unsigned char* const smem_raw = emu::dyn_smem();
#else
  extern __shared__ __align__(16) unsigned char smem_raw[];
#endif
  __shared__ __align__(8) uint64_t stage_bar;
  PROF_DECL
  stage_hot_issue(smem_raw, p.hot, p.hot_layout.bytes, &stage_bar);
  bool hot_ready = false;     // the wait is deferred until the first use, behind the prologue's global loads

  const HotLayout& hl = p.hot_layout;
  Hot h;
  h.yup = reinterpret_cast<const double2*>(smem_raw + hl.yup);
  h.ydn = reinterpret_cast<const double2*>(smem_raw + hl.ydn);
  h.yii = reinterpret_cast<const double2*>(smem_raw + hl.yii);
  h.ndesc = reinterpret_cast<const uint64_t*>(smem_raw + hl.ndesc);
  h.esched = reinterpret_cast<const uint64_t*>(smem_raw + hl.esched);
  h.bsched = reinterpret_cast<const uint64_t*>(smem_raw + hl.bsched);
  h.lptr = reinterpret_cast<const uint16_t*>(smem_raw + hl.lptr);
  h.lidx = reinterpret_cast<const uint16_t*>(smem_raw + hl.lidx);
  h.sptr = reinterpret_cast<const uint16_t*>(smem_raw + hl.sptr);
  h.sidx = reinterpret_cast<const uint16_t*>(smem_raw + hl.sidx);
  h.xptr = reinterpret_cast<const uint16_t*>(smem_raw + hl.xptr);
  h.xidx = reinterpret_cast<const uint16_t*>(smem_raw + hl.xidx);
  h.node_of_bus = reinterpret_cast<const uint16_t*>(smem_raw + hl.node_of_bus);
  h.ysl = hl.tables_in_blob ? reinterpret_cast<const double2*>(smem_raw + hl.ysl) : p.ysl;
  h.in_blob = hl.tables_in_blob != 0;
  h.blob = smem_raw;
#ifndef MAPDN_HOST_EMU
  if (!hl.tables_in_blob) {      // L2 was possibly flushed: fetch the cold tables now, long before the epilogue needs them
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int k = tid * 128; k < 2 * p.n_sgen * p.obs_dim; k += nt * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(p.obs_off) + k));
    for (int k = tid * 128; k < 4 * p.n_line; k += nt * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(p.line_nodes) + k));
    for (int k = tid * 128; k < 32 * p.n_line; k += nt * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(p.line_c) + k));
    for (int k = tid * 128; k < 16 * p.npq; k += nt * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(p.ysl) + k));
  }
#endif
#ifndef MAPDN_HOST_EMU
  if (!DENSE) {   // the factors of the static first Newton iteration (96 B per bus, read by every solve's flat-start pass): after an
                  // L2 flush their first touch would be a chain of DRAM round trips in front of the first sweep - fetch them
                  // into L2 now, behind the prologue
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int k = tid * 128; k < 96 * p.npq; k += nt * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(p.first_tab) + k));
  }
#endif
  h.nbr_ptr = reinterpret_cast<const uint16_t*>(smem_raw + hl.nbr_ptr);
  h.nbr_idx = reinterpret_cast<const uint16_t*>(smem_raw + hl.nbr_idx);
  h.nbr_y = reinterpret_cast<const double2*>(smem_raw + hl.nbr_y);

  // MODE_STEP: the last warp of the CTA is a helper that draws the next profile rows (+ noise) of the CTA's
  // envs while the solver warps run the Newton iteration (the two only meet at two named barriers)
  const int n_helper_threads = (MODE == MODE_STEP) ? p.helper_threads : 0;
  const int n_solver_threads = blockDim.x - n_helper_threads;
  const bool is_helper = (MODE == MODE_STEP) && threadIdx.x >= n_solver_threads;
  const int hl_bytes = p.hot_layout.bytes;
  const int gl = threadIdx.x % G;
  const int gidx = is_helper ? 0 : threadIdx.x / G;
  const int epb = n_solver_threads / G;
  const int npq = p.npq, n = p.n_bus, nl = p.n_load, ng = p.n_sgen;
  Slab s;
  {
    double2* base = reinterpret_cast<double2*>(smem_raw + hl.bytes) + static_cast<size_t>(gidx) * p.env_stride2;
    s.nodes = base;
    s.base = reinterpret_cast<double*>(base);
    s.pv = reinterpret_cast<double*>(base + p.pvq_off2);
    s.q = s.pv + ng;
    s.scratch = reinterpret_cast<double*>(base + p.scratch_off2);
  }
  // scratch: [0, n_sgen) the helper warps' new sgen.p_mw (MODE_STEP) / the previous PV-bus voltages (MODE_DROOP), then the
  // per-warp partials of the multi-warp group reductions, then - only when they do not fit there - the staged loads.
  // Staged (scaled) load p / q of the prologue, 2 n_load doubles: they normally live in the Newton fields of the node
  // records (UP .. R = 12 contiguous doubles per record), which are dead until the flat start overwrites them.
  double* next_row = s.scratch;
  double* red_scratch = s.scratch + ng;
  const bool stage_rec = p.stage_in_records != 0;
  double* stage_lin = s.scratch + ng + (G > 32 ? 10 * (G / 32) : 0);
  const uint32_t k0 = static_cast<uint32_t>(p.seed), k1 = static_cast<uint32_t>(p.seed >> 32);

  for (int base = blockIdx.x * epb; base < p.nb; base += gridDim.x * epb) {
    if (is_helper) {
      // ---- helper warps: next profile row of every env of this round (reference _set_demand_and_pv :491-513:
      //      t = self.steps before the increment) + |N(0,1)| * std noise in Box-Muller pairs (2m, 2m+1) over the
      //      elements [pv | load_p | load_q]; new pv goes to the env's scratch (for the obs), loads straight to HBM.
      //      Two dependent global round trips in total: (A) the per-env scalars of the whole round -> shared memory,
      //      (B) the profile values, four work items per thread in flight, addresses selected without branches. ----
      const int n_elem = ng + 2 * nl, n_pair = (n_elem + 1) / 2, n_work = epb * n_pair;
      const int ht = threadIdx.x - n_solver_threads, T = n_helper_threads;
      int4* hs = reinterpret_cast<int4*>(smem_raw + p.helper_off);     // per env: (row lo, row hi, steps, episode)
#ifdef MAPDN_HOST_EMU
      emu::bar_sync(15, T);
#else
      asm volatile("bar.sync 15, %0;" ::"r"(T) : "memory");     // helper threads only: the previous round's reads of hs are done
#endif
      for (int e = ht; e < epb; e += T) {
        const int env_h = base + e;
        int4 v = make_int4(0, 0, 0, 0);
        if (env_h < p.nb) {
          const int steps_h = p.steps[env_h];
          long long nrow = p.start_row[env_h] + steps_h;
          if (nrow > p.n_rows - 1) nrow = p.n_rows - 1;
          v = make_int4(static_cast<int>(nrow & 0xFFFFFFFFll), static_cast<int>(nrow >> 32), steps_h,
                        static_cast<int>(p.episode[env_h]));
        }
        hs[e] = v;
      }
#ifdef MAPDN_HOST_EMU
      emu::bar_sync(15, T);
#else
      asm volatile("bar.sync 15, %0;" ::"r"(T) : "memory");     // helper threads only
#endif
      named_bar_sync(1, blockDim.x);                   // the solvers have read the current rows
      constexpr int U = 4;
      for (int w0 = ht; w0 < n_work; w0 += U * T) {
        double val[U][2], sd[U][2];
        int e_[U], m_[U];
        bool ok[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int w = w0 + u * T;
          ok[u] = w < n_work;
          const int e = ok[u] ? w / n_pair : 0;
          e_[u] = e; m_[u] = w - e * n_pair;
          ok[u] = ok[u] && (base + e < p.nb);
          const int4 sc = hs[e];
          const long long nrow = (static_cast<long long>(sc.y) << 32) | static_cast<unsigned>(sc.x);
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int el = min(2 * m_[u] + k, n_elem - 1);          // an odd n_elem re-reads the last element (not stored)
            const bool is_pv = el < ng, is_lp = el < ng + nl;
            const int j = is_pv ? el : (is_lp ? el - ng : el - ng - nl);
            const double* src = is_pv ? p.prof_pv + nrow * ng : (is_lp ? p.prof_lp + nrow * nl : p.prof_lq + nrow * nl);
            const double* sds = is_pv ? p.pv_std : (is_lp ? p.lp_std : p.lq_std);
            val[u][k] = ok[u] ? __ldg(src + j) : 0.0;
            sd[u][k] = ok[u] ? __ldg(sds + j) : 0.0;
          }
        }
        // one copy of Philox + log + sqrt + sincos (not four: the solver warps need the instruction cache); the work
        // item is picked out of the registers with select chains
#pragma unroll 1
        for (int u = 0; u < U; ++u) {
          bool oku = ok[0]; int e = e_[0], m = m_[0];
          double va = val[0][0], vb = val[0][1], sa = sd[0][0], sb = sd[0][1];
#pragma unroll
          for (int q = 1; q < U; ++q)
            if (u == q) { oku = ok[q]; e = e_[q]; m = m_[q]; va = val[q][0]; vb = val[q][1]; sa = sd[q][0]; sb = sd[q][1]; }
          if (!oku) continue;
          const int env_h = base + e;
          const int4 sc = hs[e];
          RngKey key_h{k0, k1, static_cast<uint32_t>(p.env_id_offset + env_h), static_cast<uint32_t>(sc.w) * 8u};
          double z0 = 0.0, z1 = 0.0;
          if (p.add_noise) half_normal_pair(key_h, static_cast<uint32_t>(sc.z), m, z0, z1);
          double* pv_next = reinterpret_cast<double*>(reinterpret_cast<double2*>(smem_raw + hl_bytes) +
                                                       static_cast<size_t>(e) * p.env_stride2 + p.scratch_off2);
          const size_t hL = static_cast<size_t>(env_h) * nl, hG = static_cast<size_t>(env_h) * ng;
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int el = 2 * m + k;
            if (el >= n_elem) break;
            const double v = (k == 0) ? va + sa * z0 : vb + sb * z1;
            const bool is_pv = el < ng, is_lp = el < ng + nl;
            double* dst = is_pv ? p.cur_pv + hG + el : (is_lp ? p.cur_pl + hL + (el - ng) : p.cur_ql + hL + (el - ng - nl));
            *dst = v;
            if (is_pv) pv_next[el] = v;
          }
        }
      }
      named_bar_arrive(2, blockDim.x);                 // new pv of every env is in shared memory
      continue;
    }
    int env = base + gidx;
    bool valid = env < p.nb;
    if (!valid) env = p.nb - 1;
    if (MODE == MODE_RESET && p.mask != nullptr && !p.mask[env]) valid = false;
    const size_t eL = static_cast<size_t>(env) * nl, eG = static_cast<size_t>(env) * ng,
                 eN = static_cast<size_t>(env) * n;

    RngKey key{k0, k1, static_cast<uint32_t>(p.env_id_offset + env), 0u};
    long long start = 0;
    int steps_old = 0;
    // (groups beyond the batch work on a clamped env id without storing anything: they must not read the scalars that the
    // env's real group rewrites at the end of its step / reset - a benign race, but a race)
    if (MODE == MODE_STEP && valid) {
      key.c3base = p.episode[env] * 8u;
      start = p.start_row[env];
      steps_old = p.steps[env];
    }
    if (MODE == MODE_RESET && valid) key.c3base = (p.episode[env] + 1u) * 8u;

    bool conv = false;
    int iters = 0;
    int attempt = 0;
    bool solved = false;
    bool dr_active = valid;      // MODE_DROOP: this env has not met the stopping rule yet
    int dr_iters = 0;
    double* v_last = s.scratch;                    // MODE_DROOP: PV-bus voltages of the previous power flow [n_sgen]
    const int n_rounds = (MODE == MODE_RESET) ? kMaxResetAttempts : (MODE == MODE_DROOP ? p.droop_max_ite : 1);
    for (int round = 0; round < n_rounds; ++round) {
      // ---------------- prologue: element values -> sgen p/q and bus injections ----------------
      if (MODE == MODE_RESET) {
        int day, hour, interval;
        if (p.start_dhi != nullptr) {                               // manual_reset :137-152
          day = p.start_dhi[env * 3 + 0]; hour = p.start_dhi[env * 3 + 1]; interval = p.start_dhi[env * 3 + 2];
        } else {                                                    // :111-113, :381-398
          const u32x4 r = philox4x32_10(0u, static_cast<uint32_t>(attempt), key.env, key.c3base + kStreamTime, k0, k1);
          hour = static_cast<int>(__umulhi(r.x, 24u));
          day = static_cast<int>(__umulhi(r.y, static_cast<uint32_t>(p.n_day_choices)));
          interval = static_cast<int>(__umulhi(r.z, static_cast<uint32_t>(p.steps_per_hour)));
        }
        start = interval + static_cast<long long>(hour) * p.steps_per_hour +
                static_cast<long long>(day) * 24 * p.steps_per_hour;          // :445
        // a manual start outside the store is clamped to the last window that fits (the host shims validate and
        // raise; the kernel only guarantees in-bounds reads)
        start = max(0ll, min(start, p.n_rows - 1 - p.episode_limit));
      }
      long long row = 0;
      if (MODE == MODE_RESET) { row = start + 1; if (row > p.n_rows - 1) row = p.n_rows - 1; }   // t = steps = 1
      const uint32_t c1 = kResetFlag | static_cast<uint32_t>(attempt);
      // (1) coalesced, independent loads of the env's element values into shared memory
      if (MODE != MODE_DROOP || round == 0) {          // droop: later rounds only change q (in shared memory)
#pragma unroll 4
      for (int j = gl; j < ng; j += G) {
        double pv, q;
        if (MODE == MODE_SOLVE || MODE == MODE_DROOP) {
          pv = p.in_pv[eG + j]; q = (MODE == MODE_SOLVE) ? p.in_q[eG + j] : 0.0;     // droop starts from q = 0 (:107)
          if (MODE == MODE_DROOP) v_last[j] = 100.0;                                    // :123
        } else if (MODE == MODE_STEP) {
          pv = p.cur_pv[eG + j];
          q = clip_q(p.actions[eG + j], pv, __ldg(p.s_max + j));             // :553
        } else {
          pv = __ldg(p.prof_pv + row * ng + j);
          if (p.add_noise) pv += __ldg(p.pv_std + j) * half_normal(key, c1, j);   // :498
          q = 0.0;
          if (p.reset_action) {                                               // :120-122, :334-338
            const u32x4 r = philox4x32_10(j, static_cast<uint32_t>(attempt), key.env, key.c3base + kStreamAction, k0, k1);
            const double a = p.action_low + (p.action_high - p.action_low) * u53(r.x, r.y);
            q = clip_q(a, pv, __ldg(p.s_max + j));
          }
          if (valid) p.cur_pv[eG + j] = pv;
        }
        s.pv[j] = pv; s.q[j] = q;
      }
      }
      // (droop re-stages the loads every round: the staging area is overwritten by the Newton iteration)
      // Written once, instantiated for the two staging places (block-uniform choice): a branch per access inside the
      // loops would cost time in every step.
      auto stage_and_gather = [&](auto stg) {
#pragma unroll 4
        for (int l = gl; l < nl; l += G) {
          double pl, ql;
          if (MODE == MODE_SOLVE || MODE == MODE_DROOP) { pl = p.in_pl[eL + l]; ql = p.in_ql[eL + l]; }
          else if (MODE == MODE_STEP) { pl = p.cur_pl[eL + l]; ql = p.cur_ql[eL + l]; }
          else {
            pl = __ldg(p.prof_lp + row * nl + l);
            ql = __ldg(p.prof_lq + row * nl + l);
            if (p.add_noise) {                                                   // :503, :508
              pl += __ldg(p.lp_std + l) * half_normal(key, c1, ng + l);
              ql += __ldg(p.lq_std + l) * half_normal(key, c1, ng + nl + l);
            }
            if (valid) { p.cur_pl[eL + l] = pl; p.cur_ql[eL + l] = ql; }
          }
          const double sc = __ldg(p.lscale + l);
          *stg(l) = pl * sc; *stg(nl + l) = ql * sc;
        }
        if (!hot_ready) { stage_hot_wait(&stage_bar); hot_ready = true; }
        grp_sync<G>(gidx);
        // (2) A.1: PD/QD per bus, Sbus = -(PD + jQD)/baseMVA
        for (int i = gl; i < npq; i += G) {
          double pd = 0.0, qd = 0.0;
#pragma unroll 1
          for (int t = h.lptr[i], te = h.lptr[i + 1]; t < te; ++t) { const int l = h.lidx[t]; pd += *stg(l); qd += *stg(nl + l); }
#pragma unroll 1
          for (int t = h.sptr[i], te = h.sptr[i + 1]; t < te; ++t) {
            const int g = h.sidx[t];
            const double sc = __ldg(p.sscale + g);
            pd -= s.pv[g] * sc; qd -= s.q[g] * sc;
          }
          s.node(i)[A_SP] = make_double2(-pd * p.inv_base, -qd * p.inv_base);
        }
      };
      if (stage_rec) stage_and_gather([&](int k) -> double* { return s.base + (k / 12) * (2 * kNodeArrays2) + 2 * A_UP + (k % 12); });
      else stage_and_gather([&](int k) -> double* { return stage_lin + k; });
      grp_sync<G>(gidx);
      if (MODE == MODE_STEP) named_bar_arrive(1, blockDim.x);   // the current rows are consumed: the helper may overwrite them

      // ---------------- Newton-Raphson ----------------
      PROF(1)
      if (DENSE) {
        double* ws = p.dense_ws + (static_cast<size_t>(blockIdx.x) * epb + gidx) * p.dense_stride;
        conv = nr_solve_dense(p, h, s, ws, gl, !valid, iters);
      } else {
#ifdef MAPDN_PROFILE
        conv = nr_solve<G>(p, h, s, gidx, gl, !valid, iters, _acc, _pt);
#else
        conv = nr_solve<G>(p, h, s, gidx, gl, !valid, iters);
#endif
      }
      PROF(4)
      if (MODE == MODE_DROOP) {
        // relaxed fixed-point loop of pf_droop_matpower_all.m:121-152: stop when ||v_pv - v_pv_last||_2 < tol, else
        // q <- (1 - gain) q + gain q_droop(v). An env that has stopped keeps its q, so the power flows it still runs
        // alongside the others of its warp reproduce its final state; the last allowed round does not move q either
        // (the script reports the q of the last power flow).
        double part[1] = {0.0};
        const bool no_max[1] = {false};
        for (int j = gl; j < ng; j += G) {
          const double dv = v_last[j] - s.node(__ldg(p.sgen_node + j))[A_VV].x;
          part[0] += dv * dv;
        }
        grp_reduce<G, 1>(gidx, gl, part, no_max, red_scratch);
        const bool stop = sqrt(part[0]) < p.droop_tol;
        if (dr_active) { dr_iters = round + 1; if (stop) dr_active = false; }
        if (grp_exit<G>(!dr_active) || round == n_rounds - 1) break;
        if (dr_active) {
          for (int j = gl; j < ng; j += G) {
            const double v = s.node(__ldg(p.sgen_node + j))[A_VV].x;
            v_last[j] = v;
            const double q_new = droop_q(s.pv[j], __ldg(p.droop_s + j), v, __ldg(p.droop_qmm + j));
            s.q[j] = (1.0 - p.droop_gain) * s.q[j] + p.droop_gain * q_new;
          }
        }
        grp_sync<G>(gidx);
        continue;
      }
      if (MODE != MODE_RESET) break;
      if (conv) solved = true;
      if (grp_exit<G>(solved)) break;
      if (!solved) ++attempt;                       // re-draw this env (reference retry loop :108-133)
      grp_sync<G>(gidx);
    }

    // ---------------- epilogue ----------------
    // divergence branch (reference :188-196): fall back to the previous solution kept in HBM
    if (MODE == MODE_STEP && !conv) {
      for (int i = gl; i < npq; i += G) {
        const int b = __ldg(p.bus_of_node + i);
        const double vm = p.res_vm[eN + b], va = p.res_va[eN + b];
        double sn, cs;
        sincos(va, &sn, &cs);
        double2* nd = s.node(i);
        nd[A_VV] = make_double2(vm, va);
        nd[A_EF] = make_double2(vm * cs, vm * sn);
        nd[A_SP] = make_double2(-p.res_p[eN + b] * p.inv_base, -p.res_q[eN + b] * p.inv_base);
      }
    }
    grp_sync<G>(gidx);
    // a reset whose kMaxResetAttempts draws all diverged keeps the env's previous state and reports it (reset_ok)
    constexpr bool kExplicit = (MODE == MODE_SOLVE || MODE == MODE_DROOP);     // explicit inputs / outputs, no env state
    const bool write_res = valid && (kExplicit || conv);
    if (MODE == MODE_RESET && valid && gl == 0 && p.reset_ok != nullptr) p.reset_ok[env] = conv ? 1 : 0;
    if (!kExplicit && valid && gl == 0) p.nr_iters[env] = conv ? iters : p.max_iter;

    // slack injection (pfsoln, SURVEY A.5): S0 = V0 conj(Ybus[0,:] V) -> sentinel record's SP
    {
      const double vv = p.vm0 * p.vm0;
      double P0 = p.ysl_g0 * vv, Q0 = -p.ysl_b0 * vv;
      for (int k = 0; k < p.n_slack_adj; ++k) {
        const int i = __ldg(p.sl_node + k);
        const double g = __ldg(p.sl_y + 2 * k), b = __ldg(p.sl_y + 2 * k + 1);
        const double2 vi = s.node(i)[A_EF];
        const double cc = p.e0 * vi.x + p.f0 * vi.y, ss = p.f0 * vi.x - p.e0 * vi.y;   // V0 Vi cos/sin(t0 - ti)
        P0 += g * cc + b * ss;
        Q0 += g * ss - b * cc;
      }
      if (gl == 0) s.node(npq)[A_SP] = make_double2(P0, Q0);
    }
    PROF(7)
    // sgen.q_mvar after the step: the clipped action, or the previous q on divergence (:189-196)
    double sum_q_eff = 0.0, sum_q_try = 0.0;
    if (MODE == MODE_STEP) {
      for (int j = gl; j < ng; j += G) {
        const double q_try = s.q[j];
        const double q_eff = conv ? q_try : p.cur_q[eG + j];
        sum_q_try += fabs(q_try);
        sum_q_eff += fabs(q_eff * __ldg(p.sscale + j));     // res_sgen.q_mvar = q * scaling (:604-605)
        s.q[j] = q_eff;
        if (write_res) p.cur_q[eG + j] = q_eff;
      }
    }
    // the helper warp has drawn the next profile row meanwhile: take over the new sgen.p_mw (Appendix B.3: the
    // observation mixes this solve's bus results with the NEXT row's PV)
    if (MODE == MODE_STEP) {
      named_bar_sync(2, blockDim.x);
      for (int j = gl; j < ng; j += G) s.pv[j] = next_row[j];
    }
    grp_sync<G>(gidx);
    PROF(8)
    // res_bus columns per node (BP) and the "demand" columns of get_obs (OP = BP + sgens of the bus's own zone)
    for (int i = gl; i <= npq; i += G) {
      double2* nd = s.node(i);
      const double2 sp = nd[A_SP];
      double2 bp = make_double2(-sp.x * p.base_mva, -sp.y * p.base_mva);
      if (p.has_shunt) {                   // warp-uniform; pandapower adds the bus shunts' p/q (x vm^2) to res_bus
        const double2 ef = nd[A_EF];
        const double v2 = ef.x * ef.x + ef.y * ef.y;
        bp.x += __ldg(p.sh_g + i) * v2; bp.y -= __ldg(p.sh_b + i) * v2;
      }
      double2 op = bp;
#pragma unroll 1
      for (int t = h.xptr[i], te = h.xptr[i + 1]; t < te; ++t) { const int g = h.xidx[t]; op.x += s.pv[g]; op.y += s.q[g]; }
      nd[A_BP] = bp; nd[A_OP] = op;
    }
    grp_sync<G>(gidx);
    // per-bus results + voltage statistics (reference _calc_reward :584-596, :610)
    double cnt_lo = 0, cnt_hi = 0, sum_dev = 0, sum_v = 0, max_drop = 0, max_rise = 0, sum_bar = 0;
    const double v_ref = 0.5 * (p.v_lower + p.v_upper);
#pragma unroll 4
    for (int b = gl; b < n; b += G) {
      const double2* nd = s.node(h.node_of_bus[b]);
      const double2 vv = nd[A_VV], bp = nd[A_BP];
      const double v = vv.x, th = vv.y;
      if (kExplicit) {
        if (valid) {
          if (p.out_vm) p.out_vm[eN + b] = v;
          if (p.out_va) p.out_va[eN + b] = th * kRad2Deg;
          if (p.out_p) p.out_p[eN + b] = bp.x;
          if (p.out_q) p.out_q[eN + b] = bp.y;
        }
      } else {
        if (write_res) {
          p.res_vm[eN + b] = v; p.res_va[eN + b] = th; p.res_p[eN + b] = bp.x; p.res_q[eN + b] = bp.y;
        }
        if (MODE == MODE_STEP) {
          cnt_lo += (v < p.v_lower) ? 1.0 : 0.0;
          cnt_hi += (v > p.v_upper) ? 1.0 : 0.0;
          sum_dev += fabs(v - v_ref);
          sum_v += v;
          max_drop = fmax(max_drop, (v < p.v_lower) ? (p.v_lower - v) : 0.0);
          max_rise = fmax(max_rise, (v > p.v_upper) ? (v - p.v_upper) : 0.0);
          sum_bar += barrier_fn(p.barrier, v);
        }
      }
    }
    // line losses: res_line.pl_mw = Re(Sf + St) (SURVEY A.5), 4 static coefficients per line. The two tables are either
    // part of the staged blob (LDS) or cold in global memory (read-only path): one block-uniform branch, two typed loops.
    double sum_pl = 0.0;
    {
      const size_t ePL = static_cast<size_t>(env) * p.n_line;
      auto lines = [&](const ushort2* __restrict__ ln, const double2* __restrict__ lc) {
#pragma unroll 4
        for (int k = gl; k < p.n_line; k += G) {
          const ushort2 ft = ln[k];
          const double2 vf = s.node(ft.x)[A_EF], vt = s.node(ft.y)[A_EF];
          const double cc = vf.x * vt.x + vf.y * vt.y, ss = vf.y * vt.x - vf.x * vt.y;
          const double2 c01 = lc[2 * k], c23 = lc[2 * k + 1];
          const double pl = c01.x * (vf.x * vf.x + vf.y * vf.y) + c01.y * (vt.x * vt.x + vt.y * vt.y) + c23.x * cc + c23.y * ss;
          sum_pl += pl;
          if (kExplicit) { if (valid && p.out_pl) p.out_pl[ePL + k] = pl; }
          else if (write_res) p.res_pl[ePL + k] = pl;
        }
      };
      if (h.in_blob) lines(reinterpret_cast<const ushort2*>(smem_raw + hl.line_nodes), reinterpret_cast<const double2*>(smem_raw + hl.line_c));
      else lines(reinterpret_cast<const ushort2*>(p.line_nodes), reinterpret_cast<const double2*>(p.line_c));
    }
    PROF(9)
    if (kExplicit) {
      if (MODE == MODE_DROOP) {
        double tot[1] = {sum_pl};
        const bool no_max[1] = {false};
        grp_reduce<G, 1>(gidx, gl, tot, no_max, red_scratch);
        if (valid) {
          for (int j = gl; j < ng; j += G) p.droop_q_out[eG + j] = s.q[j];
          if (gl == 0) { p.droop_loss_out[env] = tot[0]; p.out_iters[env] = dr_iters; }
        }
      }
      if (valid && gl == 0) {
        if (MODE == MODE_SOLVE && p.out_iters) p.out_iters[env] = conv ? iters : p.max_iter;
        if (p.out_conv) p.out_conv[env] = conv ? 1 : 0;
      }
      grp_sync<G>(gidx);
      continue;
    }

    if (MODE == MODE_STEP) {
      {
        double rv[10] = {cnt_lo, cnt_hi, sum_dev, sum_v, sum_bar, max_drop, max_rise, sum_pl, sum_q_eff, sum_q_try};
        const bool rmax[10] = {false, false, false, false, false, true, true, false, false, false};
        grp_reduce<G, 10>(gidx, gl, rv, rmax, red_scratch);
        cnt_lo = rv[0]; cnt_hi = rv[1]; sum_dev = rv[2]; sum_v = rv[3]; sum_bar = rv[4];
        max_drop = rv[5]; max_rise = rv[6]; sum_pl = rv[7]; sum_q_eff = rv[8]; sum_q_try = rv[9];
      }
      const double inv_n = 1.0 / n;
      const double pct = (cnt_lo + cnt_hi) * inv_n;
      const double q_loss = sum_q_eff / ng;
      const double v_loss = sum_bar * inv_n * p.voltage_weight;
      const double loss = p.use_line_weight ? (sum_pl / p.n_line) * p.line_weight + v_loss
                                            : q_loss * p.q_weight + v_loss;     // :612-618
      double reward = -loss;
      if (!conv) reward -= 200.0;                                               // :192
      const int steps_new = steps_old + 1;                                      // :202
      if (valid && gl == 0) {
        p.reward[env] = reward;
        p.term[env] = (steps_new >= p.episode_limit || !conv) ? 1 : 0;          // :204
        p.steps[env] = steps_new;
        p.sum_rewards[env] += reward;                                           // :203
      }
      if (valid && p.info != nullptr) {
        // the 11 info scalars, one per lane (every lane of the group holds the reduced values): one or two store
        // instructions per env instead of eleven from lane 0 - it matters when `info` is pinned host memory
        double* o = p.info + static_cast<size_t>(env) * 11;
        const double i3 = (!conv || pct > 1e-3) ? 0.0 : 1.0;                     // :589, :195
        const double i9 = conv ? q_loss : sum_q_try / ng, i10 = conv ? 0.0 : 1.0;
        for (int k = gl; k < 11; k += G) {
          double v = pct;                                                         // select chain, no divergent branches
          v = (k == 1) ? cnt_lo * inv_n : v; v = (k == 2) ? cnt_hi * inv_n : v; v = (k == 3) ? i3 : v;
          v = (k == 4) ? sum_dev * inv_n : v; v = (k == 5) ? sum_v * inv_n : v; v = (k == 6) ? max_drop : v;
          v = (k == 7) ? max_rise : v; v = (k == 8) ? sum_pl : v; v = (k == 9) ? i9 : v; v = (k == 10) ? i10 : v;
          o[k] = v;
        }
      }
    } else {  // MODE_RESET
      for (int j = gl; j < ng; j += G) if (valid) p.cur_q[eG + j] = s.q[j];
      if (valid && gl == 0) {
        p.steps[env] = 1;                         // :100
        p.sum_rewards[env] = 0.0;                 // :101
        p.start_row[env] = start;
        p.episode[env] = p.episode[env] + 1u;
      }
    }
    PROF(10)
    // observations of the new state (reference get_obs :232-316): a pure gather - the program maps every entry to a
    // double inside this env's slab, or to a constant-zero slot for the padding. A lane copies 16 bytes per
    // instruction (two fp64 / four fp32 entries) and consecutive lanes consecutive 16-byte pieces, so one store
    // instruction writes 128 contiguous bytes per env (full lines when the destination is pinned host memory).
    // obs_skip_off: entries reading that slot (the padding) are not stored.
    if ((p.obs != nullptr || (MODE == MODE_STEP && p.obs32 != nullptr)) && valid) {
      const bool compact = p.obs_compact_len > 0;          // rows without the per-agent padding (staged host path)
      const int tot = compact ? p.obs_compact_len : ng * p.obs_dim;
      const int skip = p.obs_skip_off;
      auto gather = [&](const uint16_t* __restrict__ prog, auto cold) {   // prog: shared (blob) or global (cold copy: read-only path)
        constexpr bool kCold = decltype(cold)::value;
        int done_to = 0;
        if (p.obs != nullptr) {
          double* o = p.obs + static_cast<size_t>(env) * tot;
          if ((tot & 1) == 0 && (reinterpret_cast<uintptr_t>(p.obs) & 15) == 0) {
            const uint32_t* offv = reinterpret_cast<const uint32_t*>(prog);
            const int npair = tot >> 1;
#pragma unroll (kCold ? 8 : 4)
            for (int c = gl; c < npair; c += G) {
              const uint32_t w = kCold ? __ldg(offv + c) : offv[c];
              const int o0 = static_cast<int>(w & 0xFFFFu), o1 = static_cast<int>(w >> 16);
              const double v0 = s.base[o0], v1 = s.base[o1];
              if (o0 != skip && o1 != skip) *reinterpret_cast<double2*>(o + 2 * c) = make_double2(v0, v1);
              else { if (o0 != skip) o[2 * c] = v0; if (o1 != skip) o[2 * c + 1] = v1; }
            }
            done_to = tot;
          }
          for (int idx = done_to + gl; idx < tot; idx += G) {
            const int off = prog[idx];
            if (off != skip) o[idx] = s.base[off];
          }
        } else {
          float* o = p.obs32 + static_cast<size_t>(env) * tot;
          if ((tot & 3) == 0 && (reinterpret_cast<uintptr_t>(p.obs32) & 15) == 0) {
            const uint2* offv = reinterpret_cast<const uint2*>(prog);
            const int nquad = tot >> 2;
#pragma unroll (kCold ? 8 : 4)
            for (int c = gl; c < nquad; c += G) {
              const uint2 w = kCold ? __ldg(offv + c) : offv[c];
              const int o0 = static_cast<int>(w.x & 0xFFFFu), o1 = static_cast<int>(w.x >> 16);
              const int o2 = static_cast<int>(w.y & 0xFFFFu), o3 = static_cast<int>(w.y >> 16);
              const float v0 = static_cast<float>(s.base[o0]), v1 = static_cast<float>(s.base[o1]);
              const float v2 = static_cast<float>(s.base[o2]), v3 = static_cast<float>(s.base[o3]);
              if (o0 != skip && o1 != skip && o2 != skip && o3 != skip) *reinterpret_cast<float4*>(o + 4 * c) = make_float4(v0, v1, v2, v3);
              else {
                if (o0 != skip) o[4 * c] = v0; if (o1 != skip) o[4 * c + 1] = v1;
                if (o2 != skip) o[4 * c + 2] = v2; if (o3 != skip) o[4 * c + 3] = v3;
              }
            }
            done_to = tot;
          }
          for (int idx = done_to + gl; idx < tot; idx += G) {
            const int off = prog[idx];
            if (off != skip) o[idx] = static_cast<float>(s.base[off]);
          }
        }
      };
      if (h.in_blob && !compact) gather(reinterpret_cast<const uint16_t*>(smem_raw + hl.obs_off), std::false_type{});
      else gather(compact ? p.obs_compact_prog : p.obs_off, std::true_type{});
    }
    if (MODE == MODE_RESET && p.state != nullptr) {
      // get_state (:213-230): [P_bus | Q_bus | pv | q | vm | va(deg)] restricted to state_space (cold program)
      double* o = p.state + static_cast<size_t>(env) * p.state_dim;
      for (int idx = gl; idx < p.state_dim; idx += G) {
        const unsigned src = __ldg(p.state_src + idx);
        const int kind = static_cast<int>(src >> 28), ix = static_cast<int>(src & 0x0FFFFFFFu);
        double v = 0.0;
        if (kind == OBS_PBUS) v = s.node(h.node_of_bus[ix])[A_BP].x;
        else if (kind == OBS_QBUS) v = s.node(h.node_of_bus[ix])[A_BP].y;
        else if (kind == OBS_PV) v = s.pv[ix];
        else if (kind == OBS_QSG) v = s.q[ix];
        else if (kind == OBS_VM) v = s.node(h.node_of_bus[ix])[A_VV].x;
        else if (kind == OBS_VA_DEG) v = s.node(h.node_of_bus[ix])[A_VV].y * kRad2Deg;
        if (valid) o[idx] = v;
      }
    }
    grp_sync<G>(gidx);
    PROF(11)
  }
#ifdef MAPDN_PROFILE
  if (p.prof != nullptr && blockIdx.x == 0 && threadIdx.x == 0) for (int k = 0; k < 16; ++k) p.prof[k] = _acc[k];
#endif
  if (!hot_ready) stage_hot_wait(&stage_bar);   // never exit with the bulk copy still in flight
}

}  // namespace mapdn
