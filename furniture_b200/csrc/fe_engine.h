// fe_engine.h -- one mj_step for one environment, executed by one warp out of its shared-memory slice.
//
// This is the GPU-native replacement of the per-env MjSim.step() hot loop (reference call site
// furniture/env/furniture.py:2878-2879; the arithmetic is MuJoCo's mj_step, see DESIGN.md for the stage map):
//   fe_kin_smooth : forward kinematics over the fused link tree, link velocities, composite inertia (CRBA) of the
//                   robot block, spatial inertia of every free part, RNE bias wrench, actuation, qacc_smooth
//   fe_collide    : geom poses, broad phase over the compile-time pair list with the per-env contype/conaffinity
//                   masks, narrow phase (fe_collide.h), per-part finger/floor touch flags
//   fe_assemble   : contact / weld / joint-limit rows (impedance, regularisation R, reference acceleration aref)
//   fe_solve      : primal Newton solver with exact line search over elliptic friction cones (impratio scaling)
//   fe_integrate  : semi-implicit Euler with implicit joint damping, quaternion integration
// Solver coordinates z: robot joint accelerations, then for every free part the world-frame spatial acceleration
// [alpha; vdot_origin] (a fixed orthogonal change of variables of the part's qacc, so the Newton iterates coincide).
#pragma once
#include "../../include/furniture_b200.h"
#include "fe_collide.h"
#include "fe_model.h"
#include "fe_warp.h"

#define FE_MINVAL 1e-15f
#define FE_MINIMP 0.0001f
#define FE_MAXIMP 0.9999f
// Broad-phase result in the slice: per lane, its 64-bit hit mask over its range of the pair list (two words) and the scan
// offset of its first hit.  Any number of candidates fits; the narrow phase recovers candidate i from the owning lane's mask.
#define FE_CAND_WORDS (3 * 32)
static_assert(FE_MAXPAIR <= 32 * 64, "a broad-phase lane holds at most 64 pairs in its hit mask");
// Line search: stop when |p'(alpha)| <= FE_LS_TOL |p'(0)|.  MuJoCo's default ls_tolerance is 0.01; the Newton loop's own
// stopping test decides the final accuracy.  (1e-5 was below the fp32 noise of p' for a resting part: every line search of the
// grouped part solver ran all 20 evaluations for bit-identical steps -- 20.0 passes per call against 4.0, measured on the
// emulated build over 64 envs x 20 env steps; the cooperative solver went from 6.1 to 3.2 evaluations per Newton iteration
// with the same number of iterations.)
#define FE_LS_TOL 1e-2f

struct FeOpt {
  int maxcon;       // contact capacity per env
  int newton_iters; // max Newton iterations
  int ls_iters;     // max line-search evaluations
  float tolerance;  // scaled improvement / gradient tolerance (MuJoCo: 1e-8 in double)
};

// ---- shared-memory slice of one warp (= one env).  All sizes in 4-byte words.
// The slice starts with a small header (FeWarp) followed by the arrays below.  Where each array starts depends only on
// the model and the contact capacity, so the offsets live in one FeLayout table -- __constant__ memory on the device,
// where every thread reads the same entry -- and `w->qpos()` is header address + table entry: no per-thread pointer
// table, no local-memory traffic to reach the slice.
#define FE_SLICE_F(X) /* float arrays */ \
  X(qpos) X(qvel) X(warm) X(ctrl) X(qfrc_applied) X(gravcomp) X(eq_data) X(mpos) /* persistent state */ \
  X(lpos) X(lquat) X(lmat) X(S) X(lvel) X(lacc) X(lfrc) X(linert) X(lcrb) X(Mr) X(fs) X(as) X(bias) X(lacc2) /* kinematics / dynamics */ \
  X(gpos) X(gmat) /* collision */ \
  X(c_dist) X(c_pos) X(c_frame) X(c_aref) X(c_D) X(c_mu) X(c_fric) X(c_jar) X(c_f) /* contacts (SoA, maxcon each) */ \
  X(w_r1) X(w_G) X(w_aref) X(w_D) X(w_jar) X(w_jv) X(w_f) /* welds (neq each) */ \
  X(l_sign) X(l_aref) X(l_D) X(l_jar) X(l_f) /* joint limits (nr each) */ \
  X(x) X(grad) X(search) X(Mv) X(fc) X(Hm) X(Jc) X(scr) /* solver */
#define FE_SLICE_I(X) /* int arrays */ \
  X(contype) X(conaff) X(eq_active) X(cand) X(touch) X(c_geom) X(c_link) X(c_state) X(c_kind) X(plist) X(first) X(iscr) X(colmap) \
  X(u) /* uniform scalars: the FE_U_* words */
// Arrays only the cooperative fallback solver (fe_solve_coop) uses: the full tri(nv) Hessian, its line-search rows and block
// flags.  They live in a per-env block of global memory (FeState::coop, reached through FeWarp::coop), not in the slice: the
// fallback runs only for a component beyond 32 dofs or 32 contacts, and keeping them out of the slice lets more envs share an SM.
#define FE_COOP_F(X) X(H) X(Ma) X(c_jv) X(l_jv)
#define FE_COOP_I(X) X(skip)

#define FE_NSTAT 28 /* per-call statistics: the FE_STAT_* columns of the `stats` field (include/furniture_b200.h) */
// words of u: the per-call scalars, then the statistics (column c of `stats` in word FE_U_STAT + c)
enum { FE_U_NCON = 0, FE_U_NCAND = 1, FE_U_FLAGS = 2, FE_U_NITER = 3, FE_U_STAT = 4 };
static_assert(FE_STAT_NEWTON_LS < FE_NSTAT && FE_U_STAT + FE_NSTAT <= 32, "u holds every column and is cleared by one lane each");
struct FeLayout {
#define X(f) int f;
  FE_SLICE_F(X) FE_SLICE_I(X) FE_COOP_F(X) FE_COOP_I(X)
#undef X
  int coop_words; // size of an env's block of FE_COOP_* arrays
};
static FeLayout fe_h_lay; // host copy: what the lane-emulated build reads, and what the CUDA build uploads
#if FE_DEVICE_BUILD
extern __shared__ float fe_smem[];
__constant__ FeLayout fe_c_lay;
#define FE_ACC __host__ __device__ __forceinline__
#else
#define FE_ACC inline
#endif
#if defined(__CUDA_ARCH__)
#define FE_LAY fe_c_lay
#else
#define FE_LAY fe_h_lay
#endif

#define FE_WARP_HDR_WORDS 10 /* sizeof(FeWarp) is 8 words; the 2 spare words keep every array at the offset the kernels were tuned with */
struct FeWarp { // header at word 0 of the slice
  const fe_model* m;
  FeOpt opt;
  float* coop; // this env's block of the FE_COOP_* arrays in global memory (set by fe_load)
  // Device: the slice address is rebuilt from the dynamic shared-memory symbol plus the warp's byte offset, so that the compiler
  // sees a shared-memory pointer and emits LDS / STS with 32-bit addresses (through the generic `this` every slice access was
  // a generic LD.E / ST.E with a 64-bit address pair).
#if defined(__CUDA_ARCH__)
  __device__ __forceinline__ char* base_() const { return (char*)fe_smem + (unsigned)(__cvta_generic_to_shared(this) - __cvta_generic_to_shared(fe_smem)); }
#else
  FE_ACC char* base_() const { return (char*)this; }
#endif
#define X(f) FE_ACC float* f() const { return (float*)base_() + FE_LAY.f; }
  FE_SLICE_F(X)
#undef X
#define X(f) FE_ACC int* f() const { return (int*)base_() + FE_LAY.f; }
  FE_SLICE_I(X)
#undef X
#define X(f) FE_ACC float* f() const { return coop + FE_LAY.f; }
  FE_COOP_F(X)
#undef X
#define X(f) FE_ACC int* f() const { return (int*)coop + FE_LAY.f; }
  FE_COOP_I(X)
#undef X
};
static_assert(sizeof(FeWarp) <= 4 * FE_WARP_HDR_WORDS, "slice header too small");

FE_BOTH int fe_tri(int n) { return n * (n + 1) / 2; }

// Lays the slice out; returns the number of words used.
FE_BOTH int fe_layout_build(FeLayout* L, const fe_model* m, const FeOpt& opt) {
  int o = FE_WARP_HDR_WORDS;
  const int nq = m->nq, nv = m->nv, nu = m->nu, nl = m->nlink, nr = m->nr, np = m->npart, ng = m->ngeom, ne = m->neq, mc = opt.maxcon;
#define CARVE(field, n) L->field = o; o += (n);
  CARVE(qpos, nq) CARVE(qvel, nv) CARVE(warm, nv) CARVE(ctrl, nu) CARVE(qfrc_applied, nr) CARVE(gravcomp, np) CARVE(eq_data, 7 * ne) CARVE(mpos, 3 * m->nmov)
  CARVE(contype, ng) CARVE(conaff, ng) CARVE(eq_active, ne)
  CARVE(lpos, 3 * nl) CARVE(lquat, 4 * nl) CARVE(lmat, 9 * nl) CARVE(S, 6 * nr) CARVE(lvel, 6 * nl) CARVE(lfrc, 6 * nl)
  L->lacc2 = L->lfrc; /* RNE wrench (smooth stage) and solver link accelerations are never live together */
  CARVE(linert, 10 * nl) CARVE(lcrb, (10 * nr > 96 ? 10 * nr : 96)) CARVE(Mr, nr * nr) CARVE(fs, nv) CARVE(as, nv) CARVE(bias, nr)
  CARVE(touch, np)
  CARVE(c_dist, mc) CARVE(c_pos, 3 * mc) CARVE(c_frame, 6 * mc) CARVE(c_aref, 3 * mc) CARVE(c_D, 2 * mc) CARVE(c_mu, mc) CARVE(c_fric, mc)
  CARVE(c_jar, 3 * mc) CARVE(c_f, 3 * mc) CARVE(c_geom, mc) CARVE(c_link, mc) CARVE(c_state, mc) CARVE(c_kind, mc) CARVE(plist, 9 * np)
  CARVE(w_r1, 3 * ne) CARVE(w_G, 9 * ne) CARVE(w_aref, 6 * ne) CARVE(w_D, 6 * ne) CARVE(w_jar, 6 * ne) CARVE(w_jv, 6 * ne) CARVE(w_f, 6 * ne)
  CARVE(l_sign, nr) CARVE(l_aref, nr) CARVE(l_D, nr) CARVE(l_jar, nr) CARVE(l_f, nr)
  CARVE(x, nv) CARVE(grad, nv) CARVE(search, nv) CARVE(Mv, nv) CARVE(fc, nv)
  L->Jc = L->lcrb; /* composite inertias (smooth stage) vs row staging of fe_build_H */
  CARVE(scr, 2 * 32) CARVE(first, nv) CARVE(iscr, 32) CARVE(colmap, 32) CARVE(u, FE_U_STAT + FE_NSTAT)
  // Three users of one region, never live together: the RNE link accelerations (smooth stage), the collision scratch (geom
  // poses, candidate list) and the constant part of the register solver's Hessian (fe_solve_comp: packed lower triangle over
  // the component's at most 32 active dofs).
  const int nh = nv < 32 ? nv : 32, hwords = fe_tri(nh), cwords = 12 * ng + FE_CAND_WORDS, awords = 6 * nl;
  L->Hm = o; L->gpos = o; L->gmat = o + 3 * ng; L->cand = o + 12 * ng; L->lacc = o;
  o += hwords > cwords ? (hwords > awords ? hwords : awords) : (cwords > awords ? cwords : awords);
  // the cooperative solver's arrays, in the env's block of global memory
  int g = 0;
#define GCARVE(field, n) L->field = g; g += (n);
  GCARVE(H, fe_tri(nv)) GCARVE(Ma, nv) GCARVE(c_jv, 3 * mc) GCARVE(l_jv, nr) GCARVE(skip, nv)
#undef GCARVE
  L->coop_words = g;
#undef CARVE
  return o;
}

// Writes the slice header; the arrays are reached through the layout table.
FE_FN FeWarp* fe_warp_bind(float* slice, const fe_model* m, const FeOpt& opt) {
  FeWarp* w = (FeWarp*)slice;
  LANES_BEGIN
    if (lane == 0) { w->m = m; w->opt = opt; }
  LANES_END
  return w;
}

// ---------------------------------------------------------------- 6x6 SPD helpers (packed lower, index i(i+1)/2+j)
FE_HD void fe_inert_sym6(float* A, const float* I, float diag_add) {
  const float m = I[0], hx = I[1], hy = I[2], hz = I[3];
  // rows 0-2: [Io, [h]x]; rows 3-5: [[h]x^T, m 1]
  A[0] = I[4] + diag_add;
  A[1] = I[7]; A[2] = I[5] + diag_add;
  A[3] = I[8]; A[4] = I[9]; A[5] = I[6] + diag_add;
  // row 3 (v_x): [h]x^T row 0 = (0, hz, -hy)
  A[6] = 0.f; A[7] = hz; A[8] = -hy; A[9] = m + diag_add;
  A[10] = -hz; A[11] = 0.f; A[12] = hx; A[13] = 0.f; A[14] = m + diag_add;
  A[15] = hy; A[16] = -hx; A[17] = 0.f; A[18] = 0.f; A[19] = 0.f; A[20] = m + diag_add;
}
// A += the same matrix (for a Hessian accumulated in place on top of contact terms)
FE_HD void fe_inert_sym6_add(float* A, const float* I) {
  const float m = I[0], hx = I[1], hy = I[2], hz = I[3];
  A[0] += I[4]; A[1] += I[7]; A[2] += I[5]; A[3] += I[8]; A[4] += I[9]; A[5] += I[6];
  A[7] += hz; A[8] -= hy; A[9] += m;
  A[10] -= hz; A[12] += hx; A[14] += m;
  A[15] += hy; A[16] -= hx; A[20] += m;
}
FE_HD bool fe_chol6(float* A) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    float s = A[k * (k + 1) / 2 + k];
#pragma unroll
    for (int j = 0; j < k; ++j) s -= A[k * (k + 1) / 2 + j] * A[k * (k + 1) / 2 + j];
    if (!(s > 1e-30f)) { ok = false; s = 1e-30f; }
    float l = sqrtf(s), inv = 1.0f / l;
    A[k * (k + 1) / 2 + k] = l;
#pragma unroll
    for (int i = k + 1; i < 6; ++i) {
      float t = A[i * (i + 1) / 2 + k];
#pragma unroll
      for (int j = 0; j < k; ++j) t -= A[i * (i + 1) / 2 + j] * A[k * (k + 1) / 2 + j];
      A[i * (i + 1) / 2 + k] = t * inv;
    }
  }
  return ok;
}
FE_HD void fe_chol6_solve(const float* L, float* x) {
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    float s = x[i];
#pragma unroll
    for (int j = 0; j < i; ++j) s -= L[i * (i + 1) / 2 + j] * x[j];
    x[i] = s / L[i * (i + 1) / 2 + i];
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    float s = x[i];
#pragma unroll
    for (int j = i + 1; j < 6; ++j) s -= L[j * (j + 1) / 2 + i] * x[j];
    x[i] = s / L[i * (i + 1) / 2 + i];
  }
}

// ---------------------------------------------------------------- cooperative skyline Cholesky (packed lower H)
// first[i] = first column of row i's envelope. Returns false (uniform) if a pivot is not positive.
FE_FN bool fe_chol(FeWarp* w, float* H, const int* first, int n, const int* skip = nullptr) {
  bool ok = true;
  for (int k = 0; k < n; ++k) {
    if (skip && skip[k]) continue; // column of an independent 6x6 block, factored in registers by fe_chol_blocks
    const int fk = first[k];
    LANES_BEGIN
      for (int i = k + lane; i < n; i += 32) {
        int fi = first[i];
        if (fi > k) continue;
        int j0 = fi > fk ? fi : fk;
        const float* Hi = H + fe_tri(i);
        const float* Hk = H + fe_tri(k);
        float s = Hi[k];
        for (int j = j0; j < k; ++j) s -= Hi[j] * Hk[j];
        H[fe_tri(i) + k] = s;
      }
    LANES_END
    float pk = H[fe_tri(k) + k];
    FE_SYNC; // every lane has read the pivot before the row-k lane overwrites it
    if (!(pk > 1e-30f)) { ok = false; pk = 1e-30f; }
    const float lkk = sqrtf(pk), inv = 1.0f / lkk;
    LANES_BEGIN
      for (int i = k + lane; i < n; i += 32) {
        if (first[i] > k) continue;
        if (i == k) H[fe_tri(k) + k] = lkk; else H[fe_tri(i) + k] *= inv;
      }
    LANES_END
  }
  return ok;
}
// x <- (L L^T)^-1 x ; tmp is an n-vector scratch
FE_FN void fe_chol_solve(FeWarp* w, const float* L, const int* first, int n, float* x, float* tmp, const int* skip = nullptr) {
  for (int k = 0; k < n; ++k) { // forward: tmp = L^-1 x
    if (skip && skip[k]) continue;
    const float xk = x[k] / L[fe_tri(k) + k];
    LANES_BEGIN
      if (lane == 0) tmp[k] = xk;
      for (int i = k + 1 + lane; i < n; i += 32)
        if (first[i] <= k) x[i] -= L[fe_tri(i) + k] * xk;
    LANES_END
  }
  for (int k = n - 1; k >= 0; --k) { // backward: x = L^-T tmp
    if (skip && skip[k]) continue;
    const float xk = tmp[k] / L[fe_tri(k) + k];
    const int fk = first[k];
    LANES_BEGIN
      if (lane == 0) x[k] = xk;
      for (int j = fk + lane; j < k; j += 32) tmp[j] -= L[fe_tri(k) + j] * xk;
    LANES_END
  }
}

// Free-part blocks whose rows start at their own block and that no later row reaches are independent 6x6 systems:
// flag their columns (skip) so that the synchronised column loops above leave them to one lane each.
FE_FN void fe_mark_indep_blocks(FeWarp* w, const int* first, int* skip) {
  const fe_model* m = w->m;
  const int nr = m->nr, np = m->npart;
  LANES_BEGIN
    for (int d = lane; d < nr; d += 32) skip[d] = 0;
    for (int p = lane; p < np; p += 32) {
      const int sp = nr + 6 * p;
      int indep = first[sp] == sp;
      for (int q = p + 1; q < np && indep; ++q) if (first[nr + 6 * q] <= sp) indep = 0;
      for (int k = 0; k < 6; ++k) skip[sp + k] = indep;
    }
  LANES_END
}
FE_FN void fe_chol_blocks(FeWarp* w, float* H, const int* skip) {
  const fe_model* m = w->m;
  const int nr = m->nr, np = m->npart;
  LANES_BEGIN
    for (int p = lane; p < np; p += 32) {
      const int sp = nr + 6 * p;
      if (skip[sp]) {
        float A[21];
        for (int i = 0; i < 6; ++i) for (int j = 0; j <= i; ++j) A[i * (i + 1) / 2 + j] = H[fe_tri(sp + i) + sp + j];
        if (!fe_chol6(A)) w->u()[FE_U_FLAGS] |= FE_FLAG_NEWTON_PIVOT;
        for (int i = 0; i < 6; ++i) for (int j = 0; j <= i; ++j) H[fe_tri(sp + i) + sp + j] = A[i * (i + 1) / 2 + j];
      }
    }
  LANES_END
}
FE_FN void fe_solve_blocks(FeWarp* w, const float* L, const int* skip, float* x) {
  const fe_model* m = w->m;
  const int nr = m->nr, np = m->npart;
  LANES_BEGIN
    for (int p = lane; p < np; p += 32) {
      const int sp = nr + 6 * p;
      if (skip[sp]) {
        float A[21], b[6];
        for (int i = 0; i < 6; ++i) { b[i] = x[sp + i]; for (int j = 0; j <= i; ++j) A[i * (i + 1) / 2 + j] = L[fe_tri(sp + i) + sp + j]; }
        fe_chol6_solve(A, b);
        for (int i = 0; i < 6; ++i) x[sp + i] = b[i];
      }
    }
  LANES_END
}

// Solves an SPD system held by rows in registers: lane i owns row i of the lower triangle in row_[0..NMAX) (rows and columns
// beyond the system padded with the identity) and its right-hand side in b_, which holds x_i on exit.  Right-looking
// Cholesky with the pivot column broadcast by shuffle, then y = L^-1 b and x = L^-T y (column k of L is spread over the
// lanes: one butterfly sum per unknown).  bad_ is set where a pivot was not positive (it is replaced by 1e-30).
#define FE_REG_CHOL_SOLVE(NMAX, row_, b_, bad_)                                                                                  \
  {                                                                                                                                \
    FE_PRIV(float, s0_); FE_PRIV(float, s1_); FE_PRIV(float, dinv_); FE_PRIV(float, q_);                                          \
    REGS_BEGIN PV(bad_) = 0; PV(dinv_) = 1.f; REGS_END                                                                             \
    _Pragma("unroll") for (int k = 0; k < (NMAX); ++k) {                                                                           \
      FE_SHFLA(s0_, row_, k, k);                                                                                                   \
      REGS_BEGIN                                                                                                                   \
        float pk = PV(s0_);                                                                                                        \
        if (!(pk > 1e-30f)) { PV(bad_) = 1; pk = 1e-30f; }                                                                         \
        const float lkk = sqrtf(pk), inv = 1.0f / lkk;                                                                             \
        const float lik = lane > k ? PV(row_)[k] * inv : (lane == k ? lkk : 0.f);                                                  \
        PV(row_)[k] = lik;                                                                                                         \
        PV(q_) = lik;                                                                                                              \
        if (lane == k) PV(dinv_) = inv;                                                                                            \
      REGS_END                                                                                                                     \
      _Pragma("unroll") for (int j = k + 1; j < (NMAX); ++j) {                                                                     \
        FE_SHFL(s1_, q_, j);                                                                                                       \
        REGS_BEGIN PV(row_)[j] -= PV(q_) * PV(s1_); REGS_END                                                                       \
      }                                                                                                                            \
    }                                                                                                                              \
    _Pragma("unroll") for (int k = 0; k < (NMAX); ++k) { /* y = L^-1 b */                                                         \
      REGS_BEGIN PV(q_) = PV(b_) * PV(dinv_); REGS_END                                                                             \
      FE_SHFL(s0_, q_, k);                                                                                                         \
      REGS_BEGIN                                                                                                                   \
        if (lane > k) PV(b_) -= PV(row_)[k] * PV(s0_);                                                                             \
        else if (lane == k) PV(b_) = PV(s0_);                                                                                      \
      REGS_END                                                                                                                     \
    }                                                                                                                              \
    _Pragma("unroll") for (int k = (NMAX) - 1; k >= 0; --k) { /* x = L^-T y */                                                    \
      REGS_BEGIN PV(q_) = (lane > k && lane < (NMAX)) ? PV(row_)[k] * PV(b_) : 0.f; REGS_END                                       \
      FE_WSUM(q_);                                                                                                                 \
      REGS_BEGIN if (lane == k) PV(b_) = (PV(b_) - PV(q_)) * PV(dinv_); REGS_END                                                   \
    }                                                                                                                              \
  }

// ---------------------------------------------------------------- kinematics + smooth dynamics
// x = (Mr + hdamp * diag(dof_damping) + diag(dadd))^-1 b for the robot block (nr <= NMAX; dadd may be null): lane i owns row i of the lower triangle in
// registers, factored and solved by FE_REG_CHOL_SOLVE.  Two lane regions in all, against some forty for the cooperative
// slice version (a region per column step of fe_chol and per unknown of fe_chol_solve): the smooth acceleration of
// fe_kin_smooth and the implicit-damping
// solve of fe_integrate were mostly barriers.  b and x may alias.  Rows and columns beyond nr are padded with the identity.
template <int NMAX>
FE_FN void fe_robot_solve_regs(FeWarp* w, float hdamp, const float* dadd, const float* b, float* x, int flagbit) {
  const fe_model* m = w->m;
  const int nr = m->nr;
  FE_PRIVA(float, row_, NMAX);
  FE_PRIV(float, b_); FE_PRIV(int, bad_);
  REGS_BEGIN
    const int i = lane;
#pragma unroll
    for (int j = 0; j < NMAX; ++j) {
      float v = (j == i) ? 1.f : 0.f;
      if (i < nr && j <= i) v = w->Mr()[i * nr + j] + (j == i ? hdamp * m->dof_damping[i] + (dadd ? dadd[i] : 0.f) : 0.f);
      PV(row_)[j] = v;
    }
    PV(b_) = i < nr ? b[i] : 0.f;
  REGS_END
  FE_REG_CHOL_SOLVE(NMAX, row_, b_, bad_)
  LANES_BEGIN
    if (lane < nr) x[lane] = PV(b_);
    if (PV(bad_) && lane == 0) w->u()[FE_U_FLAGS] |= flagbit;
  LANES_END
}
FE_FN void fe_robot_solve(FeWarp* w, float hdamp, const float* dadd, const float* b, float* x, int flagbit) {
  const int nr = w->m->nr;
  if (nr <= 12) fe_robot_solve_regs<12>(w, hdamp, dadd, b, x, flagbit);
  else if (nr <= 16) fe_robot_solve_regs<16>(w, hdamp, dadd, b, x, flagbit);
  else fe_robot_solve_regs<24>(w, hdamp, dadd, b, x, flagbit);
}

FE_FN void fe_kin_smooth(FeWarp* w) {
  const fe_model* m = w->m;
  const int nl = m->nlink, nr = m->nr, nrl = m->nrlink, nv = m->nv;
  const float Pr[3] = {m->robot_ref[0], m->robot_ref[1], m->robot_ref[2]};
  const float g[3] = {m->gravity[0], m->gravity[1], m->gravity[2]};
  FE_PRIVA(float, Atmp_, 6);
  // Forward pass without a per-level loop: every robot link first builds its own joint transform, then world poses,
  // velocities and bias accelerations are obtained by pointer jumping up the tree (log2(depth) short regions).
  int nsteps = 0;
  while ((1 << nsteps) <= m->maxdepth) ++nsteps;
  float* const bufp[2] = {w->lpos(), w->lacc()};   // position (3 of 6 words per link in the scratch buffer)
  float* const bufq[2] = {w->lquat(), w->lfrc()};  // quaternion (4 of 6 words)
  int* const bufa[2] = {w->iscr(), w->colmap()};   // ancestor pointer
  const int strp[2] = {3, 6}, strq[2] = {4, 6};
  LANES_BEGIN
    const int l = lane;
    if (l < nl) {
      const int qa = m->link_qadr[l], da = m->link_dadr[l];
      if (m->link_jtype[l] == FE_JNT_FREE) { // pose straight from qpos; V, A in closed form about the link origin
        float pos[3], quat[4], R[9], V[6], A[6], t[3];
        v3cpy(pos, w->qpos() + qa);
        quat[0] = w->qpos()[qa + 3]; quat[1] = w->qpos()[qa + 4]; quat[2] = w->qpos()[qa + 5]; quat[3] = w->qpos()[qa + 6];
        qnormalize(quat);
        q2mat(R, quat);
        m3mulv(V, R, w->qvel() + da + 3);
        v3cpy(V + 3, w->qvel() + da);
        v3cross(t, V, V + 3);
        A[0] = A[1] = A[2] = 0.f;
        A[3] = -t[0] - g[0]; A[4] = -t[1] - g[1]; A[5] = -t[2] - g[2];
        v3cpy(w->lpos() + 3 * l, pos);
        for (int k = 0; k < 4; ++k) w->lquat()[4 * l + k] = quat[k];
        for (int k = 0; k < 9; ++k) w->lmat()[9 * l + k] = R[k];
        for (int k = 0; k < 6; ++k) { w->lvel()[6 * l + k] = V[k]; w->lacc2()[6 * l + k] = A[k]; }
      } else { // joint transform in the parent link frame
        float p0[3], q0[4], R0[9], t[3], pos[3], quat[4];
        v3cpy(p0, m->link_pos[l]);
        for (int k = 0; k < 4; ++k) q0[k] = m->link_quat[l][k];
        const float q = w->qpos()[qa];
        if (m->link_jtype[l] == FE_JNT_HINGE) {
          const float sn = sinf(0.5f * q), cs = cosf(0.5f * q);
          const float ql[4] = {cs, m->link_jaxis[l][0] * sn, m->link_jaxis[l][1] * sn, m->link_jaxis[l][2] * sn};
          float R1[9], t1[3];
          qmul(quat, q0, ql);
          qnormalize(quat);
          q2mat(R0, q0);
          q2mat(R1, quat);
          m3mulv(t, R0, m->link_jpos[l]);
          m3mulv(t1, R1, m->link_jpos[l]);
          for (int k = 0; k < 3; ++k) pos[k] = p0[k] + t[k] - t1[k];
        } else {
          q2mat(R0, q0);
          m3mulv(t, R0, m->link_jaxis[l]);
          v3madd(pos, p0, t, q);
          for (int k = 0; k < 4; ++k) quat[k] = q0[k];
        }
        const int s0 = nsteps & 1; // start buffer chosen so that the result lands in lpos / lquat
        v3cpy(bufp[s0] + strp[s0] * l, pos);
        for (int k = 0; k < 4; ++k) bufq[s0][strq[s0] * l + k] = quat[k];
        bufa[s0][l] = m->link_parent[l];
      }
    }
  LANES_END
  for (int st = 0; st < nsteps; ++st) {
    const int cur = (nsteps - st) & 1, nxt = cur ^ 1;
    LANES_BEGIN
      const int l = lane;
      if (l < nrl) {
        const int a = bufa[cur][l];
        float pos[3], quat[4];
        v3cpy(pos, bufp[cur] + strp[cur] * l);
        for (int k = 0; k < 4; ++k) quat[k] = bufq[cur][strq[cur] * l + k];
        int an = a;
        if (a >= 0) { // compose with the transform accumulated at the ancestor
          float qa_[4], Ra[9], t[3], qn[4];
          for (int k = 0; k < 4; ++k) qa_[k] = bufq[cur][strq[cur] * a + k];
          q2mat(Ra, qa_);
          m3mulv(t, Ra, pos);
          v3add(pos, bufp[cur] + strp[cur] * a, t);
          qmul(qn, qa_, quat);
          for (int k = 0; k < 4; ++k) quat[k] = qn[k];
          an = bufa[cur][a];
        }
        v3cpy(bufp[nxt] + strp[nxt] * l, pos);
        for (int k = 0; k < 4; ++k) bufq[nxt][strq[nxt] * l + k] = quat[k];
        bufa[nxt][l] = an;
      }
    LANES_END
  }
  // world rotation, joint motion subspace S (about robot_ref), own velocity term
  float* const bufv[2] = {w->lvel(), w->lacc()};
  LANES_BEGIN
    const int l = lane;
    if (l < nrl) {
      float quat[4], R[9], t[3], anchor[3], axis[3], Sd[6];
      for (int k = 0; k < 4; ++k) quat[k] = w->lquat()[4 * l + k];
      qnormalize(quat);
      for (int k = 0; k < 4; ++k) w->lquat()[4 * l + k] = quat[k];
      q2mat(R, quat);
      for (int k = 0; k < 9; ++k) w->lmat()[9 * l + k] = R[k];
      m3mulv(t, R, m->link_jpos[l]);
      v3add(anchor, w->lpos() + 3 * l, t);
      m3mulv(axis, R, m->link_jaxis[l]);
      if (m->link_jtype[l] == FE_JNT_HINGE) { v3cpy(Sd, axis); v3sub(t, anchor, Pr); v3cross(Sd + 3, t, axis); }
      else { Sd[0] = Sd[1] = Sd[2] = 0.f; v3cpy(Sd + 3, axis); }
      const int da = m->link_dadr[l];
      const float qd = w->qvel()[da];
      const int s0 = nsteps & 1;
      for (int k = 0; k < 6; ++k) { w->S()[6 * da + k] = Sd[k]; bufv[s0][6 * l + k] = Sd[k] * qd; }
      bufa[s0][l] = m->link_parent[l];
    }
  LANES_END
  for (int st = 0; st < nsteps; ++st) { // V_l = sum over ancestors of S_d qd
    const int cur = (nsteps - st) & 1, nxt = cur ^ 1;
    LANES_BEGIN
      const int l = lane;
      if (l < nrl) {
        const int a = bufa[cur][l];
        for (int k = 0; k < 6; ++k) bufv[nxt][6 * l + k] = bufv[cur][6 * l + k] + (a >= 0 ? bufv[cur][6 * a + k] : 0.f);
        bufa[nxt][l] = a >= 0 ? bufa[cur][a] : -1;
      }
    LANES_END
  }
  // bias acceleration: A_l = [0; -g] + sum over ancestors of (V_parent(d) x_m S_d) qd
  float* const bufc[2] = {w->lfrc(), w->lacc()};
  LANES_BEGIN
    const int l = lane;
    if (l < nrl) {
      const int p = m->link_parent[l], da = m->link_dadr[l];
      float Vp[6] = {0, 0, 0, 0, 0, 0}, Sdot[6];
      if (p >= 0) for (int k = 0; k < 6; ++k) Vp[k] = w->lvel()[6 * p + k];
      crossm(Sdot, Vp, w->S() + 6 * da);
      const float qd = w->qvel()[da];
      const int s0 = nsteps & 1;
      for (int k = 0; k < 6; ++k) bufc[s0][6 * l + k] = Sdot[k] * qd;
      bufa[s0][l] = p;
    }
  LANES_END
  for (int st = 0; st < nsteps; ++st) {
    const int cur = (nsteps - st) & 1, nxt = cur ^ 1;
    LANES_BEGIN
      const int l = lane;
      if (l < nrl) {
        const int a = bufa[cur][l];
        for (int k = 0; k < 6; ++k) bufc[nxt][6 * l + k] = bufc[cur][6 * l + k] + (a >= 0 ? bufc[cur][6 * a + k] : 0.f);
        bufa[nxt][l] = a >= 0 ? bufa[cur][a] : -1;
      }
    LANES_END
  }
  LANES_BEGIN // result of the scan is in lfrc; move it (plus the gravity term) to lacc, where the parts already wrote theirs via lacc2
    const int l = lane;
    float A[6];
    if (l < nl) {
      if (l < nrl) { for (int k = 0; k < 6; ++k) A[k] = w->lfrc()[6 * l + k]; A[3] -= g[0]; A[4] -= g[1]; A[5] -= g[2]; }
      else for (int k = 0; k < 6; ++k) A[k] = w->lacc2()[6 * l + k];
    }
    PV(Atmp_)[0] = A[0]; PV(Atmp_)[1] = A[1]; PV(Atmp_)[2] = A[2]; PV(Atmp_)[3] = A[3]; PV(Atmp_)[4] = A[4]; PV(Atmp_)[5] = A[5];
  LANES_END
  LANES_BEGIN
    if (lane < nl) for (int k = 0; k < 6; ++k) w->lacc()[6 * lane + k] = PV(Atmp_)[k];
  LANES_END
  // spatial inertia about the link's reference point (robot_ref for robot links, own origin for parts) + RNE wrench
  LANES_BEGIN
    const int l = lane;
    if (l < nl) {
      const float* R = w->lmat() + 9 * l;
      float I[10], t[3];
      I[0] = m->link_mass[l];
      m3mulv(t, R, m->link_com[l]);
      if (l < nrl) {
        float d[3];
        v3add(d, w->lpos() + 3 * l, t);
        v3sub(d, d, Pr);
        sym3rot(I + 4, R, m->link_inertia_c[l]);
        const float mm = I[0], dd = v3dot(d, d);
        I[4] += mm * (dd - d[0] * d[0]); I[5] += mm * (dd - d[1] * d[1]); I[6] += mm * (dd - d[2] * d[2]);
        I[7] -= mm * d[0] * d[1]; I[8] -= mm * d[0] * d[2]; I[9] -= mm * d[1] * d[2];
        I[1] = mm * d[0]; I[2] = mm * d[1]; I[3] = mm * d[2];
      } else {
        sym3rot(I + 4, R, m->link_inertia_o[l]);
        I[1] = I[0] * t[0]; I[2] = I[0] * t[1]; I[3] = I[0] * t[2];
      }
      float IA[6], IV[6], X[6];
      inert_mulv(IA, I, w->lacc() + 6 * l);
      inert_mulv(IV, I, w->lvel() + 6 * l);
      crossf(X, w->lvel() + 6 * l, IV);
      for (int k = 0; k < 10; ++k) w->linert()[10 * l + k] = I[k];
      if (l < nrl) for (int k = 0; k < 10; ++k) w->lcrb()[10 * l + k] = I[k];
      for (int k = 0; k < 6; ++k) w->lfrc()[6 * l + k] = IA[k] + X[k];
    }
  LANES_END
  // robot: each dof sums the RNE wrench and the spatial inertia of its subtree (links whose ancestor mask holds it),
  // then bias force, joint-space inertia row (CRBA) and smooth force
  LANES_BEGIN
    const int d = lane;
    if (d < nr) {
      const float* Sd = w->S() + 6 * d;
      float Fs[6] = {0, 0, 0, 0, 0, 0}, Ic[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
      for (int c = d; c < nrl; ++c)
        if ((m->link_ancmask[c] >> d) & 1) {
          for (int k = 0; k < 6; ++k) Fs[k] += w->lfrc()[6 * c + k];
          for (int k = 0; k < 10; ++k) Ic[k] += w->lcrb()[10 * c + k];
        }
      const float b = dot6(Sd, Fs);
      w->bias()[d] = b;
      float F[6];
      inert_mulv(F, Ic, Sd);
      for (int a = d; a >= 0; a = m->link_parent[a]) {
        float v = dot6(w->S() + 6 * a, F);
        if (a == d) v += m->rdof_armature[d];
        w->Mr()[d * nr + a] = v;
        w->Mr()[a * nr + d] = v;
      }
      float f = -m->dof_damping[d] * w->qvel()[d] - b + w->qfrc_applied()[d];
      for (int u = 0; u < m->nu; ++u)
        if (m->act_dof[u] == d) {
          float c = w->ctrl()[u];
          if (m->act_ctrllimited[u]) c = fminf(fmaxf(c, m->act_ctrlrange[u][0]), m->act_ctrlrange[u][1]);
          const float gear = m->act_gear[u];
          float af = m->act_gain[u] * c + m->act_bias[u][0] + m->act_bias[u][1] * gear * w->qpos()[m->act_qadr[u]] + m->act_bias[u][2] * gear * w->qvel()[d];
          if (m->act_forcelimited[u]) af = fminf(fmaxf(af, m->act_forcerange[u][0]), m->act_forcerange[u][1]);
          f += gear * af;
        }
      w->fs()[d] = f;
    }
  LANES_END
  // zero the entries of Mr between unrelated dofs (branches) -- they are never written above
  LANES_BEGIN
    for (int e = lane; e < nr * nr; e += 32) {
      int i = e / nr, j = e % nr;
      int lo = i < j ? i : j, hi = i < j ? j : i;
      if (!((m->link_ancmask[hi] >> lo) & 1)) w->Mr()[e] = 0.f;
    }
    for (int e = lane; e < nr; e += 32) w->first()[e] = 0;
  LANES_END
  // parts: smooth wrench and acceleration in z coordinates
  LANES_BEGIN
    const int p = lane;
    if (p < m->npart) {
      const int l = nrl + p, z = nr + 6 * p, da = m->link_dadr[l];
      const float* I = w->linert() + 10 * l;
      const float* V = w->lvel() + 6 * l;
      const float damp = m->dof_damping[da];
      float W[6];
      for (int k = 0; k < 6; ++k) W[k] = -w->lfrc()[6 * l + k] - damp * V[k];
      const float gc = w->gravcomp()[p];
      if (gc != 0.f) { // xfrc_applied = -gc * gravity * mass at the CoM (furniture.py:2778-2790)
        float F[3] = {-gc * g[0] * I[0], -gc * g[1] * I[0], -gc * g[2] * I[0]}, r[3] = {I[1] / I[0], I[2] / I[0], I[3] / I[0]}, t[3];
        v3cross(t, r, F);
        W[0] += t[0]; W[1] += t[1]; W[2] += t[2]; W[3] += F[0]; W[4] += F[1]; W[5] += F[2];
      }
      float A[21], a[6];
      fe_inert_sym6(A, I, 0.f);
      if (!fe_chol6(A)) w->u()[FE_U_FLAGS] |= FE_FLAG_NUMERIC;
      for (int k = 0; k < 6; ++k) { w->fs()[z + k] = W[k]; a[k] = W[k]; }
      fe_chol6_solve(A, a);
      for (int k = 0; k < 6; ++k) w->as()[z + k] = a[k];
    }
  LANES_END
  // robot smooth acceleration: as = Mr^-1 fs
  if (nr > 0) {
    fe_robot_solve(w, 0.f, nullptr, w->fs(), w->as(), FE_FLAG_NUMERIC);
  }
  (void)nv;
}

// ---------------------------------------------------------------- collision
#if FE_DEVICE_BUILD
FE_HD int fe_lane_excl_scan(int n) {
  int v = n;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, o);
    if ((int)(threadIdx.x & 31u) >= o) v += t;
  }
  return v - n;
}
#define FE_SCAN(run, n) fe_lane_excl_scan(n)
#else
#define FE_SCAN(run, n) ((run += (n)), (run - (n)))
#endif

// position of the j-th set bit (from 0) of the 64-bit mask hi:lo; requires j < its population count
FE_HD int fe_nth_bit(unsigned lo, unsigned hi, int j) {
#if FE_DEVICE_BUILD
#define FE_POPC(v) __popc(v)
#else
#define FE_POPC(v) __builtin_popcount(v)
#endif
  unsigned h = lo;
  int pos = 0;
  if (j >= FE_POPC(lo)) { j -= FE_POPC(lo); h = hi; pos = 32; }
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    const unsigned low = h & ((1u << s) - 1u);
    const int c = FE_POPC(low);
    if (j >= c) { j -= c; h >>= s; pos += s; } else h = low;
  }
#undef FE_POPC
  return pos;
}

// A pair with a sensor geom (gap > 0; mj_collision reports its contacts, mj_makeConstraint skips those with dist >= margin - gap):
// the contacts at or beyond `active` only raise the touch flags; the (rare) closer ones stay.  Returns the contacts kept.
FE_HDN int fe_sensor_pair(FeWarp* w, int g1, int g2, FeCon* res, int n, float active) {
  const fe_model* m = w->m;
  bool touching = false;
  for (int i = 0; i < n; ++i) touching |= res[i].dist >= active;
  if (touching) {
    const int t1 = m->geom_tag[g1], t2 = m->geom_tag[g2];
    const int pa = ((t1 >> FE_TAG_PART_SHIFT) & 0xff) - 1, pb = ((t2 >> FE_TAG_PART_SHIFT) & 0xff) - 1;
    const int bits1 = ((t1 & FE_TAG_LFINGER) ? 1 : 0) | ((t1 & FE_TAG_RFINGER) ? 2 : 0), bits2 = ((t2 & FE_TAG_LFINGER) ? 1 : 0) | ((t2 & FE_TAG_RFINGER) ? 2 : 0);
#if FE_DEVICE_BUILD
    if (pb >= 0 && bits1) atomicOr(w->touch() + pb, bits1);
    if (pa >= 0 && bits2) atomicOr(w->touch() + pa, bits2);
#else
    if (pb >= 0 && bits1) w->touch()[pb] |= bits1;
    if (pa >= 0 && bits2) w->touch()[pa] |= bits2;
#endif
  }
  int keep = 0;
  for (int i = 0; i < n; ++i) if (res[i].dist < active) res[keep++] = res[i];
  return keep;
}

FE_FN void fe_collide(FeWarp* w) {
  const fe_model* m = w->m;
  const int ng = m->ngeom, npair = m->npair, nrl = m->nrlink, mc = w->opt.maxcon;
  const bool hasm = m->has_margin != 0;
  LANES_BEGIN
    for (int gi = lane; gi < ng; gi += 32) {
      const int l = m->geom_link[gi];
      float* gp = w->gpos() + 3 * gi;
      float* gm = w->gmat() + 9 * gi;
      if (l < 0) {
        const int mv = m->nmov > 0 ? m->geom_mov[gi] : 0;
        v3cpy(gp, mv ? w->mpos() + 3 * (mv - 1) : m->geom_pos[gi]); // movable static geom: its world position is per-env state
        for (int k = 0; k < 9; ++k) gm[k] = m->geom_mat[gi][k];
      }
      else {
        float t[3];
        m3mulv(t, w->lmat() + 9 * l, m->geom_pos[gi]);
        v3add(gp, w->lpos() + 3 * l, t);
        m3mul(gm, w->lmat() + 9 * l, m->geom_mat[gi]);
      }
    }
    if (lane < m->npart) w->touch()[lane] = 0;
  LANES_END
  // broad phase: every lane tests a contiguous range of the pair list (order preserved), one scan gives each lane the offset of
  // its first hit in the candidate list
  const int per = (npair + 31) / 32;
  int ncand = 0;
  {
    int run = 0;
    (void)run;
    LANES_BEGIN
      unsigned long long hits = 0ull;
      const int k0 = lane * per, k1 = (k0 + per < npair) ? k0 + per : npair;
      for (int k = k0; k < k1; ++k) {
        const int g1 = m->pair_g1[k], g2 = m->pair_g2[k];
        if ((w->contype()[g1] & w->conaff()[g2]) || (w->contype()[g2] & w->conaff()[g1])) {
          float t[3];
          v3sub(t, w->gpos() + 3 * g2, w->gpos() + 3 * g1);
          bool hit;
          const float mg = hasm ? fmaxf(m->geom_margin[g1], m->geom_margin[g2]) : 0.f;
          if (m->geom_type[g1] == FE_GEOM_PLANE) {
            float n[3];
            fe_col(n, w->gmat() + 9 * g1, 2);
            hit = v3dot(t, n) <= m->geom_rbound[g2] + mg;
          } else {
            const float bnd = m->geom_rbound[g1] + m->geom_rbound[g2] + mg;
            hit = v3dot(t, t) <= bnd * bnd;
          }
          if (hit) hits |= 1ull << (k - k0);
        }
      }
#if FE_DEVICE_BUILD
      const int n = __popcll(hits);
#else
      const int n = __builtin_popcountll(hits);
#endif
      const int off = FE_SCAN(run, n);
      w->cand()[lane] = (int)(unsigned)hits;
      w->cand()[32 + lane] = (int)(unsigned)(hits >> 32);
      w->cand()[64 + lane] = off;
      if (lane == 31) w->iscr()[0] = off + n;
    LANES_END
    ncand = w->iscr()[0];
    LANES_BEGIN LANES_END
  }
  int ncon = 0;
  for (int base = 0; base < ncand; base += 32) {
    int run = 0;
    (void)run;
    LANES_BEGIN
      const int ci = base + lane;
      FeCon res[8];
      int n = 0, g1 = 0, g2 = 0;
      if (ci < ncand) {
        // candidate ci (pair-list order): owned by the last lane whose first hit is at or before ci -- a lane without hits shares
        // its offset with the next lane, so the last such lane has hits -- and it is that lane's (ci - offset)-th hit
        int o = 0;
        for (int s = 16; s >= 1; s >>= 1)
          if (w->cand()[64 + o + s] <= ci) o += s;
        const int k = o * per + fe_nth_bit((unsigned)w->cand()[o], (unsigned)w->cand()[32 + o], ci - w->cand()[64 + o]);
        g1 = m->pair_g1[k]; g2 = m->pair_g2[k];
        const float mg = hasm ? fmaxf(m->geom_margin[g1], m->geom_margin[g2]) : 0.f;
        n = fe_narrowphase(m, g1, g2, w->gpos() + 3 * g1, w->gmat() + 9 * g1, w->gpos() + 3 * g2, w->gmat() + 9 * g2, mg, res);
        if (m->has_gap) { const float gap = fmaxf(m->geom_gap[g1], m->geom_gap[g2]); if (gap > 0.f) n = fe_sensor_pair(w, g1, g2, res, n, mg - gap); }
      }
      const int off = FE_SCAN(run, n);
      for (int i = 0; i < n; ++i) {
        const int c = ncon + off + i;
        if (c < mc) {
          w->c_dist()[c] = res[i].dist;
          v3cpy(w->c_pos() + 3 * c, res[i].pos);
          v3cpy(w->c_frame() + 6 * c, res[i].n);
          w->c_geom()[c] = g1 | (g2 << 8);
        }
      }
      if (lane == 31) w->iscr()[0] = off + n;
    LANES_END
    ncon += w->iscr()[0];
    LANES_BEGIN LANES_END
  }
  if (ncon > mc) { ncon = mc; LANES_BEGIN if (lane == 0) w->u()[FE_U_FLAGS] |= FE_FLAG_CONTACT_FULL; LANES_END }
  // touch flags per part: bit0 left finger, bit1 right finger, bit2 floor, bit3 / bit4 the fingers of a second arm (furniture.py:500-520, :1290-1322)
  LANES_BEGIN
    const int p = lane;
    if (p < m->npart) {
      int bits = 0;
      for (int c = 0; c < ncon; ++c) {
        const int g1 = w->c_geom()[c] & 255, g2 = w->c_geom()[c] >> 8;
        const int t1 = m->geom_tag[g1], t2 = m->geom_tag[g2];
        const int p1 = ((t1 >> FE_TAG_PART_SHIFT) & 0xff) - 1, p2 = ((t2 >> FE_TAG_PART_SHIFT) & 0xff) - 1;
        if (p1 == p) bits |= ((t2 & FE_TAG_LFINGER) ? 1 : 0) | ((t2 & FE_TAG_RFINGER) ? 2 : 0) | ((t2 & FE_TAG_FLOOR) ? 4 : 0) | ((t2 & FE_TAG_LFINGER2) ? 8 : 0) | ((t2 & FE_TAG_RFINGER2) ? 16 : 0);
        if (p2 == p) bits |= ((t1 & FE_TAG_LFINGER) ? 1 : 0) | ((t1 & FE_TAG_RFINGER) ? 2 : 0) | ((t1 & FE_TAG_FLOOR) ? 4 : 0) | ((t1 & FE_TAG_LFINGER2) ? 8 : 0) | ((t1 & FE_TAG_RFINGER2) ? 16 : 0);
      }
      w->touch()[p] |= bits; // sensor pairs have set their bits during the narrow phase
    }
    if (lane == 0) { w->u()[FE_U_NCON] = ncon; w->u()[FE_U_NCAND] = ncand; }
  LANES_END
  (void)nrl;
}

// ---------------------------------------------------------------- constraint rows
FE_HD float fe_impedance(const float* si, float dist_abs) {
  float d0 = fminf(fmaxf(si[0], FE_MINIMP), FE_MAXIMP), d1 = fminf(fmaxf(si[1], FE_MINIMP), FE_MAXIMP);
  float width = fmaxf(si[2], FE_MINVAL);
  if (d0 == d1) return d0;
  float x = dist_abs / width;
  if (x >= 1.f) return d1;
  float y = x <= 0.5f ? 2.f * x * x : 1.f - 2.f * (1.f - x) * (1.f - x); // midpoint 0.5, power 2
  return d0 + y * (d1 - d0);
}
FE_HD void fe_kb(const float* solref, float dmax_in, float h, float* k, float* b) {
  float tc = solref[0], dr = solref[1];
  if (tc > 0.f && tc < 2.f * h) tc = 2.f * h; // refsafe
  float dmax = fminf(fmaxf(dmax_in, FE_MINIMP), FE_MAXIMP);
  *k = 1.f / (dmax * dmax * tc * tc * dr * dr);
  *b = 2.f / (dmax * tc);
}
// reference point of a link (world)
FE_HD void fe_link_ref(const FeWarp* w, int l, float* P) {
  if (l < w->m->nrlink) { P[0] = w->m->robot_ref[0]; P[1] = w->m->robot_ref[1]; P[2] = w->m->robot_ref[2]; }
  else v3cpy(P, w->lpos() + 3 * l);
}
// velocity-like quantity of the point p fixed to link l, from per-link spatial vectors X (6*nlink): X.v + X.w x (p - P)
FE_HD void fe_point_vel(const FeWarp* w, const float* X, int l, const float* p, float* out) {
  if (l < 0) { out[0] = out[1] = out[2] = 0.f; return; }
  float P[3], r[3], t[3];
  fe_link_ref(w, l, P);
  v3sub(r, p, P);
  v3cross(t, X + 6 * l, r);
  out[0] = X[6 * l + 3] + t[0]; out[1] = X[6 * l + 4] + t[1]; out[2] = X[6 * l + 5] + t[2];
}
FE_HD void fe_make_frame(float* F) {
  float* x = F;
  float* y = F + 3;
  float* z = F + 6;
  v3normalize(x);
  if (fabsf(x[1]) < 0.5f) { y[0] = 0.f; y[1] = 1.f; y[2] = 0.f; } else { y[0] = 0.f; y[1] = 0.f; y[2] = 1.f; }
  float dt = v3dot(x, y);
  v3madd(y, y, x, -dt);
  v3normalize(y);
  v3cross(z, x, y);
}

// The slice keeps the normal and the first tangent of a contact frame (6 words); the second tangent is their cross product
// (fe_make_frame builds it exactly so), recomputed where the frame is read: 3 words per contact buy 4 more contacts of capacity.
FE_HD void fe_frame_load(const FeWarp* w, int c, float* F) {
  const float* s = w->c_frame() + 6 * c;
#pragma unroll
  for (int k = 0; k < 6; ++k) F[k] = s[k];
  v3cross(F + 6, F, F + 3);
}

FE_FN void fe_assemble(FeWarp* w) {
  const fe_model* m = w->m;
  const int ncon = w->u()[FE_U_NCON], nr = m->nr, ne = m->neq;
  const float h = m->timestep;
  LANES_BEGIN
    for (int c = lane; c < ncon; c += 32) {
      const int g1 = w->c_geom()[c] & 255, g2 = w->c_geom()[c] >> 8;
      const int A = m->geom_link[g1], B = m->geom_link[g2];
      w->c_link()[c] = (A + 1) | ((B + 1) << 8);
      { // 0: one free part against the static world; 1: robot only; 2: robot against a part; 3: part against part (2, 3 couple moving blocks)
        const int nrl_ = m->nrlink;
        const bool pa = A >= nrl_, pb = B >= nrl_;
        w->c_kind()[c] = ((pa && B < 0) || (pb && A < 0)) ? 0 : ((pa && pb) ? 3 : ((pa || pb) ? 2 : 1));
      }
      float F[9];
      v3cpy(F, w->c_frame() + 6 * c);
      fe_make_frame(F);
      for (int k = 0; k < 6; ++k) w->c_frame()[6 * c + k] = F[k];
      const float fric = fmaxf(fmaxf(m->geom_friction[g1], m->geom_friction[g2]), 1e-5f);
      float sr[2], si[3];
      const float *s1 = m->geom_solref[g1], *s2 = m->geom_solref[g2];
      if (s1[0] > 0.f && s2[0] > 0.f) { sr[0] = 0.5f * (s1[0] + s2[0]); sr[1] = 0.5f * (s1[1] + s2[1]); }
      else { sr[0] = fminf(s1[0], s2[0]); sr[1] = fminf(s1[1], s2[1]); }
      for (int k = 0; k < 3; ++k) si[k] = 0.5f * (m->geom_solimp[g1][k] + m->geom_solimp[g2][k]);
      const float dist = w->c_dist()[c] - (m->has_margin ? fmaxf(m->geom_margin[g1], m->geom_margin[g2]) : 0.f); // efc_pos - efc_margin
      const float imp = fe_impedance(si, fabsf(dist));
      float kk, bb;
      fe_kb(sr, si[1], h, &kk, &bb);
      const float diag = fmaxf(m->geom_invweight[g1] + m->geom_invweight[g2], FE_MINVAL);
      const float R0 = fmaxf((1.f - imp) / imp * diag, FE_MINVAL);
      const float R1 = fmaxf(R0 / m->impratio, FE_MINVAL);
      w->c_D()[2 * c] = 1.f / R0;
      w->c_D()[2 * c + 1] = 1.f / R1;
      w->c_mu()[c] = fric * sqrtf(R1 / R0);
      w->c_fric()[c] = fric;
      float vA[3], vB[3], dv[3];
      fe_point_vel(w, w->lvel(), A, w->c_pos() + 3 * c, vA);
      fe_point_vel(w, w->lvel(), B, w->c_pos() + 3 * c, vB);
      v3sub(dv, vB, vA);
      w->c_aref()[3 * c] = -bb * v3dot(F, dv) - kk * imp * dist;
      w->c_aref()[3 * c + 1] = -bb * v3dot(F + 3, dv);
      w->c_aref()[3 * c + 2] = -bb * v3dot(F + 6, dv);
    }
    // weld rows
    for (int e = lane; e < ne; e += 32) {
      if (!w->eq_active()[e]) continue;
      const int A = m->eq_link1[e], B = m->eq_link2[e];
      const float* data = w->eq_data() + 7 * e;
      float r1[3], p1[3], err[6];
      m3mulv(r1, w->lmat() + 9 * A, data);
      v3add(p1, w->lpos() + 3 * A, r1);
      v3sub(err, p1, w->lpos() + 3 * B);
      float quat[4], qc[4], qe[4];
      qmul(quat, w->lquat() + 4 * A, data + 3);
      qc[0] = w->lquat()[4 * B]; qc[1] = -w->lquat()[4 * B + 1]; qc[2] = -w->lquat()[4 * B + 2]; qc[3] = -w->lquat()[4 * B + 3];
      qmul(qe, qc, quat);
      err[3] = qe[1]; err[4] = qe[2]; err[5] = qe[3];
      float G[9];
      for (int j = 0; j < 3; ++j) {
        float ax[4] = {0.f, j == 0 ? 1.f : 0.f, j == 1 ? 1.f : 0.f, j == 2 ? 1.f : 0.f}, t1[4], t2[4];
        qmul(t1, qc, ax);
        qmul(t2, t1, quat);
        G[0 + j] = 0.5f * t2[1]; G[3 + j] = 0.5f * t2[2]; G[6 + j] = 0.5f * t2[3];
      }
      v3cpy(w->w_r1() + 3 * e, r1);
      for (int k = 0; k < 9; ++k) w->w_G()[9 * e + k] = G[k];
      const float *VA = w->lvel() + 6 * A, *VB = w->lvel() + 6 * B;
      float vel[6], t[3], dw[3];
      v3cross(t, VA, r1);
      for (int k = 0; k < 3; ++k) vel[k] = VA[3 + k] + t[k] - VB[3 + k];
      v3sub(dw, VA, VB);
      m3mulv(vel + 3, G, dw);
      float kk, bb;
      fe_kb(m->eq_solref[e], m->eq_solimp[e][1], h, &kk, &bb);
      for (int k = 0; k < 6; ++k) {
        const float imp = fe_impedance(m->eq_solimp[e], fabsf(err[k]));
        const float diag = fmaxf(k < 3 ? m->eq_invw_t[e] : m->eq_invw_r[e], FE_MINVAL);
        const float R = fmaxf((1.f - imp) / imp * diag, FE_MINVAL);
        w->w_D()[6 * e + k] = 1.f / R;
        w->w_aref()[6 * e + k] = -bb * vel[k] - kk * imp * err[k];
      }
    }
    // joint limits
    for (int d = lane; d < nr; d += 32) {
      float sgn = 0.f, dist = 0.f;
      if (m->rdof_limited[d]) {
        const float q = w->qpos()[d];
        if (q - m->rdof_range[d][0] < 0.f) { sgn = 1.f; dist = q - m->rdof_range[d][0]; }
        else if (m->rdof_range[d][1] - q < 0.f) { sgn = -1.f; dist = m->rdof_range[d][1] - q; }
      }
      w->l_sign()[d] = sgn;
      if (sgn != 0.f) {
        const float imp = fe_impedance(m->rdof_solimp[d], fabsf(dist));
        float kk, bb;
        fe_kb(m->rdof_solref[d], m->rdof_solimp[d][1], h, &kk, &bb);
        const float R = fmaxf((1.f - imp) / imp * fmaxf(m->rdof_invweight[d], FE_MINVAL), FE_MINVAL);
        w->l_D()[d] = 1.f / R;
        w->l_aref()[d] = -bb * sgn * w->qvel()[d] - kk * imp * dist;
      } else { w->l_D()[d] = 0.f; w->l_aref()[d] = 0.f; }
    }
  LANES_END
}

// ---------------------------------------------------------------- solver pieces
// Zone logic of one elliptic contact, inlined (outputs stay in registers): forces f, cost, and with WANTW the 3x3 weight
// (xx yy zz xy xz yz); returns the state
template <bool WANTW>
FE_HD int fe_cone_t(float j0, float j1, float j2, float mu, float fr, float D0, float D1, float* f, float* cost, float* W) {
  const float N = j0 * mu, U1 = j1 * fr, U2 = j2 * fr, T = sqrtf(U1 * U1 + U2 * U2);
  if (N >= mu * T || (T <= 0.f && N >= 0.f)) { f[0] = f[1] = f[2] = 0.f; if (WANTW) { W[0] = W[1] = W[2] = W[3] = W[4] = W[5] = 0.f; } return 0; }
  if (mu * N + T <= 0.f || (T <= 0.f && N < 0.f)) {
    f[0] = -D0 * j0; f[1] = -D1 * j1; f[2] = -D1 * j2;
    *cost += 0.5f * (D0 * j0 * j0 + D1 * (j1 * j1 + j2 * j2));
    if (WANTW) { W[0] = D0; W[1] = D1; W[2] = D1; W[3] = W[4] = W[5] = 0.f; }
    return 1;
  }
  const float Dm = D0 / (mu * mu * (1.f + mu * mu)), NmT = N - mu * T;
  *cost += 0.5f * Dm * NmT * NmT;
  f[0] = -Dm * NmT * mu;
  f[1] = -f[0] / T * U1 * fr;
  f[2] = -f[0] / T * U2 * fr;
  if (WANTW) {
    const float iT = 1.f / T, a = Dm * mu * mu * iT * iT, b = Dm * NmT * mu * iT;
    const float h11 = a * U1 * U1 - b * (1.f - U1 * U1 * iT * iT), h22 = a * U2 * U2 - b * (1.f - U2 * U2 * iT * iT), h12 = a * U1 * U2 + b * U1 * U2 * iT * iT;
    const float h01 = -Dm * mu * U1 * iT, h02 = -Dm * mu * U2 * iT;
    W[0] = mu * mu * Dm; W[1] = fr * fr * h11; W[2] = fr * fr * h22; W[3] = mu * fr * h01; W[4] = mu * fr * h02; W[5] = fr * fr * h12;
  }
  return 2;
}
// One contact's terms of p'(alpha) and p''(alpha) along the search direction: rows j + alpha v, with v the rows of the
// direction.  They are applied to d1 / d2 with `op` (= or +=) inside each zone; the zone without force leaves d1 / d2 alone.
// A macro rather than a function that returns the terms: fe_line_eval's += then stays inside each zone's expression, as
// the product it may be fused with, instead of becoming a separate add after the branch.
#define FE_CONE_LS(j, v, alpha, mu_, fr_, D0_, D1_, d1, op, d2)                                                                    \
  {                                                                                                                                \
    const float *cj_ = (j), *cv_ = (v);                                                                                            \
    const float al = (alpha), mu = (mu_), fr = (fr_), D0 = (D0_), D1 = (D1_);                                                      \
    const float v0 = cv_[0], v1 = cv_[1], v2 = cv_[2];                                                                             \
    const float x0 = cj_[0] + al * v0, x1 = cj_[1] + al * v1, x2 = cj_[2] + al * v2;                                               \
    const float N = x0 * mu, U1 = x1 * fr, U2 = x2 * fr, T = sqrtf(U1 * U1 + U2 * U2);                                             \
    if (N >= mu * T || (T <= 0.f && N >= 0.f)) {                                                                                   \
    } else if (mu * N + T <= 0.f || (T <= 0.f && N < 0.f)) {                                                                       \
      d1 op D0 * x0 * v0 + D1 * (x1 * v1 + x2 * v2);                                                                               \
      d2 op D0 * v0 * v0 + D1 * (v1 * v1 + v2 * v2);                                                                               \
    } else {                                                                                                                       \
      const float Dm = D0 / (mu * mu * (1.f + mu * mu)), NmT = N - mu * T, N1 = v0 * mu, V1 = v1 * fr, V2 = v2 * fr;               \
      const float T1 = (U1 * V1 + U2 * V2) / T, T2 = (V1 * V1 + V2 * V2 - T1 * T1) / T, a = N1 - mu * T1;                          \
      d1 op Dm * NmT * a;                                                                                                          \
      d2 op Dm * (a * a - NmT * mu * T2);                                                                                          \
    }                                                                                                                              \
  }

// Exact line search along the Newton direction: safeguarded Newton on p'(alpha) = 0.  p' is only piecewise smooth (rows
// change cone zone along the ray): a Newton step is kept only while it at least halves the previous one (rtsafe rule),
// otherwise bisect -- else the iterates can hop between the two ends of the bracket and shrink it by almost nothing.
// The caller evaluates p'(alpha), p''(alpha) and passes them to start() for the first evaluation (alpha = 0) and to step()
// after that; both return false when the search is over.  alpha stays 0 when the direction is not a descent direction.
struct FeLineSearch {
  float alpha = 0.f, p1_0 = 0.f, lo = 0.f, hi = -1.f, dxold = 0.f;
  FE_MEMBER bool start(float p1, float p2) {
    if (!(p1 < 0.f) || !(p2 > 0.f)) return false;
    p1_0 = p1;
    alpha = -p1 / p2;
    dxold = alpha;
    return true;
  }
  FE_MEMBER bool step(float p1, float p2) {
    if (fabsf(p1) <= FE_LS_TOL * fabsf(p1_0)) return false;
    if (p1 < 0.f) lo = alpha; else hi = alpha;
    float next = alpha - p1 / p2;
    if (hi > 0.f && (!(next > lo && next < hi) || fabsf(2.f * p1) > fabsf(dxold * p2))) next = 0.5f * (lo + hi);
    if (hi < 0.f && !(next > lo)) next = 2.f * alpha;
    const bool more = !(fabsf(next - alpha) <= 1e-6f * fabsf(alpha)); // relative step below 1e-6: take it and stop
    dxold = fabsf(next - alpha);
    alpha = next;
    return more;
  }
  // predicted decrease of the cost, -alpha p'(0) / 2 (exact for a quadratic): the improvement of the Newton stop test
  FE_MEMBER float impr() const { return -0.5f * alpha * p1_0; }
};
// Newton stop test on the scaled improvement of the last step and the scaled gradient norm, then the iteration limit
FE_HD bool fe_newton_stop(int iter, int maxit, float scale, float impr, float gnorm, float tol) {
  if (iter > 0 ? (scale * impr < tol || scale * gnorm < tol) : scale * gnorm < tol) return true;
  return iter >= maxit;
}

// Weld rows of weld e under the link accelerations staged in lacc2: v_A + w_A x r1 - v_B, then G (w_A - w_B)
FE_HD void fe_weld_rows(const FeWarp* w, int e, float* r) {
  const float *XA = w->lacc2() + 6 * w->m->eq_link1[e], *XB = w->lacc2() + 6 * w->m->eq_link2[e];
  float t[3], dw[3];
  v3cross(t, XA, w->w_r1() + 3 * e);
  for (int k = 0; k < 3; ++k) r[k] = XA[3 + k] + t[k] - XB[3 + k];
  v3sub(dw, XA, XB);
  m3mulv(r + 3, w->w_G() + 9 * e, dw);
}
// Wr += the wrench of weld e's force w_f on link l (about the link's reference point), if l is one of its two links
FE_HD void fe_weld_wrench(const FeWarp* w, int e, int l, float* Wr) {
  const int A = w->m->eq_link1[e], B = w->m->eq_link2[e];
  if (A != l && B != l) return;
  const float* f = w->w_f() + 6 * e;
  float tq[3], t[3];
  m3tmulv(tq, w->w_G() + 9 * e, f + 3); // G^T f_rot
  if (A == l) {
    v3cross(t, w->w_r1() + 3 * e, f);
    Wr[0] += t[0] + tq[0]; Wr[1] += t[1] + tq[1]; Wr[2] += t[2] + tq[2]; Wr[3] += f[0]; Wr[4] += f[1]; Wr[5] += f[2];
  } else {
    Wr[0] -= tq[0]; Wr[1] -= tq[1]; Wr[2] -= tq[2]; Wr[3] -= f[0]; Wr[4] -= f[1]; Wr[5] -= f[2];
  }
}
// out = M_z in
FE_FN void fe_mul_M(FeWarp* w, const float* in, float* out) {
  const fe_model* m = w->m;
  const int nr = m->nr, np = m->npart, nrl = m->nrlink;
  LANES_BEGIN
    for (int d = lane; d < nr; d += 32) {
      float s = 0.f;
      for (int j = 0; j < nr; ++j) s += w->Mr()[d * nr + j] * in[j];
      out[d] = s;
    }
    for (int p = lane; p < np; p += 32) inert_mulv(out + nr + 6 * p, w->linert() + 10 * (nrl + p), in + nr + 6 * p);
  LANES_END
}
// rows = J_z in  (contacts -> cout[3*c..], welds -> wout[6*e..], limits -> lout[d]); `sub_aref` subtracts aref
FE_FN void fe_mul_J(FeWarp* w, const float* in, float* cout, float* wout, float* lout, bool sub_aref) {
  const fe_model* m = w->m;
  const int nr = m->nr, nrl = m->nrlink, nl = m->nlink, ncon = w->u()[FE_U_NCON], ne = m->neq;
  LANES_BEGIN
    const int l = lane;
    if (l < nl) {
      float X[6] = {0, 0, 0, 0, 0, 0};
      if (l < nrl) {
        const int mask = m->link_ancmask[l];
        for (int d = 0; d < nr; ++d)
          if ((mask >> d) & 1) { const float xd = in[d]; for (int k = 0; k < 6; ++k) X[k] += w->S()[6 * d + k] * xd; }
      } else for (int k = 0; k < 6; ++k) X[k] = in[nr + 6 * (l - nrl) + k];
      for (int k = 0; k < 6; ++k) w->lacc2()[6 * l + k] = X[k];
    }
  LANES_END
  LANES_BEGIN
    for (int c = lane; c < ncon; c += 32) {
      const int A = (w->c_link()[c] & 255) - 1, B = (w->c_link()[c] >> 8) - 1;
      float aA[3], aB[3], da[3];
      fe_point_vel(w, w->lacc2(), A, w->c_pos() + 3 * c, aA);
      fe_point_vel(w, w->lacc2(), B, w->c_pos() + 3 * c, aB);
      v3sub(da, aB, aA);
      float F[9];
      fe_frame_load(w, c, F);
      for (int k = 0; k < 3; ++k) cout[3 * c + k] = v3dot(F + 3 * k, da) - (sub_aref ? w->c_aref()[3 * c + k] : 0.f);
    }
    for (int e = lane; e < ne; e += 32) {
      if (!w->eq_active()[e]) continue;
      float r[6];
      fe_weld_rows(w, e, r);
      for (int k = 0; k < 6; ++k) wout[6 * e + k] = r[k] - (sub_aref ? w->w_aref()[6 * e + k] : 0.f);
    }
    for (int d = lane; d < nr; d += 32) lout[d] = w->l_sign()[d] * in[d] - (sub_aref ? w->l_aref()[d] : 0.f);
  LANES_END
}
// constraint forces/states from jar; returns the constraint cost
FE_FN float fe_update(FeWarp* w) {
  const fe_model* m = w->m;
  const int ncon = w->u()[FE_U_NCON], ne = m->neq, nr = m->nr;
  LANES_BEGIN
    float cost = 0.f;
    for (int c = lane; c < ncon; c += 32) {
      float f[3];
      const int st = fe_cone_t<false>(w->c_jar()[3 * c], w->c_jar()[3 * c + 1], w->c_jar()[3 * c + 2], w->c_mu()[c], w->c_fric()[c], w->c_D()[2 * c], w->c_D()[2 * c + 1], f, &cost, nullptr);
      w->c_f()[3 * c] = f[0]; w->c_f()[3 * c + 1] = f[1]; w->c_f()[3 * c + 2] = f[2];
      w->c_state()[c] = st;
    }
    for (int e = lane; e < ne; e += 32) {
      if (!w->eq_active()[e]) continue;
      for (int k = 0; k < 6; ++k) {
        const float D = w->w_D()[6 * e + k], j = w->w_jar()[6 * e + k];
        w->w_f()[6 * e + k] = -D * j;
        cost += 0.5f * D * j * j;
      }
    }
    for (int d = lane; d < nr; d += 32) {
      float f = 0.f;
      if (w->l_sign()[d] != 0.f && w->l_jar()[d] < 0.f) { f = -w->l_D()[d] * w->l_jar()[d]; cost += 0.5f * w->l_D()[d] * w->l_jar()[d] * w->l_jar()[d]; }
      w->l_f()[d] = f;
    }
    w->scr()[lane] = cost;
  LANES_END
  return fe_sum32(w->scr());
}
// out = J_z^T force
FE_FN void fe_mul_JT(FeWarp* w, float* out) {
  const fe_model* m = w->m;
  const int nr = m->nr, nrl = m->nrlink, nl = m->nlink, ncon = w->u()[FE_U_NCON], ne = m->neq;
  LANES_BEGIN
    const int l = lane;
    if (l < nl) {
      float P[3], Wr[6] = {0, 0, 0, 0, 0, 0};
      fe_link_ref(w, l, P);
      for (int c = 0; c < ncon; ++c) {
        if (w->c_state()[c] == 0) continue;
        const int A = (w->c_link()[c] & 255) - 1, B = (w->c_link()[c] >> 8) - 1;
        if (A != l && B != l) continue;
        const float sg = (B == l ? 1.f : 0.f) - (A == l ? 1.f : 0.f);
        if (sg == 0.f) continue;
        float F[9];
      fe_frame_load(w, c, F);
        const float *f = w->c_f() + 3 * c;
        float fw[3] = {F[0] * f[0] + F[3] * f[1] + F[6] * f[2], F[1] * f[0] + F[4] * f[1] + F[7] * f[2], F[2] * f[0] + F[5] * f[1] + F[8] * f[2]};
        float r[3], t[3];
        v3sub(r, w->c_pos() + 3 * c, P);
        v3cross(t, r, fw);
        Wr[0] += sg * t[0]; Wr[1] += sg * t[1]; Wr[2] += sg * t[2]; Wr[3] += sg * fw[0]; Wr[4] += sg * fw[1]; Wr[5] += sg * fw[2];
      }
      for (int e = 0; e < ne; ++e)
        if (w->eq_active()[e]) fe_weld_wrench(w, e, l, Wr);
      for (int k = 0; k < 6; ++k) w->lacc2()[6 * l + k] = Wr[k];
      if (l >= nrl) for (int k = 0; k < 6; ++k) out[nr + 6 * (l - nrl) + k] = Wr[k];
    }
  LANES_END
  LANES_BEGIN
    for (int d = lane; d < nr; d += 32) {
      float s = w->l_sign()[d] * w->l_f()[d];
      for (int l = d; l < nrl; ++l)
        if ((m->link_ancmask[l] >> d) & 1) s += dot6(w->S() + 6 * d, w->lacc2() + 6 * l);
      out[d] = s;
    }
  LANES_END
}

// one 1-D cost evaluation along the search direction: returns p'(alpha), p''(alpha) (uniform)
FE_FN void fe_line_eval(FeWarp* w, float alpha, float g1, float g2, float* d1, float* d2) {
  const fe_model* m = w->m;
  const int ncon = w->u()[FE_U_NCON], ne = m->neq, nr = m->nr;
  LANES_BEGIN
    float p1 = 0.f, p2 = 0.f;
    for (int c = lane; c < ncon; c += 32) {
      FE_CONE_LS(w->c_jar() + 3 * c, w->c_jv() + 3 * c, alpha, w->c_mu()[c], w->c_fric()[c], w->c_D()[2 * c], w->c_D()[2 * c + 1], p1, +=, p2)
    }
    for (int e = lane; e < ne; e += 32) {
      if (!w->eq_active()[e]) continue;
      for (int k = 0; k < 6; ++k) {
        const float D = w->w_D()[6 * e + k], v = w->w_jv()[6 * e + k], x = w->w_jar()[6 * e + k] + alpha * v;
        p1 += D * x * v; p2 += D * v * v;
      }
    }
    for (int d = lane; d < nr; d += 32) {
      if (w->l_sign()[d] == 0.f) continue;
      const float v = w->l_jv()[d], x = w->l_jar()[d] + alpha * v;
      if (x < 0.f) { p1 += w->l_D()[d] * x * v; p2 += w->l_D()[d] * v * v; }
    }
    w->scr()[lane] = p1; w->scr()[32 + lane] = p2;
  LANES_END
  *d1 = fe_sum32(w->scr()) + g1 + 2.f * alpha * g2;
  *d2 = fe_sum32(w->scr() + 32) + 2.f * g2;
}

// rows of one part-vs-world contact in the part's coordinates: J[k] = sgn * [(r x F_k), F_k], r = pos - origin
FE_HD void fe_part_rows(const FeWarp* w, int c, int l, float sgn, float* J) {
  float F[9];
      fe_frame_load(w, c, F);
  float r[3];
  v3sub(r, w->c_pos() + 3 * c, w->lpos() + 3 * l);
  for (int k = 0; k < 3; ++k) {
    float t[3];
    v3cross(t, r, F + 3 * k);
    J[6 * k + 0] = sgn * t[0]; J[6 * k + 1] = sgn * t[1]; J[6 * k + 2] = sgn * t[2];
    J[6 * k + 3] = sgn * F[3 * k]; J[6 * k + 4] = sgn * F[3 * k + 1]; J[6 * k + 5] = sgn * F[3 * k + 2];
  }
}

// 3x3 weight of an active contact: diag(D) in the quadratic zone (st 1), cone Hessian in the middle zone (st 2)
FE_HD void fe_contact_weight(const FeWarp* w, int c, int st, float* W) {
  const float mu = w->c_mu()[c], fr = w->c_fric()[c], D0 = w->c_D()[2 * c], D1 = w->c_D()[2 * c + 1];
  if (st == 1) { W[0] = D0; W[4] = D1; W[8] = D1; W[1] = W[2] = W[3] = W[5] = W[6] = W[7] = 0.f; }
  else {
    const float N = w->c_jar()[3 * c] * mu, U[3] = {N, w->c_jar()[3 * c + 1] * fr, w->c_jar()[3 * c + 2] * fr};
    const float T = sqrtf(U[1] * U[1] + U[2] * U[2]), Dm = D0 / (mu * mu * (1.f + mu * mu)), NmT = N - mu * T;
    const float sc[3] = {mu, fr, fr};
    float HU[9];
    HU[0] = Dm;
    for (int a = 1; a < 3; ++a) HU[a] = HU[3 * a] = -Dm * mu * U[a] / T;
    for (int a = 1; a < 3; ++a)
      for (int b = 1; b < 3; ++b) HU[3 * a + b] = Dm * mu * mu * U[a] * U[b] / (T * T) - Dm * NmT * mu * ((a == b ? 1.f : 0.f) / T - U[a] * U[b] / (T * T * T));
    for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) W[3 * a + b] = sc[a] * HU[3 * a + b] * sc[b];
  }
}
// twist [angular; linear at p0] that a unit of dof z (solver coordinates) gives the link pair (A, B), B side minus A side.
// mA / mB are the robot ancestor masks of A / B (0 for a part or the world).
FE_HD void fe_unit_twist(const FeWarp* w, int z, int A, int B, int mA, int mB, const float* p0, const float* Pr, float* d) {
  const int nr = w->m->nr, nrl = w->m->nrlink;
#pragma unroll
  for (int q = 0; q < 6; ++q) d[q] = 0.f;
  if (z >= 0 && z < nr) {
    const float sg = (float)((mB >> z) & 1) - (float)((mA >> z) & 1);
    if (sg != 0.f) {
      const float* S = w->S() + 6 * z;
      const float r[3] = {p0[0] - Pr[0], p0[1] - Pr[1], p0[2] - Pr[2]};
      float t[3];
      v3cross(t, S, r);
      d[0] = sg * S[0]; d[1] = sg * S[1]; d[2] = sg * S[2]; d[3] = sg * (S[3] + t[0]); d[4] = sg * (S[4] + t[1]); d[5] = sg * (S[5] + t[2]);
    }
  } else if (z >= nr) {
    const int part = (z - nr) / 6, jj = (z - nr) % 6, l = nrl + part;
    const float sg = l == B ? 1.f : (l == A ? -1.f : 0.f);
    if (sg != 0.f) {
      if (jj < 3) {
        const float e[3] = {jj == 0 ? 1.f : 0.f, jj == 1 ? 1.f : 0.f, jj == 2 ? 1.f : 0.f};
        const float r[3] = {p0[0] - w->lpos()[3 * l], p0[1] - w->lpos()[3 * l + 1], p0[2] - w->lpos()[3 * l + 2]};
        float t[3];
        v3cross(t, e, r);
        d[0] = sg * e[0]; d[1] = sg * e[1]; d[2] = sg * e[2]; d[3] = sg * t[0]; d[4] = sg * t[1]; d[5] = sg * t[2];
      } else { d[3] = jj == 3 ? sg : 0.f; d[4] = jj == 4 ? sg : 0.f; d[5] = jj == 5 ? sg : 0.f; } // selects keep d in registers
    }
  }
}

// fe_cone_t<true> behind a call, for fe_build_H's grouped block: inlined there it changes the last bits of the
// cooperative solver's results on sm_90a, so it stays out of line as it always was
FE_HDN int fe_cone(float j0, float j1, float j2, float mu, float fr, float D0, float D1, float* f, float* cost, float* W) {
  return fe_cone_t<true>(j0, j1, j2, mu, fr, D0, D1, f, cost, W);
}
// H = M_z + J^T W J  (packed lower, skyline first[]).  With regs set, the contacts that couple moving blocks are left to
// fe_newton_regs (they are added to the register-resident rows there).
FE_FN void fe_build_H(FeWarp* w, bool regs = false) {
  const fe_model* m = w->m;
  const int nr = m->nr, nrl = m->nrlink, np = m->npart, nv = m->nv, ncon = w->u()[FE_U_NCON], ne = m->neq;
  // envelope: a part row starts at its own block unless it is coupled to the robot or to a lower part
  LANES_BEGIN
    for (int d = lane; d < nr; d += 32) w->first()[d] = 0;
    for (int p = lane; p < np; p += 32) {
      const int l = nrl + p;
      int f = nr + 6 * p;
      for (int c = 0; c < ncon; ++c) {
        if (w->c_state()[c] == 0) continue;
        const int A = (w->c_link()[c] & 255) - 1, B = (w->c_link()[c] >> 8) - 1;
        int o = -2;
        if (A == l) o = B; else if (B == l) o = A;
        if (o < 0) continue;
        const int fo = o < nrl ? 0 : nr + 6 * (o - nrl);
        if (fo < f) f = fo;
      }
      for (int e = 0; e < ne; ++e) {
        if (!w->eq_active()[e]) continue;
        const int A = m->eq_link1[e], B = m->eq_link2[e];
        int o = -1;
        if (A == l) o = B; else if (B == l) o = A;
        if (o < 0) continue;
        const int fo = nr + 6 * (o - nrl);
        if (fo < f) f = fo;
      }
      for (int k = 0; k < 6; ++k) w->first()[nr + 6 * p + k] = f;
    }
  LANES_END
  // M_z inside the envelope
  LANES_BEGIN
    for (int i = lane; i < nv; i += 32) {
      float* Hi = w->H() + fe_tri(i);
      for (int j = w->first()[i]; j <= i; ++j) Hi[j] = 0.f;
      if (i < nr) { for (int j = 0; j <= i; ++j) Hi[j] = w->Mr()[i * nr + j]; if (w->l_sign()[i] != 0.f && w->l_jar()[i] < 0.f) Hi[i] += w->l_D()[i]; }
      else {
        const int p = (i - nr) / 6, r = (i - nr) % 6;
        float A[21];
        fe_inert_sym6(A, w->linert() + 10 * (nrl + p), 0.f);
        for (int c = 0; c <= r; ++c) Hi[nr + 6 * p + c] = A[fe_tri(r) + c];
      }
    }
  LANES_END
  // contacts of a free part against the static world only touch that part's 6x6 diagonal block; unless a part has more
  // than 8 of them, they are accumulated 8 lanes per part (lane = contact) with group reductions, like fe_solve_parts_grouped
  bool grouped = true;
  for (int p = 0; p < np; ++p) if (w->plist()[9 * p + 8] > 8) grouped = false;
  if (grouped) {
    for (int pass = 0; pass * 4 < np; ++pass) {
      FE_PRIVA(float, hacc_, 21);
      LANES_BEGIN
        for (int k = 0; k < 21; ++k) PV(hacc_)[k] = 0.f;
        const int part = pass * 4 + (lane >> 3), slot = lane & 7;
        if (part < np && slot < w->plist()[9 * part + 8]) {
          const int c = w->plist()[9 * part + slot];
          if (w->c_state()[c] != 0) {
            const int l = nrl + part, B_ = (w->c_link()[c] >> 8) - 1;
            float J[18], f[3], W[6], dummy = 0.f, WJ[18];
            fe_part_rows(w, c, l, B_ == l ? 1.f : -1.f, J);
            fe_cone(w->c_jar()[3 * c], w->c_jar()[3 * c + 1], w->c_jar()[3 * c + 2], w->c_mu()[c], w->c_fric()[c], w->c_D()[2 * c], w->c_D()[2 * c + 1], f, &dummy, W);
            for (int i = 0; i < 6; ++i) {
              WJ[i] = W[0] * J[i] + W[3] * J[6 + i] + W[4] * J[12 + i];
              WJ[6 + i] = W[3] * J[i] + W[1] * J[6 + i] + W[5] * J[12 + i];
              WJ[12 + i] = W[4] * J[i] + W[5] * J[6 + i] + W[2] * J[12 + i];
            }
            for (int i = 0; i < 6; ++i)
              for (int j = 0; j <= i; ++j) PV(hacc_)[i * (i + 1) / 2 + j] = J[i] * WJ[j] + J[6 + i] * WJ[6 + j] + J[12 + i] * WJ[12 + j];
          }
        }
      LANES_END
      FE_GSUM8_ARR(hacc_, 21);
      LANES_BEGIN
        const int part = pass * 4 + (lane >> 3);
        if (part < np && (lane & 7) == 0 && w->plist()[9 * part + 8] > 0) {
          const int z = nr + 6 * part;
          for (int i = 0; i < 6; ++i) for (int j = 0; j <= i; ++j) w->H()[fe_tri(z + i) + z + j] += PV(hacc_)[i * (i + 1) / 2 + j];
        }
      LANES_END
    }
  }
  // remaining contacts, one at a time: dof-space rows staged in Jc (3 x ncols), then the ncols x ncols outer product
  for (int c = 0; c < ncon && !regs; ++c) {
    const int st = w->c_state()[c];
    if (st == 0 || (grouped && w->c_kind()[c] == 0)) continue;
    const int A = (w->c_link()[c] & 255) - 1, B = (w->c_link()[c] >> 8) - 1;
    const bool robot = (A >= 0 && A < nrl) || (B >= 0 && B < nrl);
    const int partA = A >= nrl ? A - nrl : -1, partB = B >= nrl ? B - nrl : -1;
    const int ncols = (robot ? nr : 0) + (partA >= 0 ? 6 : 0) + (partB >= 0 ? 6 : 0);
    float W[9];
    fe_contact_weight(w, c, st, W);
    LANES_BEGIN
      const int j = lane;
      if (j < ncols) {
        float F[9];
      fe_frame_load(w, c, F);
        const float* p = w->c_pos() + 3 * c;
        float col[3] = {0.f, 0.f, 0.f};
        int z;
        int jj = j;
        if (robot && jj < nr) {
          z = jj;
          const float sg = ((B >= 0 && B < nrl && ((m->link_ancmask[B] >> jj) & 1)) ? 1.f : 0.f) - ((A >= 0 && A < nrl && ((m->link_ancmask[A] >> jj) & 1)) ? 1.f : 0.f);
          if (sg != 0.f) {
            float r[3], t[3], v[3];
            v3sub(r, p, m->robot_ref);
            v3cross(t, w->S() + 6 * jj, r);
            v3add(v, w->S() + 6 * jj + 3, t);
            for (int k = 0; k < 3; ++k) col[k] = sg * v3dot(F + 3 * k, v);
          }
        } else {
          if (robot) jj -= nr;
          int part; float sg;
          if (partA >= 0 && jj < 6) { part = partA; sg = -1.f; } else { if (partA >= 0) jj -= 6; part = partB; sg = 1.f; }
          z = nr + 6 * part + jj;
          float r[3];
          v3sub(r, p, w->lpos() + 3 * (nrl + part));
          for (int k = 0; k < 3; ++k) {
            if (jj < 3) { float t[3]; v3cross(t, r, F + 3 * k); col[k] = sg * (jj == 0 ? t[0] : (jj == 1 ? t[1] : t[2])); }
            else col[k] = sg * (jj == 3 ? F[3 * k] : (jj == 4 ? F[3 * k + 1] : F[3 * k + 2])); // selects keep F in registers
          }
        }
        w->Jc()[j] = col[0]; w->Jc()[32 + j] = col[1]; w->Jc()[64 + j] = col[2];
        w->colmap()[j] = z;
      }
    LANES_END
    LANES_BEGIN
      for (int e = lane; e < fe_tri(ncols); e += 32) {
        int i = (int)((sqrtf(8.f * (float)e + 1.f) - 1.f) * 0.5f);
        while (fe_tri(i + 1) <= e) ++i;
        while (fe_tri(i) > e) --i;
        const int j = e - fe_tri(i);
        float v = 0.f;
        for (int a = 0; a < 3; ++a) {
          const float ja = w->Jc()[32 * a + i];
          if (ja == 0.f) continue;
          v += ja * (W[3 * a] * w->Jc()[j] + W[3 * a + 1] * w->Jc()[32 + j] + W[3 * a + 2] * w->Jc()[64 + j]);
        }
        if (v != 0.f) {
          int zi = w->colmap()[i], zj = w->colmap()[j];
          if (zi < zj) { int t = zi; zi = zj; zj = t; }
          w->H()[fe_tri(zi) + zj] += v;
        }
      }
    LANES_END
  }
  // welds: 6 rows over the two parts' 12 columns, diagonal weights (column map staged in iscr: colmap holds the active-dof list)
  for (int e = 0; e < ne; ++e) {
    if (!w->eq_active()[e]) continue;
    const int A = m->eq_link1[e], B = m->eq_link2[e];
    for (int half = 0; half < 2; ++half) { // rows 0-2 (translation) then 3-5 (rotation), staged 3 at a time
      LANES_BEGIN
        const int j = lane;
        if (j < 12) {
          const bool sideA = j < 6;
          const int jj = sideA ? j : j - 6;
          float col[3] = {0.f, 0.f, 0.f};
          if (half == 0) { // v_A + w_A x r1 - v_B
            if (sideA) {
              if (jj < 3) { // d/dw_A of (w_A x r1)_k = (e_jj x r1)_k
                float ej[3] = {jj == 0 ? 1.f : 0.f, jj == 1 ? 1.f : 0.f, jj == 2 ? 1.f : 0.f}, t[3];
                v3cross(t, ej, w->w_r1() + 3 * e);
                col[0] = t[0]; col[1] = t[1]; col[2] = t[2];
              } else col[jj - 3] = 1.f;
            } else if (jj >= 3) col[jj - 3] = -1.f;
          } else if (jj < 3) {
            const float sg = sideA ? 1.f : -1.f;
            for (int k = 0; k < 3; ++k) col[k] = sg * w->w_G()[9 * e + 3 * k + jj];
          }
          w->Jc()[j] = col[0]; w->Jc()[32 + j] = col[1]; w->Jc()[64 + j] = col[2];
          w->iscr()[j] = nr + 6 * ((sideA ? A : B) - nrl) + jj;
        }
      LANES_END
      LANES_BEGIN
        for (int en = lane; en < fe_tri(12); en += 32) {
          int i = (int)((sqrtf(8.f * (float)en + 1.f) - 1.f) * 0.5f);
          while (fe_tri(i + 1) <= en) ++i;
          while (fe_tri(i) > en) --i;
          const int j = en - fe_tri(i);
          float v = 0.f;
          for (int a = 0; a < 3; ++a) v += w->w_D()[6 * e + 3 * half + a] * w->Jc()[32 * a + i] * w->Jc()[32 * a + j];
          if (v != 0.f) {
            int zi = w->iscr()[i], zj = w->iscr()[j];
            if (zi < zj) { int t = zi; zi = zj; zj = t; }
            w->H()[fe_tri(zi) + zj] += v;
          }
        }
      LANES_END
    }
  }
}

// Newton direction of the active dofs (robot + coupled parts, at most 32): lane i owns row i of the lower triangle of H in
// registers.  Rows start from the slice copy (M_z, static-world contacts of the parts, welds, limits); the contacts that
// couple blocks are added as rank-6 updates whose columns travel by shuffle; FE_REG_CHOL_SOLVE factors and solves.  No slice
// traffic, no barriers inside.
// NMAX (16 / 24 / 32) bounds the unrolled loops; rows and columns beyond nA are padded with the identity.
template <int NMAX>
FE_FN void fe_newton_regs(FeWarp* w, int nA) {
  const int ncon = w->u()[FE_U_NCON];
  FE_PRIVA(float, row_, NMAX);
  FE_PRIV(float, b_); FE_PRIV(int, z_); FE_PRIV(int, bad_);
  REGS_BEGIN
    const int i = lane, zi = i < nA ? w->colmap()[i] : -1;
    PV(z_) = zi;
    const int fi = zi >= 0 ? w->first()[zi] : 0;
    const float* Hi = w->H() + fe_tri(zi >= 0 ? zi : 0);
#pragma unroll
    for (int j = 0; j < NMAX; ++j) {
      float v = (j == i) ? 1.f : 0.f;
      if (j <= i && i < nA) { const int zj = w->colmap()[j]; v = zj >= fi ? Hi[zj] : 0.f; }
      PV(row_)[j] = v;
    }
    PV(b_) = zi >= 0 ? -w->grad()[zi] : 0.f;
  REGS_END
  // Coupling contacts, grouped by the pair of links they join.  A contact row is G_c d, with d the 6-vector [angular; linear at
  // p0] that a unit of the dof contributes to the relative motion of the two links (B side minus A side) and
  // G_c = [(r_c x F_k)^T, F_k^T] (3 x 6, r_c = p_c - p0, p0 = the first contact point of the pair).  So the contacts of one
  // pair add d_i^T K d_j to H with ONE 6x6 matrix K = sum_c G_c^T W_c G_c: lane = contact builds its term, a warp sum per
  // entry of K, then a rank-6 update of the rows (6 shuffles per column) instead of a rank-3 update per contact.
  {
    const fe_model* m = w->m;
    const int nrl = m->nrlink;
    FE_PRIVA(float, kq_, 21);
    FE_PRIVA(float, d_, 6); FE_PRIVA(float, u_, 6);
    FE_PRIV(float, px_); FE_PRIV(float, py_); FE_PRIV(float, pz_); FE_PRIV(float, ox_); FE_PRIV(float, oy_); FE_PRIV(float, oz_);
    FE_PRIV(float, ks_); FE_PRIV(float, kf_);
    FE_PRIV(int, key_); FE_PRIV(int, lead_); FE_PRIV(int, isl_);
    for (int base = 0; base < ncon; base += 32) {
      REGS_BEGIN
        const int c = base + lane;
        int key = -1 - lane; // lanes without a coupling contact: keys that match nobody
        PV(px_) = PV(py_) = PV(pz_) = 0.f;
        if (c < ncon && w->c_state()[c] != 0 && w->c_kind()[c] != 0) {
          key = w->c_link()[c];
          PV(px_) = w->c_pos()[3 * c]; PV(py_) = w->c_pos()[3 * c + 1]; PV(pz_) = w->c_pos()[3 * c + 2];
        }
        PV(key_) = key;
      REGS_END
      FE_MATCH_LEADER(lead_, PV_ALL(key_));
      FE_SHFLV(ox_, PV_ALL(px_), PV_ALL(lead_)); FE_SHFLV(oy_, PV_ALL(py_), PV_ALL(lead_)); FE_SHFLV(oz_, PV_ALL(pz_), PV_ALL(lead_));
      REGS_BEGIN
        const int c = base + lane;
#pragma unroll
        for (int k = 0; k < 21; ++k) PV(kq_)[k] = 0.f;
        PV(isl_) = (PV(key_) >= 0 && PV(lead_) == lane) ? 1 : 0;
        if (PV(key_) >= 0) {
          float F[9], W[9], G[18], WG[18];
          fe_frame_load(w, c, F);
          fe_contact_weight(w, c, w->c_state()[c], W);
          const float r[3] = {PV(px_) - PV(ox_), PV(py_) - PV(oy_), PV(pz_) - PV(oz_)};
#pragma unroll
          for (int k = 0; k < 3; ++k) { v3cross(G + 6 * k, r, F + 3 * k); G[6 * k + 3] = F[3 * k]; G[6 * k + 4] = F[3 * k + 1]; G[6 * k + 5] = F[3 * k + 2]; }
#pragma unroll
          for (int i = 0; i < 6; ++i) {
            WG[i] = W[0] * G[i] + W[1] * G[6 + i] + W[2] * G[12 + i];
            WG[6 + i] = W[3] * G[i] + W[4] * G[6 + i] + W[5] * G[12 + i];
            WG[12 + i] = W[6] * G[i] + W[7] * G[6 + i] + W[8] * G[12 + i];
          }
#pragma unroll
          for (int i = 0; i < 6; ++i)
#pragma unroll
            for (int j = 0; j <= i; ++j) PV(kq_)[i * (i + 1) / 2 + j] = G[i] * WG[j] + G[6 + i] * WG[6 + j] + G[12 + i] * WG[12 + j];
        }
      REGS_END
      unsigned todo = FE_BALLOTP(PV_ALL(isl_));
      while (todo) {
        int g = 0;
        while (!((todo >> g) & 1u)) ++g;
        todo &= todo - 1u;
        // uniform description of the pair: key, reference point
        FE_SHFL(ks_, PV_ALL(px_), g); const float p0x = FE_UNI(ks_);
        FE_SHFL(ks_, PV_ALL(py_), g); const float p0y = FE_UNI(ks_);
        FE_SHFL(ks_, PV_ALL(pz_), g); const float p0z = FE_UNI(ks_);
        REGS_BEGIN PV(kf_) = (float)PV(key_); REGS_END // link ids fit a float exactly (two bytes)
        FE_SHFL(ks_, PV_ALL(kf_), g);
        const int gkey = (int)FE_UNI(ks_), A = (gkey & 255) - 1, B = (gkey >> 8) - 1;
        const int mA = (A >= 0 && A < nrl) ? m->link_ancmask[A] : 0, mB = (B >= 0 && B < nrl) ? m->link_ancmask[B] : 0;
        const float p0[3] = {p0x, p0y, p0z};
        // this lane's dof: its unit contribution to the relative twist of the pair, at p0
        REGS_BEGIN fe_unit_twist(w, PV(z_), A, B, mA, mB, p0, m->robot_ref, PV(d_)); REGS_END
        // K d_i: entry by entry, K[a][b] = warp sum of the members' terms
#pragma unroll
        for (int k = 0; k < 6; ++k) { REGS_BEGIN PV(u_)[k] = 0.f; REGS_END }
#pragma unroll
        for (int a = 0; a < 6; ++a) {
#pragma unroll
          for (int b = 0; b <= a; ++b) {
            REGS_BEGIN PV(ks_) = ((float)PV(key_) == (float)gkey) ? PV(kq_)[a * (a + 1) / 2 + b] : 0.f; REGS_END
            FE_WSUM(ks_);
            REGS_BEGIN
              PV(u_)[a] += PV(ks_) * PV(d_)[b];
              if (a != b) PV(u_)[b] += PV(ks_) * PV(d_)[a];
            REGS_END
          }
        }
        // rank-6 update: row_i[j] += u_i . d_j
#pragma unroll
        for (int j = 0; j < NMAX; ++j) {
#pragma unroll
          for (int k = 0; k < 6; ++k) {
            FE_SHFLA(ks_, d_, k, j);
            REGS_BEGIN PV(row_)[j] += PV(u_)[k] * PV(ks_); REGS_END
          }
        }
      }
    }
  }
  FE_REG_CHOL_SOLVE(NMAX, row_, b_, bad_)
  LANES_BEGIN
    if (PV(z_) >= 0) w->search()[PV(z_)] = PV(b_);
    if (PV(bad_) && lane == 0) w->u()[FE_U_FLAGS] |= FE_FLAG_NEWTON_PIVOT;
  LANES_END
}

// cooperative Newton solve over all dofs.  cplmask: the parts that a constraint couples to another moving block (bit p for
// part p, as fe_solve decides it); they join the robot dofs in the register-resident Newton direction, the other parts are
// independent 6x6 blocks.
FE_FN void fe_solve_coop(FeWarp* w, unsigned cplmask) {
  FE_TICK_START
  const fe_model* m = w->m;
  const int nr = m->nr, nrl = m->nrlink, np = m->npart, nv = m->nv, ncon = w->u()[FE_U_NCON], ne = m->neq;
  // any constraint at all?
  LANES_BEGIN
    int any = lane < ncon;
    for (int e = lane; e < ne; e += 32) any |= w->eq_active()[e] != 0;
    for (int d = lane; d < nr; d += 32) any |= w->l_sign()[d] != 0.f;
    w->iscr()[lane] = any;
    for (int i = lane; i < nv; i += 32) w->fc()[i] = 0.f;
  LANES_END
  if (fe_ballot32(w->iscr()) == 0u) {
    LANES_BEGIN
      for (int i = lane; i < nv; i += 32) w->x()[i] = w->as()[i];
    LANES_END
    return;
  }
  LANES_BEGIN if (lane == 0) w->u()[FE_U_STAT + FE_STAT_NEWTON_SOLVES] += 1; LANES_END
  const float scale = 1.0f / (m->meaninertia * (float)(m->nv > 1 ? m->nv : 1));
  // warm start candidate (stored in qacc coordinates) -> z coordinates; pick the cheaper of warm / smooth.  The smooth
  // candidate is costed first: the warm start usually wins, and its products (Ma, jar) are then already in place.
  LANES_BEGIN
    for (int i = lane; i < nv; i += 32) w->search()[i] = w->as()[i];
    for (int d = lane; d < nr; d += 32) w->x()[d] = w->warm()[d];
    for (int p = lane; p < np; p += 32) {
      const int da = m->link_dadr[nrl + p], z = nr + 6 * p;
      m3mulv(w->x() + z, w->lmat() + 9 * (nrl + p), w->warm() + da + 3);
      v3cpy(w->x() + z + 3, w->warm() + da);
    }
  LANES_END
  float cost_smooth = 0.f, cost_warm = 0.f;
  for (int pass = 0; pass < 2; ++pass) {
    float* cand = pass == 0 ? w->search() : w->x();
    fe_mul_M(w, cand, w->Ma());
    fe_mul_J(w, cand, w->c_jar(), w->w_jar(), w->l_jar(), true);
    float cost = fe_update(w);
    LANES_BEGIN
      float s = 0.f;
      for (int i = lane; i < nv; i += 32) s += 0.5f * (w->Ma()[i] - w->fs()[i]) * (cand[i] - w->as()[i]);
      w->scr()[lane] = s;
    LANES_END
    cost += fe_sum32(w->scr());
    if (pass == 0) cost_smooth = cost; else cost_warm = cost;
  }
  if (cost_smooth < cost_warm || !(cost_warm == cost_warm)) { // the unconstrained acceleration is the better start: redo its products
    LANES_BEGIN for (int i = lane; i < nv; i += 32) w->x()[i] = w->as()[i]; LANES_END
    fe_mul_M(w, w->x(), w->Ma());
    fe_mul_J(w, w->x(), w->c_jar(), w->w_jar(), w->l_jar(), true);
  }
  // active set of the register-resident Newton direction: the robot dofs, then the coupled parts (fixed for the whole
  // solve); the remaining parts are independent 6x6 blocks (skip[] = 1)
  LANES_BEGIN
    if (lane == 0) {
      int n = 0;
      for (int d = 0; d < nr; ++d) { w->skip()[d] = 0; if (n < 32) w->colmap()[n] = d; ++n; }
      for (int p = 0; p < np; ++p) {
        const int cpl = (cplmask >> p) & 1u;
        for (int k = 0; k < 6; ++k) { w->skip()[nr + 6 * p + k] = !cpl; if (cpl) { if (n < 32) w->colmap()[n] = nr + 6 * p + k; ++n; } }
      }
      w->iscr()[32 - 1] = n;
    }
  LANES_END
  const int nA = w->iscr()[31];
  bool regs = nA <= 32;
  for (int p = 0; p < np; ++p) if (w->plist()[9 * p + 8] > 8) regs = false; // needs the grouped static-contact path
  int iter = 0;
  float cost = 0.f, impr = 0.f;
  FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_SETUP) // this solver's phases in the FE_STAT_NEWTON_* columns: include/furniture_b200.h
  for (;;) {
    const float ccost = fe_update(w);
    fe_mul_JT(w, w->fc());
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_START)
    LANES_BEGIN
      float s = 0.f, gsq = 0.f;
      for (int i = lane; i < nv; i += 32) {
        const float r = w->Ma()[i] - w->fs()[i];
        s += 0.5f * r * (w->x()[i] - w->as()[i]);
        const float gi = r - w->fc()[i];
        w->grad()[i] = gi;
        gsq += gi * gi;
      }
      w->scr()[lane] = s; w->scr()[32 + lane] = gsq;
    LANES_END
    const float gauss = fe_sum32(w->scr()), gnorm = sqrtf(fe_sum32(w->scr() + 32));
    cost = gauss + ccost;
    if (!(cost == cost)) { LANES_BEGIN if (lane == 0) w->u()[FE_U_FLAGS] |= FE_FLAG_NUMERIC; LANES_END break; }
    // MuJoCo stops on scale*(oldcost - cost) < tol; in fp32 that difference of two large costs is round-off, so the
    // improvement is taken from the line search instead: -alpha p'(0) / 2 (exact for a quadratic, the Newton decrement)
    if (fe_newton_stop(iter, w->opt.newton_iters, scale, impr, gnorm, w->opt.tolerance)) break;
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_GRAD)
    fe_build_H(w, regs);
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_HESSIAN)
    if (regs) {
      LANES_BEGIN for (int i = lane; i < nv; i += 32) w->search()[i] = -w->grad()[i]; LANES_END
      fe_chol_blocks(w, w->H(), w->skip());
      fe_solve_blocks(w, w->H(), w->skip(), w->search());
      FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_CHOL)
      if (nA <= 16) fe_newton_regs<16>(w, nA); else if (nA <= 24) fe_newton_regs<24>(w, nA); else fe_newton_regs<32>(w, nA);
    } else {
      // independent part blocks are factored / solved by one lane each
      const int* skip = w->skip();
      fe_mark_indep_blocks(w, w->first(), w->skip());
      fe_chol_blocks(w, w->H(), skip);
      LANES_BEGIN for (int i = lane; i < nv; i += 32) w->search()[i] = -w->grad()[i]; LANES_END
      fe_solve_blocks(w, w->H(), skip, w->search());
      if (!fe_chol(w, w->H(), w->first(), nv, skip)) { LANES_BEGIN if (lane == 0) w->u()[FE_U_FLAGS] |= FE_FLAG_NEWTON_PIVOT; LANES_END }
      FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_CHOL)
      fe_chol_solve(w, w->H(), w->first(), nv, w->search(), w->Mv(), skip);
    }
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_PRODUCTS)
    fe_mul_M(w, w->search(), w->Mv());
    fe_mul_J(w, w->search(), w->c_jv(), w->w_jv(), w->l_jv(), false);
    LANES_BEGIN
      float a = 0.f, b = 0.f;
      for (int i = lane; i < nv; i += 32) { a += w->search()[i] * (w->Ma()[i] - w->fs()[i]); b += 0.5f * w->search()[i] * w->Mv()[i]; }
      w->scr()[lane] = a; w->scr()[32 + lane] = b;
    LANES_END
    const float g1 = fe_sum32(w->scr()), g2 = fe_sum32(w->scr() + 32);
    FeLineSearch ls;
    float p1, p2;
    fe_line_eval(w, 0.f, g1, g2, &p1, &p2);
    if (!ls.start(p1, p2)) break;
    for (int k = 0; k < w->opt.ls_iters; ++k) {
      fe_line_eval(w, ls.alpha, g1, g2, &p1, &p2);
      if (!ls.step(p1, p2)) break;
    }
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_LS)
    const float alpha = ls.alpha;
    if (!(alpha > 0.f)) break;
    impr = ls.impr();
    LANES_BEGIN
      for (int i = lane; i < nv; i += 32) { w->x()[i] += alpha * w->search()[i]; w->Ma()[i] += alpha * w->Mv()[i]; }
      for (int c = lane; c < ncon; c += 32)
        for (int k = 0; k < 3; ++k) w->c_jar()[3 * c + k] += alpha * w->c_jv()[3 * c + k];
      for (int e = lane; e < 6 * ne; e += 32) w->w_jar()[e] += alpha * w->w_jv()[e];
      for (int d = lane; d < nr; d += 32) w->l_jar()[d] += alpha * w->l_jv()[d];
    LANES_END
    ++iter;
    // the top of the next iteration would stop on this same test after recomputing forces, J^T f and the gradient: stop now
    // (the forces of the final iterate are computed once, below)
    if (scale * impr < w->opt.tolerance) break;
  }
  fe_update(w);
  fe_mul_JT(w, w->fc());
  LANES_BEGIN if (lane == 0) { if (iter > w->u()[FE_U_NITER]) w->u()[FE_U_NITER] = iter; w->u()[FE_U_STAT + FE_STAT_NEWTON_ITERS] += iter; } LANES_END
  FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_SETUP)
}

// ---- free parts whose contacts are all against the static world (the parts in skipmask are left out), on each part's own
// 6 unknowns [alpha; vdot] with the cost, cones and exact line search of the cooperative solver.  8 lanes per part (4 parts
// per pass), one lane per contact.  Per Newton iteration each lane evaluates its contact (cone zone, force, 3x3 weight,
// J^T f and J^T W J), the group sums them with 3 xor-shuffles per value, every lane of the group then factors the same 6x6
// Hessian and runs the same exact line search, whose per-contact terms are again group-summed.  Parts are independent
// blocks here, so block-wise Newton reaches the same minimiser as the global iteration.
FE_FN void fe_solve_parts_grouped(FeWarp* w, unsigned skipmask) {
  const fe_model* m = w->m;
  const int nr = m->nr, nrl = m->nrlink, np = m->npart, maxit = w->opt.newton_iters, maxls = w->opt.ls_iters;
  const float tol = w->opt.tolerance;
  // Lanes are handed out in units of 4: a part with up to 4 contacts against the static world takes one unit, one with 5-8
  // takes an aligned pair of units; parts are placed in order until the 8 units are used up, the rest wait for the next pass
  // (five parts with <= 4 contacts each, the resting state of this furniture, fit in one pass).
  for (int p0 = 0; p0 < np;) {
    int p_end = p0;
    // lane-private state that lives across regions is kept small (the Jacobian rows, the reduction buffer, the iterate):
    // inertia, smooth force / acceleration and the contact's reference acceleration are re-read from the slice where used
    FE_PRIV(int, c_); FE_PRIV(int, part_); FE_PRIV(int, act_); FE_PRIV(int, iter_); FE_PRIV(int, lsact_); FE_PRIV(int, wide_); FE_PRIV(int, lead_);
    FE_PRIVA(float, J_, 18); FE_PRIVA(float, par_, 4); // par_: D0, D1, mu, friction scale
    FE_PRIVA(float, x_, 6);
    FE_PRIVA(float, acc_, 28); FE_PRIVA(float, sd_, 6); FE_PRIVA(float, jx_, 3); FE_PRIVA(float, jv_, 3);
    FE_PRIV(float, scale_); FE_PRIV(float, impr_); FE_PRIV(float, g1_); FE_PRIV(float, g2_); FE_PRIV(FeLineSearch, ls_);
    LANES_BEGIN
      int part = np, slot = 0;
      PV(wide_) = 0; PV(lead_) = 0;
      {
        const int unit = lane >> 2;
        int nu = 0, p = p0;
        for (; p < np; ++p) {
          if ((skipmask >> p) & 1u) continue; // part of the coupled component: solved there
          const int need = w->plist()[9 * p + 8] > 4 ? 2 : 1;
          if (need == 2 && (nu & 1)) ++nu;
          if (nu + need > 8) break;
          if (unit >= nu && unit < nu + need) { part = p; slot = (lane & 3) + 4 * (unit - nu); PV(wide_) = need == 2; PV(lead_) = (unit == nu) && (lane & 3) == 0; }
          nu += need;
        }
        p_end = p;
      }
      PV(part_) = part < np ? part : -1;
      PV(c_) = -1; PV(act_) = 0; PV(iter_) = 0; PV(impr_) = 0.f; PV(lsact_) = 0;
      PV(acc_)[0] = 0.f; PV(acc_)[1] = 0.f;
      if (part < np) {
        const int l = nrl + part, z = nr + 6 * part, da = m->link_dadr[l];
        const int cnt = w->plist()[9 * part + 8];
        if (cnt > 0) PV(act_) = 1;
        if (slot < cnt) PV(c_) = w->plist()[9 * part + slot];
        const float* I = w->linert() + 10 * l;
        PV(scale_) = 1.0f / (3.f * I[0] + I[4] + I[5] + I[6]);
        const int c = PV(c_);
        if (c >= 0) {
          float xw[6];
          m3mulv(xw, w->lmat() + 9 * l, w->warm() + da + 3);
          v3cpy(xw + 3, w->warm() + da);
          const int B_ = (w->c_link()[c] >> 8) - 1;
          fe_part_rows(w, c, l, B_ == l ? 1.f : -1.f, PV(J_));
          PV(par_)[0] = w->c_D()[2 * c]; PV(par_)[1] = w->c_D()[2 * c + 1]; PV(par_)[2] = w->c_mu()[c]; PV(par_)[3] = w->c_fric()[c];
          float f[3], cw = 0.f, cs = 0.f;
          const float* J = PV(J_);
          const float* q = PV(par_);
          const float* ar = w->c_aref() + 3 * c;
          const float* as = w->as() + z;
          fe_cone_t<false>(dot6(J, xw) - ar[0], dot6(J + 6, xw) - ar[1], dot6(J + 12, xw) - ar[2], q[2], q[3], q[0], q[1], f, &cw, nullptr);
          fe_cone_t<false>(dot6(J, as) - ar[0], dot6(J + 6, as) - ar[1], dot6(J + 12, as) - ar[2], q[2], q[3], q[0], q[1], f, &cs, nullptr);
          PV(acc_)[0] = cw; PV(acc_)[1] = cs;
        }
      }
    LANES_END
    FE_GSUMV_ARRN(acc_, 28, 2, PV_ALL(wide_));
    LANES_BEGIN
      if (PV(part_) >= 0) { // warm start vs unconstrained acceleration: keep the cheaper one
        const int l = nrl + PV(part_), z = nr + 6 * PV(part_), da = m->link_dadr[l];
        float xw[6], Mx[6], cw = PV(acc_)[0];
        m3mulv(xw, w->lmat() + 9 * l, w->warm() + da + 3);
        v3cpy(xw + 3, w->warm() + da);
        inert_mulv(Mx, w->linert() + 10 * l, xw);
        for (int k = 0; k < 6; ++k) cw += 0.5f * (Mx[k] - w->fs()[z + k]) * (xw[k] - w->as()[z + k]);
        const bool use_warm = !(PV(acc_)[1] < cw) && (cw == cw);
        for (int k = 0; k < 6; ++k) PV(x_)[k] = use_warm ? xw[k] : w->as()[z + k];
      }
    LANES_END
    for (int it = 0; it <= maxit; ++it) {
      if (!FE_ANY(act_)) break;
      // per-contact terms at the current x
      LANES_BEGIN
        for (int k = 0; k < 28; ++k) PV(acc_)[k] = 0.f;
        const int c = PV(c_);
        if (PV(act_) && c >= 0) {
          const float* J = PV(J_);
          const float* q = PV(par_);
          const float* ar = w->c_aref() + 3 * c;
          float f[3], W[6], cc = 0.f;
          PV(jx_)[0] = dot6(J, PV(x_)) - ar[0]; PV(jx_)[1] = dot6(J + 6, PV(x_)) - ar[1]; PV(jx_)[2] = dot6(J + 12, PV(x_)) - ar[2];
          const int st = fe_cone_t<true>(PV(jx_)[0], PV(jx_)[1], PV(jx_)[2], q[2], q[3], q[0], q[1], f, &cc, W);
          if (st != 0) {
#pragma unroll
            for (int i = 0; i < 6; ++i) { // column i of W J, then row i of the lower triangle of J^T W J (W symmetric)
              PV(acc_)[i] = -(J[i] * f[0] + J[6 + i] * f[1] + J[12 + i] * f[2]);
              const float w0 = W[0] * J[i] + W[3] * J[6 + i] + W[4] * J[12 + i];
              const float w1 = W[3] * J[i] + W[1] * J[6 + i] + W[5] * J[12 + i];
              const float w2 = W[4] * J[i] + W[5] * J[6 + i] + W[2] * J[12 + i];
#pragma unroll
              for (int j = 0; j <= i; ++j) PV(acc_)[6 + i * (i + 1) / 2 + j] = w0 * J[j] + w1 * J[6 + j] + w2 * J[12 + j];
            }
          }
          PV(acc_)[27] = cc;
        }
      LANES_END
      FE_GSUMV_ARRN(acc_, 28, 28, PV_ALL(wide_));
      // gradient, Hessian, convergence test, Newton direction (identical in the 8 lanes of a group)
      LANES_BEGIN
        if (PV(act_)) {
          const int l = nrl + PV(part_), z = nr + 6 * PV(part_);
          const float* I = w->linert() + 10 * l;
          float g[6], Mx[6], gsq = 0.f;
          float* H = PV(acc_) + 6; // the group-summed J^T W J becomes the Hessian in place
          inert_mulv(Mx, I, PV(x_));
          fe_inert_sym6_add(H, I);
          for (int k = 0; k < 6; ++k) { Mx[k] -= w->fs()[z + k]; g[k] = Mx[k] + PV(acc_)[k]; gsq += g[k] * g[k]; }
          const float gnorm = sqrtf(gsq);
          bool stop = true;
          if (!(gnorm == gnorm)) { if (PV(lead_)) w->u()[FE_U_FLAGS] |= FE_FLAG_NUMERIC; }
          else stop = fe_newton_stop(PV(iter_), maxit, PV(scale_), PV(impr_), gnorm, tol);
          if (stop) PV(act_) = 0;
          else {
            if (!fe_chol6(H) && PV(lead_)) w->u()[FE_U_FLAGS] |= FE_FLAG_NEWTON_PIVOT;
            for (int k = 0; k < 6; ++k) PV(sd_)[k] = -g[k];
            fe_chol6_solve(H, PV(sd_));
            float Ms[6], g1 = 0.f, g2 = 0.f;
            inert_mulv(Ms, I, PV(sd_));
            for (int k = 0; k < 6; ++k) { g1 += PV(sd_)[k] * Mx[k]; g2 += 0.5f * PV(sd_)[k] * Ms[k]; }
            PV(g1_) = g1; PV(g2_) = g2; PV(ls_) = FeLineSearch(); PV(lsact_) = 1;
            if (PV(c_) >= 0) {
              const float* J = PV(J_);
              for (int k = 0; k < 3; ++k) PV(jv_)[k] = dot6(J + 6 * k, PV(sd_));
            }
          }
        }
        if (!PV(act_)) PV(lsact_) = 0;
      LANES_END
      // exact line search; evaluation 0 is at alpha = 0
      for (int ls = 0; ls <= maxls; ++ls) {
        if (!FE_ANY(lsact_)) break;
        LANES_BEGIN
          float p1 = 0.f, p2 = 0.f;
          if (PV(lsact_) && PV(c_) >= 0) {
            const float* q = PV(par_);
            FE_CONE_LS(PV(jx_), PV(jv_), PV(ls_).alpha, q[2], q[3], q[0], q[1], p1, =, p2)
          }
          PV(acc_)[0] = p1; PV(acc_)[1] = p2;
        LANES_END
        FE_GSUMV_ARRN(acc_, 28, 2, PV_ALL(wide_));
        LANES_BEGIN
          if (PV(lsact_)) {
            const float al = PV(ls_).alpha;
            const float p1 = PV(acc_)[0] + PV(g1_) + 2.f * al * PV(g2_), p2 = PV(acc_)[1] + 2.f * PV(g2_);
            if (!(ls == 0 ? PV(ls_).start(p1, p2) : PV(ls_).step(p1, p2))) PV(lsact_) = 0;
          }
        LANES_END
      }
      LANES_BEGIN
        if (PV(act_)) {
          const float al = PV(ls_).alpha;
          if (!(al > 0.f)) PV(act_) = 0;
          else {
            PV(impr_) = PV(ls_).impr();
            for (int k = 0; k < 6; ++k) PV(x_)[k] += al * PV(sd_)[k];
            PV(iter_) += 1;
            // the next pass would stop on this same test before doing anything with its gradient: stop now and spare the
            // pass (per-contact terms, the 28-value group reduction); the final forces are computed after the loop either way
            if (PV(scale_) * PV(impr_) < tol) PV(act_) = 0;
          }
        }
        PV(lsact_) = 0;
      LANES_END
    }
    // final forces of this pass' contacts, constraint wrench of each part
    LANES_BEGIN
      for (int k = 0; k < 6; ++k) PV(acc_)[k] = 0.f;
      const int c = PV(c_);
      if (c >= 0) {
        const float* J = PV(J_);
        const float* q = PV(par_);
        const float* ar = w->c_aref() + 3 * c;
        float f[3], dummy = 0.f;
        const int st = fe_cone_t<false>(dot6(J, PV(x_)) - ar[0], dot6(J + 6, PV(x_)) - ar[1], dot6(J + 12, PV(x_)) - ar[2], q[2], q[3], q[0], q[1], f, &dummy, nullptr);
        w->c_state()[c] = st;
        for (int k = 0; k < 3; ++k) w->c_f()[3 * c + k] = f[k];
        for (int i = 0; i < 6; ++i) PV(acc_)[i] = J[i] * f[0] + J[6 + i] * f[1] + J[12 + i] * f[2];
      }
    LANES_END
    FE_GSUMV_ARRN(acc_, 28, 6, PV_ALL(wide_));
    LANES_BEGIN
      const int part = PV(part_);
      if (part >= 0 && PV(lead_)) {
        const int z = nr + 6 * part;
        const bool any = w->plist()[9 * part + 8] > 0;
        for (int k = 0; k < 6; ++k) { w->x()[z + k] = any ? PV(x_)[k] : w->as()[z + k]; w->fc()[z + k] = any ? PV(acc_)[k] : 0.f; }
        w->iscr()[part] = PV(iter_);
      }
    LANES_END
    p0 = p_end;
  }
}

// ---- robot block whose only constraint rows are joint limits (no robot contact): the common case, e.g. the
// gripper fingers resting on their stops.  Lane d owns dof d in registers; M products are 9 shuffles + 9 FMAs per lane,
// reductions are xor-butterflies, only the small Cholesky goes through the slice.  Same cost function as fe_solve_coop, with
// the stop test fe_newton_stop and the exact line search FeLineSearch that every Newton solver here uses.
FE_FN void fe_solve_robot_limits(FeWarp* w) {
  const fe_model* m = w->m;
  const int nr = m->nr, maxit = w->opt.newton_iters, maxls = w->opt.ls_iters;
  const float tol = w->opt.tolerance, scale = 1.0f / (m->meaninertia * (float)(m->nv > 1 ? m->nv : 1));
  FE_PRIV(float, x_); FE_PRIV(float, as_); FE_PRIV(float, sg_); FE_PRIV(float, ar_); FE_PRIV(float, D_);
  FE_PRIV(float, t_); FE_PRIV(float, u_); FE_PRIV(float, r_); FE_PRIV(float, s_); FE_PRIV(float, Ms_); FE_PRIV(float, f_);
  FE_PRIV(float, a_); FE_PRIV(float, b_); FE_PRIV(int, any_);
  REGS_BEGIN
    const bool on = lane < nr;
    PV(x_) = on ? w->warm()[lane] : 0.f; PV(as_) = on ? w->as()[lane] : 0.f;
    PV(sg_) = on ? w->l_sign()[lane] : 0.f; PV(ar_) = on ? w->l_aref()[lane] : 0.f; PV(D_) = on ? w->l_D()[lane] : 0.f;
    PV(any_) = PV(sg_) != 0.f;
    PV(u_) = PV(x_) - PV(as_); PV(r_) = 0.f; PV(f_) = 0.f;
  REGS_END
  if (!FE_ANY(any_)) {
    LANES_BEGIN if (lane < nr) { w->x()[lane] = PV(as_); w->fc()[lane] = 0.f; w->l_f()[lane] = 0.f; } LANES_END
    return;
  }
  LANES_BEGIN if (lane == 0) w->u()[FE_U_STAT + FE_STAT_NEWTON_SOLVES] += 1; LANES_END
  // r = M (warm - as); warm start kept only if it is cheaper than the unconstrained acceleration
  for (int j = 0; j < nr; ++j) {
    FE_SHFL(t_, u_, j);
    REGS_BEGIN if (lane < nr) PV(r_) += w->Mr()[lane * nr + j] * PV(t_); REGS_END
  }
  REGS_BEGIN
    const float jw = PV(sg_) * PV(x_) - PV(ar_), js = PV(sg_) * PV(as_) - PV(ar_);
    PV(a_) = 0.5f * PV(u_) * PV(r_) + ((PV(sg_) != 0.f && jw < 0.f) ? 0.5f * PV(D_) * jw * jw : 0.f);
    PV(b_) = (PV(sg_) != 0.f && js < 0.f) ? 0.5f * PV(D_) * js * js : 0.f;
  REGS_END
  FE_WSUM(a_); FE_WSUM(b_);
  if (!(FE_UNI(a_) <= FE_UNI(b_))) { REGS_BEGIN PV(x_) = PV(as_); PV(r_) = 0.f; REGS_END }
  int iter = 0;
  float impr = 0.f;
  for (;;) {
    REGS_BEGIN
      const float jar = PV(sg_) * PV(x_) - PV(ar_);
      const bool act = PV(sg_) != 0.f && jar < 0.f;
      PV(f_) = act ? -PV(D_) * jar : 0.f;
      const float gi = PV(r_) - PV(sg_) * PV(f_);
      PV(t_) = gi;       // gradient
      PV(a_) = gi * gi;
      PV(u_) = act ? PV(D_) : 0.f;
    REGS_END
    FE_WSUM(a_);
    const float gnorm = sqrtf(FE_UNI(a_));
    if (!(gnorm == gnorm)) { LANES_BEGIN if (lane == 0) w->u()[FE_U_FLAGS] |= FE_FLAG_NUMERIC; LANES_END break; }
    if (fe_newton_stop(iter, maxit, scale, impr, gnorm, tol)) break;
    LANES_BEGIN
      if (lane < nr) { w->Mv()[lane] = PV(u_); w->search()[lane] = -PV(t_); } // H = Mr + diag(D of the active limit rows)
    LANES_END
    fe_robot_solve(w, 0.f, w->Mv(), w->search(), w->search(), FE_FLAG_NEWTON_PIVOT);
    REGS_BEGIN PV(s_) = lane < nr ? w->search()[lane] : 0.f; PV(Ms_) = 0.f; REGS_END
    for (int j = 0; j < nr; ++j) {
      FE_SHFL(t_, s_, j);
      REGS_BEGIN if (lane < nr) PV(Ms_) += w->Mr()[lane * nr + j] * PV(t_); REGS_END
    }
    REGS_BEGIN PV(a_) = PV(s_) * PV(r_); PV(b_) = 0.5f * PV(s_) * PV(Ms_); REGS_END
    FE_WSUM(a_); FE_WSUM(b_);
    const float g1 = FE_UNI(a_), g2 = FE_UNI(b_);
    FeLineSearch ls; // evaluation -1 is at alpha = 0
    for (int k = -1; k < maxls; ++k) {
      const float alpha = ls.alpha;
      REGS_BEGIN
        const float jv = PV(sg_) * PV(s_), xx = PV(sg_) * PV(x_) - PV(ar_) + alpha * jv;
        const bool act = PV(sg_) != 0.f && xx < 0.f;
        PV(a_) = act ? PV(D_) * xx * jv : 0.f;
        PV(b_) = act ? PV(D_) * jv * jv : 0.f;
      REGS_END
      FE_WSUM(a_); FE_WSUM(b_);
      const float p1 = g1 + 2.f * g2 * alpha + FE_UNI(a_), p2 = 2.f * g2 + FE_UNI(b_);
      if (!(k < 0 ? ls.start(p1, p2) : ls.step(p1, p2))) break;
    }
    const float alpha = ls.alpha;
    if (!(alpha > 0.f)) break;
    impr = ls.impr();
    REGS_BEGIN PV(x_) += alpha * PV(s_); PV(r_) += alpha * PV(Ms_); REGS_END
    ++iter;
  }
  LANES_BEGIN
    if (lane < nr) {
      const float jar = PV(sg_) * PV(x_) - PV(ar_);
      const float f = (PV(sg_) != 0.f && jar < 0.f) ? -PV(D_) * jar : 0.f;
      w->x()[lane] = PV(x_); w->fc()[lane] = PV(sg_) * f; w->l_f()[lane] = f; w->l_jar()[lane] = jar;
    }
    if (lane == 0) { if (iter > w->u()[FE_U_NITER]) w->u()[FE_U_NITER] = iter; w->u()[FE_U_STAT + FE_STAT_NEWTON_ITERS] += iter; }
  LANES_END
}

#include "fe_solve_comp.h"

// fe_solve_parts_grouped over the parts not in skipmask; their largest iteration count goes to FE_U_NITER and is added to
// the FE_STAT_PART_ITERS column
FE_HD void fe_solve_free_parts(FeWarp* w, unsigned skipmask) {
  fe_solve_parts_grouped(w, skipmask);
  LANES_BEGIN
    if (lane == 0) {
      int mx = 0;
      for (int p = 0; p < w->m->npart; ++p) if (!((skipmask >> p) & 1u)) mx = w->iscr()[p] > mx ? w->iscr()[p] : mx;
      w->u()[FE_U_NITER] = mx; w->u()[FE_U_STAT + FE_STAT_PART_ITERS] += mx;
    }
  LANES_END
}

// mj_fwdConstraint.  The constraint set of this mj_step is split into independent pieces (the cost is separable over them):
// free parts that only touch the static world (8 lanes per part, fe_solve_parts_grouped), the robot block when its only
// rows are joint limits (fe_solve_robot_limits), and the coupled component -- robot block with contacts, parts in contact
// with the robot or each other, welded parts -- solved by fe_solve_comp with its rows in registers.  A component beyond 32
// dofs or 32 contacts falls back to the cooperative solver over all dofs (fe_solve_coop; its Hessian in global memory).
FE_FN void fe_solve(FeWarp* w) {
  const fe_model* m = w->m;
  const int ncon = w->u()[FE_U_NCON], ne = m->neq, np = m->npart, nrl = m->nrlink, nr = m->nr;
  FE_TICK_START
  LANES_BEGIN
    int rcon = 0, cpl = 0;
    for (int c = lane; c < ncon; c += 32) { const int k = w->c_kind()[c]; rcon |= (k == 1 || k == 2); }
    if (lane < np) { // contacts of part `lane`: against the static world (at most 8 handled by the grouped solver) or coupling
      const int l = nrl + lane;
      int cnt = 0;
      for (int c = 0; c < ncon; ++c) {
        const int A = (w->c_link()[c] & 255) - 1, B = (w->c_link()[c] >> 8) - 1;
        if (A != l && B != l) continue;
        if (w->c_kind()[c] != 0) { cpl = 1; continue; }
        if (cnt < 8) w->plist()[9 * lane + cnt] = c;
        ++cnt;
      }
      w->plist()[9 * lane + 8] = cnt;
      if (cnt > 8) cpl = 1;
      for (int e = 0; e < ne; ++e) if (w->eq_active()[e] && (m->eq_link1[e] == l || m->eq_link2[e] == l)) cpl = 1;
    }
    w->iscr()[lane] = cpl; w->colmap()[lane] = rcon;
    if (lane == 0) w->u()[FE_U_NITER] = 0;
  LANES_END
  const unsigned cplmask = fe_ballot32(w->iscr());
  const bool robot_in = fe_ballot32(w->colmap()) != 0u;
  if (cplmask == 0u && !robot_in) { // nothing couples two moving blocks and the robot touches nothing
    fe_solve_free_parts(w, 0u);
    fe_solve_robot_limits(w);
    return;
  }
  // active dofs of the component (robot dofs first, then the coupled parts in order) and its contacts
  int* const ccl = (int*)w->Jc();
  LANES_BEGIN
    if (lane == 0) {
      int n = 0;
      if (robot_in) for (int d = 0; d < nr; ++d) { if (n < 32) w->colmap()[n] = d; ++n; }
      for (int p = 0; p < np; ++p)
        if ((cplmask >> p) & 1u) for (int k = 0; k < 6; ++k) { if (n < 32) w->colmap()[n] = nr + 6 * p + k; ++n; }
      w->iscr()[31] = n;
      if (cplmask) w->u()[FE_U_STAT + FE_STAT_COUPLED] += 1; else w->u()[FE_U_STAT + FE_STAT_ROBOT_ONLY] += 1;
    }
  LANES_END
  const int nA = w->iscr()[31];
  int ncc = 0;
  for (int base = 0; base < ncon; base += 32) {
    int run = 0;
    (void)run;
    LANES_BEGIN
      const int c = base + lane;
      int in = 0;
      if (c < ncon) {
        if (w->c_kind()[c] != 0) in = 1;
        else { const int A = (w->c_link()[c] & 255) - 1, B = (w->c_link()[c] >> 8) - 1; in = (int)((cplmask >> ((A > B ? A : B) - nrl)) & 1u); }
      }
      const int off = FE_SCAN(run, in);
      if (in && ncc + off < 32) ccl[ncc + off] = c;
      if (lane == 31) w->iscr()[30] = off + in;
    LANES_END
    ncc += w->iscr()[30];
    LANES_BEGIN LANES_END
  }
  if (nA <= 32 && ncc <= 32) {
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_SOLVE_PRE)
    fe_solve_free_parts(w, cplmask);
    if (!robot_in) fe_solve_robot_limits(w);
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_SOLVE_GROUPED)
    if (nA <= 16) fe_solve_comp<16>(w, nA, ncc, cplmask, robot_in ? 1 : 0);
    else if (nA <= 24) fe_solve_comp<24>(w, nA, ncc, cplmask, robot_in ? 1 : 0);
    else fe_solve_comp<32>(w, nA, ncc, cplmask, robot_in ? 1 : 0);
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_SOLVE_COMP)
    return;
  }
  fe_solve_coop(w, cplmask); // fallback: the cooperative solver over all dofs (FE_COOP_* arrays in global memory)
}

// ---------------------------------------------------------------- mj_Euler + mj_advance
FE_FN void fe_integrate(FeWarp* w) {
  const fe_model* m = w->m;
  const int nr = m->nr, nrl = m->nrlink, np = m->npart;
  const float h = m->timestep;
  // robot: (Mr + h B) a = fs + fc
  if (nr > 0) {
    LANES_BEGIN
      for (int d = lane; d < nr; d += 32) w->grad()[d] = w->fs()[d] + w->fc()[d];
    LANES_END
    fe_robot_solve(w, h, nullptr, w->grad(), w->grad(), FE_FLAG_NUMERIC);
  }
  LANES_BEGIN
    // warm start for the next step = solver solution, stored in qacc coordinates
    for (int d = lane; d < nr; d += 32) {
      w->warm()[d] = w->x()[d];
      const float v = w->qvel()[d] + h * w->grad()[d];
      w->qvel()[d] = v;
      w->qpos()[d] += h * v;
    }
    for (int p = lane; p < np; p += 32) {
      const int l = nrl + p, z = nr + 6 * p, da = m->link_dadr[l], qa = m->link_qadr[l];
      const float* R = w->lmat() + 9 * l;
      float t[3];
      m3tmulv(t, R, w->x() + z);
      v3cpy(w->warm() + da, w->x() + z + 3);
      v3cpy(w->warm() + da + 3, t);
      float A[21], a[6];
      fe_inert_sym6(A, w->linert() + 10 * l, h * m->dof_damping[da]);
      if (!fe_chol6(A)) w->u()[FE_U_FLAGS] |= FE_FLAG_NUMERIC;
      for (int k = 0; k < 6; ++k) a[k] = w->fs()[z + k] + w->fc()[z + k];
      fe_chol6_solve(A, a);
      m3tmulv(t, R, a);
      for (int k = 0; k < 3; ++k) { w->qvel()[da + k] += h * a[3 + k]; w->qvel()[da + 3 + k] += h * t[k]; }
      for (int k = 0; k < 3; ++k) w->qpos()[qa + k] += h * w->qvel()[da + k];
      float wl[3] = {w->qvel()[da + 3], w->qvel()[da + 4], w->qvel()[da + 5]};
      const float n = v3norm(wl);
      float* q = w->qpos() + qa + 3;
      if (n * h > 1e-12f) {
        const float s = sinf(0.5f * n * h) / n, c = cosf(0.5f * n * h);
        float dq[4] = {c, wl[0] * s, wl[1] * s, wl[2] * s}, qn[4];
        qmul(qn, q, dq);
        q[0] = qn[0]; q[1] = qn[1]; q[2] = qn[2]; q[3] = qn[3];
      }
      qnormalize(q);
    }
  LANES_END
  // divergence guard (mj_checkPos / mj_checkVel): NaN or huge values raise FE_FLAG_DIVERGED
  LANES_BEGIN
    int bad = 0;
    for (int i = lane; i < m->nq; i += 32) { float v = w->qpos()[i]; if (!(v == v) || fabsf(v) > 1e6f) bad = 1; }
    for (int i = lane; i < m->nv; i += 32) { float v = w->qvel()[i]; if (!(v == v) || fabsf(v) > 1e6f) bad = 1; }
    w->iscr()[lane] = bad;
  LANES_END
  if (fe_ballot32(w->iscr()) != 0u) { LANES_BEGIN if (lane == 0) w->u()[FE_U_FLAGS] |= FE_FLAG_DIVERGED; LANES_END }
}

FE_FN void fe_forward(FeWarp* w) {
  fe_kin_smooth(w);
  fe_collide(w);
  fe_assemble(w);
  fe_solve(w);
}
FE_FN void fe_substep(FeWarp* w) {
  fe_forward(w);
  fe_integrate(w);
}
// same step with block barriers between the phases: the warps (= envs) of a block then fetch the same instructions at the
// same time, which is what keeps the instruction cache effective for this large, mostly straight-line code.  Every live warp
// of the block must reach the same sequence of barriers: the step loops of the env steps, whose length is the env's own
// substep count, keep it with fe_substeps_mixed (below); fe_run_env runs one count for the whole launch.
FE_FN void fe_substep_lockstep(FeWarp* w) {
  FE_TICK_START
  FE_BLOCK_SYNC; FE_TICK(w->u() + FE_U_STAT, FE_STAT_WAIT, FE_STAT_WAIT_KIN) fe_kin_smooth(w); FE_TICK(w->u() + FE_U_STAT, FE_STAT_KIN)
  FE_BLOCK_SYNC; FE_TICK(w->u() + FE_U_STAT, FE_STAT_WAIT, FE_STAT_WAIT_COLLIDE) fe_collide(w); FE_TICK(w->u() + FE_U_STAT, FE_STAT_COLLIDE)
  FE_BLOCK_SYNC; FE_TICK(w->u() + FE_U_STAT, FE_STAT_WAIT, FE_STAT_WAIT_ASSEMBLE) fe_assemble(w); FE_TICK(w->u() + FE_U_STAT, FE_STAT_ASSEMBLE)
  FE_BLOCK_SYNC; FE_TICK(w->u() + FE_U_STAT, FE_STAT_WAIT, FE_STAT_WAIT_SOLVE) fe_solve(w);
#if FE_DEVICE_BUILD
  { const int d_ = (int)((clock64() - t0_) >> 4); if ((threadIdx.x & 31u) == 0 && d_ > w->u()[FE_U_STAT + FE_STAT_SOLVE_MAX]) w->u()[FE_U_STAT + FE_STAT_SOLVE_MAX] = d_; }
#endif
  FE_TICK(w->u() + FE_U_STAT, FE_STAT_SOLVE)
  FE_BLOCK_SYNC; FE_TICK(w->u() + FE_U_STAT, FE_STAT_WAIT, FE_STAT_WAIT_INTEGRATE) fe_integrate(w); FE_TICK(w->u() + FE_U_STAT, FE_STAT_INTEGRATE)
}
// A step loop whose trip count differs between the warps of a block (each env's substeps) is fe_substeps_mixed, below.
// Every live warp runs the block's largest count of iterations: one whose own steps are done passes the five barriers of a step
// without the step.  The loop test is a barrier itself (bar.red.or on sm_90a), reached by every live thread once per iteration, and
// its result is the same on every thread, so the block's threads all leave the loop after the same iteration and every barrier
// phase sees all of them, each phase with one kind of barrier instruction.  Warps of empty slots exit before the first barrier,
// as with a uniform count: an exited warp is no longer waited for.  `n` is equal on the lanes of a warp (one env per warp).
FE_HD bool fe_block_any(bool p) {
#if FE_DEVICE_BUILD
  return __syncthreads_or(p ? 1 : 0) != 0;
#else
  return p; // the emulation runs one warp at a time
#endif
}
FE_HD void fe_substep_idle() { FE_BLOCK_SYNC; FE_BLOCK_SYNC; FE_BLOCK_SYNC; FE_BLOCK_SYNC; FE_BLOCK_SYNC; }
// the env's `n` mj_steps in a block whose warps may run different counts
FE_HD void fe_substeps_mixed(FeWarp* w, int n) {
  for (int i = 0; fe_block_any(i < n); ++i) {
    if (i < n) fe_substep_lockstep(w); else fe_substep_idle();
  }
}
