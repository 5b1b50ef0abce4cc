// fe_solve_comp.h -- Newton solve of the coupled component of one env with the constraint rows in registers.
//
// The component is the set of moving blocks that constraints tie together in this mj_step: the robot block when a robot
// geom touches anything, plus every free part that touches the robot or another part, carries an active weld, or has more
// static-world contacts than the grouped part solver takes.  Parts outside it are independent 6x6 problems
// (fe_solve_parts_grouped); a robot block outside it has joint-limit rows only (fe_solve_robot_limits).  The cost function
// is block-separable over these pieces, so solving them separately reaches the minimiser of MuJoCo's joint Newton
// iteration (mj_fwdConstraint; reference call site furniture/env/furniture.py:2878-2879).
//
// Roles of the 32 lanes (a lane holds several at once):
//   dof role      lane i < nA owns active dof colmap[i]: iterate x, smooth acceleration, r = M (x - a_smooth), its joint-limit
//                 row, and -- while the Newton direction is computed -- row i of the lower triangle of H;
//   contact role  lane k < ncc owns component contact ccl[k]: jar (3), search-direction rows jv (3), impedance weights, cone
//                 parameters: cone zone, force, cost, line-search terms and the contact's share of the Hessian are evaluated
//                 from registers;
//   link role     lane l < nlink stages the spatial acceleration of link l under a dof-space vector (J v) and gathers the
//                 link's constraint wrench (J^T f) from the per-link contact lists built once per solve.
// Exchange between roles goes through small staging arrays of the slice (link twists / wrenches, world-frame contact
// forces); there is no scan over all contacts and no Hessian in shared memory inside the iteration.  H = M + sum over link
// pairs of D^T K D is assembled in registers from the constant part (M and the weld terms, packed once per solve) and one
// 6x6 matrix K per pair of links in contact (as in fe_newton_regs), factored and solved in registers by FE_REG_CHOL_SOLVE.
#pragma once

FE_BOTH int fe_popc(unsigned v) {
#if defined(__CUDA_ARCH__)
  return __popc(v);
#else
  return __builtin_popcount(v);
#endif
}

template <int NMAX>
FE_FN void fe_solve_comp(FeWarp* w, int nA, int ncc, unsigned cplmask, int robot_in) {
  const fe_model* m = w->m;
  const int nr = m->nr, nrl = m->nrlink, nl = m->nlink, np = m->npart, ne = m->neq, nv = m->nv;
  const int maxit = w->opt.newton_iters, maxls = w->opt.ls_iters;
  const float tol = w->opt.tolerance, scale = 1.0f / (m->meaninertia * (float)(nv > 1 ? nv : 1));
  const float Pr[3] = {m->robot_ref[0], m->robot_ref[1], m->robot_ref[2]};
  int* const ccl = (int*)w->Jc(); // [32] component contacts (set by the caller)
  int* const lidx = ccl + 32;     // [64] per-link contact lists: contact | side << 8 (side 1 = the link is the B side)
  int* const lptr = w->first();   // [nlink + 1]
  float* const Hm = w->Hm();      // packed lower triangle over the active dofs (row i = colmap[i]): M + weld terms (constant during the solve)
#define COMP_INLINK(l) ((l) < nrl ? robot_in : (int)((cplmask >> ((l) - nrl)) & 1u))
  // position of active dof z in colmap: robot dofs first, then the coupled parts in order
#define COMP_POS(z) ((z) < nr ? (z) : (robot_in ? nr : 0) + 6 * fe_popc(cplmask & ((1u << (((z) - nr) / 6)) - 1u)) + ((z) - nr) % 6)

  FE_PRIV(int, z_); FE_PRIV(float, x_); FE_PRIV(float, as_); FE_PRIV(float, r_); FE_PRIV(float, fc_); FE_PRIV(float, s_); FE_PRIV(float, Ms_);
  FE_PRIV(float, lsg_); FE_PRIV(float, lar_); FE_PRIV(float, lD_); FE_PRIV(int, sub_);
  FE_PRIV(int, c_); FE_PRIV(int, ab_); FE_PRIV(int, st_); FE_PRIV(int, key_); FE_PRIV(int, lead_); FE_PRIV(int, isl_);
  FE_PRIVA(float, par_, 4); FE_PRIVA(float, jar_, 3); FE_PRIVA(float, jv_, 3); FE_PRIVA(float, f_, 3);
  FE_PRIV(float, ox_); FE_PRIV(float, oy_); FE_PRIV(float, oz_); FE_PRIV(float, px_); FE_PRIV(float, py_); FE_PRIV(float, pz_);
  FE_PRIV(float, a_); FE_PRIV(float, b_); FE_PRIV(float, t_);
  FE_PRIV(int, any_);
  FE_TICK_START

  // ---------------------------------------------------------------- set-up (once per solve)
  int run = 0;
  (void)run;
  LANES_BEGIN
    // rows of the coupled parts start with zeros left of their own block (M is block diagonal; weld terms are added below)
    for (int p = 0; p < np; ++p)
      if ((cplmask >> p) & 1u) {
        const int z = COMP_POS(nr + 6 * p);
        for (int j = lane; j < z; j += 32)
#pragma unroll
          for (int i = 0; i < 6; ++i) Hm[fe_tri(z + i) + j] = 0.f;
      }
    // warm start (stored in qacc coordinates) -> solver coordinates, staged in x()
    if (robot_in) for (int d = lane; d < nr; d += 32) w->x()[d] = w->warm()[d];
    for (int p = lane; p < np; p += 32)
      if ((cplmask >> p) & 1u) {
        const int da = m->link_dadr[nrl + p], z = nr + 6 * p;
        m3mulv(w->x() + z, w->lmat() + 9 * (nrl + p), w->warm() + da + 3);
        v3cpy(w->x() + z + 3, w->warm() + da);
      }
    // per-link contact lists
    const int l = lane;
    int cnt = 0;
    if (l < nl && COMP_INLINK(l))
      for (int k = 0; k < ncc; ++k) {
        const int lk = w->c_link()[ccl[k]];
        cnt += ((lk & 255) - 1 == l) + ((lk >> 8) - 1 == l);
      }
    int off = FE_SCAN(run, cnt);
    if (l < nl) lptr[l] = off;
    if (l == nl - 1) lptr[nl] = off + cnt;
    if (cnt > 0)
      for (int k = 0; k < ncc; ++k) {
        const int c = ccl[k], lk = w->c_link()[c];
        if ((lk & 255) - 1 == l) lidx[off++] = c;
        if ((lk >> 8) - 1 == l) lidx[off++] = c | 256;
      }
  LANES_END
  LANES_BEGIN // constant part of H: M in solver coordinates
    if (robot_in)
      for (int d = lane; d < nr; d += 32)
        for (int j = 0; j <= d; ++j) Hm[fe_tri(d) + j] = w->Mr()[d * nr + j];
    for (int p = lane; p < np; p += 32)
      if ((cplmask >> p) & 1u) {
        const int z = COMP_POS(nr + 6 * p);
        float A[21];
        fe_inert_sym6(A, w->linert() + 10 * (nrl + p), 0.f);
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
          for (int j = 0; j <= i; ++j) Hm[fe_tri(z + i) + z + j] = A[i * (i + 1) / 2 + j];
      }
    int aw = 0;
    for (int e = lane; e < ne; e += 32) aw |= w->eq_active()[e] != 0;
    PV(any_) = aw;
  LANES_END
  const bool anyweld = FE_ANY(any_);
  if (anyweld) { // weld rows have constant weights: their J^T D J is part of the constant matrix
    for (int e = 0; e < ne; ++e) {
      if (!w->eq_active()[e]) continue;
      const int A = m->eq_link1[e], B = m->eq_link2[e];
      for (int half = 0; half < 2; ++half) { // rows 0-2 (translation) then 3-5 (rotation): 3 rows x 12 columns staged in scr
        LANES_BEGIN
          const int j = lane;
          if (j < 12) {
            const bool sideA = j < 6;
            const int jj = sideA ? j : j - 6;
            float col[3] = {0.f, 0.f, 0.f};
            if (half == 0) { // v_A + w_A x r1 - v_B
              if (sideA) {
                if (jj < 3) {
                  float ej[3] = {jj == 0 ? 1.f : 0.f, jj == 1 ? 1.f : 0.f, jj == 2 ? 1.f : 0.f}, t[3];
                  v3cross(t, ej, w->w_r1() + 3 * e);
                  col[0] = t[0]; col[1] = t[1]; col[2] = t[2];
                } else col[jj - 3] = 1.f;
              } else if (jj >= 3) col[jj - 3] = -1.f;
            } else if (jj < 3) {
              const float sg = sideA ? 1.f : -1.f;
              for (int k = 0; k < 3; ++k) col[k] = sg * w->w_G()[9 * e + 3 * k + jj];
            }
            w->scr()[j] = col[0]; w->scr()[16 + j] = col[1]; w->scr()[32 + j] = col[2];
            w->iscr()[j] = COMP_POS(nr + 6 * ((sideA ? A : B) - nrl) + jj);
          }
        LANES_END
        LANES_BEGIN
          for (int en = lane; en < fe_tri(12); en += 32) {
            int i = (int)((sqrtf(8.f * (float)en + 1.f) - 1.f) * 0.5f);
            while (fe_tri(i + 1) <= en) ++i;
            while (fe_tri(i) > en) --i;
            const int j = en - fe_tri(i);
            float v = 0.f;
            for (int a = 0; a < 3; ++a) v += w->w_D()[6 * e + 3 * half + a] * w->scr()[16 * a + i] * w->scr()[16 * a + j];
            if (v != 0.f) {
              int zi = w->iscr()[i], zj = w->iscr()[j];
              if (zi < zj) { int t = zi; zi = zj; zj = t; }
              Hm[fe_tri(zi) + zj] += v;
            }
          }
        LANES_END
      }
    }
  }
  // lane-private state of the two roles
  REGS_BEGIN
    const int i = lane, z = i < nA ? w->colmap()[i] : -1;
    PV(z_) = z;
    PV(as_) = z >= 0 ? w->as()[z] : 0.f;
    PV(x_) = z >= 0 ? w->x()[z] : 0.f; // warm candidate
    PV(r_) = 0.f; PV(fc_) = 0.f; PV(s_) = 0.f; PV(Ms_) = 0.f;
    const bool rd = z >= 0 && z < nr;
    PV(lsg_) = rd ? w->l_sign()[z] : 0.f; PV(lar_) = rd ? w->l_aref()[z] : 0.f; PV(lD_) = rd ? w->l_D()[z] : 0.f;
    int sub = 0; // robot dof: the links it moves
    if (rd) for (int l = z; l < nrl; ++l) sub |= ((m->link_ancmask[l] >> z) & 1) << l;
    PV(sub_) = sub;
    const int k = lane;
    PV(c_) = -1; PV(ab_) = 0; PV(st_) = 0; PV(key_) = -1 - lane;
    PV(px_) = PV(py_) = PV(pz_) = 0.f;
    PV(par_)[0] = PV(par_)[1] = PV(par_)[2] = PV(par_)[3] = 0.f;
#pragma unroll
    for (int q = 0; q < 3; ++q) { PV(jar_)[q] = 0.f; PV(jv_)[q] = 0.f; PV(f_)[q] = 0.f; }
    if (k < ncc) {
      const int c = ccl[k];
      PV(c_) = c; PV(ab_) = w->c_link()[c]; PV(key_) = PV(ab_);
      PV(par_)[0] = w->c_D()[2 * c]; PV(par_)[1] = w->c_D()[2 * c + 1]; PV(par_)[2] = w->c_mu()[c]; PV(par_)[3] = w->c_fric()[c];
      PV(px_) = w->c_pos()[3 * c]; PV(py_) = w->c_pos()[3 * c + 1]; PV(pz_) = w->c_pos()[3 * c + 2];
    }
  REGS_END
  // contacts are grouped by the pair of links they join; the first contact of a pair lends its point as the pair's origin
  FE_MATCH_LEADER(lead_, PV_ALL(key_));
  FE_SHFLV(ox_, PV_ALL(px_), PV_ALL(lead_)); FE_SHFLV(oy_, PV_ALL(py_), PV_ALL(lead_)); FE_SHFLV(oz_, PV_ALL(pz_), PV_ALL(lead_));
  REGS_BEGIN PV(isl_) = (PV(c_) >= 0 && PV(lead_) == lane) ? 1 : 0; REGS_END
  const unsigned pairs = FE_BALLOTP(PV_ALL(isl_));

  // rows = J v for a dof-space vector v held in the slice (solver coordinates): link twists, then one contact per lane;
  // weld rows go to `wdst` (6 per weld); with `sub` the reference acceleration is subtracted
#define COMP_MULJ(vec, out_, wdst, sub)                                                                                          \
  LANES_BEGIN                                                                                                                      \
    const int l = lane;                                                                                                            \
    if (l < nl && COMP_INLINK(l)) {                                                                                                \
      float X[6] = {0, 0, 0, 0, 0, 0};                                                                                             \
      if (l < nrl) {                                                                                                               \
        const int mask = m->link_ancmask[l];                                                                                       \
        for (int d = 0; d < nr; ++d)                                                                                               \
          if ((mask >> d) & 1) { const float xd = (vec)[d]; for (int q = 0; q < 6; ++q) X[q] += w->S()[6 * d + q] * xd; }          \
      } else for (int q = 0; q < 6; ++q) X[q] = (vec)[nr + 6 * (l - nrl) + q];                                                     \
      for (int q = 0; q < 6; ++q) w->lacc2()[6 * l + q] = X[q];                                                                    \
    }                                                                                                                              \
  LANES_END                                                                                                                        \
  LANES_BEGIN                                                                                                                      \
    const int c = PV(c_);                                                                                                          \
    if (c >= 0) {                                                                                                                  \
      const int A = (PV(ab_) & 255) - 1, B = (PV(ab_) >> 8) - 1;                                                                   \
      const float p[3] = {PV(px_), PV(py_), PV(pz_)};                                                                              \
      float aA[3], aB[3], da[3], F[9];                                                                                             \
      fe_point_vel(w, w->lacc2(), A, p, aA);                                                                                       \
      fe_point_vel(w, w->lacc2(), B, p, aB);                                                                                       \
      v3sub(da, aB, aA);                                                                                                           \
      fe_frame_load(w, c, F);                                                                                                      \
      for (int q = 0; q < 3; ++q) PV(out_)[q] = v3dot(F + 3 * q, da) - ((sub) ? w->c_aref()[3 * c + q] : 0.f);                     \
    }                                                                                                                              \
    if (anyweld)                                                                                                                   \
      for (int e = lane; e < ne; e += 32) {                                                                                        \
        if (!w->eq_active()[e]) continue;                                                                                          \
        float rr[6];                                                                                                               \
        fe_weld_rows(w, e, rr);                                                                                                    \
        for (int q = 0; q < 6; ++q) (wdst)[6 * e + q] = rr[q] - ((sub) ? w->w_aref()[6 * e + q] : 0.f);                            \
      }                                                                                                                            \
  LANES_END

  // out_ (per dof lane) = (M v)_i for v in the slice
#define COMP_MULM(vec, out_)                                                                                                     \
  REGS_BEGIN                                                                                                                       \
    const int z = PV(z_);                                                                                                          \
    float o = 0.f;                                                                                                                 \
    if (z >= 0 && z < nr) { for (int j = 0; j < nr; ++j) o += w->Mr()[z * nr + j] * (vec)[j]; }                                    \
    else if (z >= nr) {                                                                                                            \
      const int p = (z - nr) / 6, jj = (z - nr) - 6 * p;                                                                           \
      float F[6];                                                                                                                  \
      inert_mulv(F, w->linert() + 10 * (nrl + p), (vec) + nr + 6 * p);                                                             \
      o = jj == 0 ? F[0] : (jj == 1 ? F[1] : (jj == 2 ? F[2] : (jj == 3 ? F[3] : (jj == 4 ? F[4] : F[5]))));                       \
    }                                                                                                                              \
    PV(out_) = o;                                                                                                                  \
  REGS_END

  // constraint cost of the rows held in (jarr_ | wjar | limits of the dof vector xv_): summed over the warp into `dst`
#define COMP_COST(jarr_, wjar, xv_, dst)                                                                                         \
  REGS_BEGIN                                                                                                                       \
    float cc = 0.f;                                                                                                                \
    if (PV(c_) >= 0) { float ff[3]; fe_cone_t<false>(PV(jarr_)[0], PV(jarr_)[1], PV(jarr_)[2], PV(par_)[2], PV(par_)[3], PV(par_)[0], PV(par_)[1], ff, &cc, nullptr); } \
    if (anyweld)                                                                                                                   \
      for (int e = lane; e < ne; e += 32) {                                                                                        \
        if (!w->eq_active()[e]) continue;                                                                                          \
        for (int q = 0; q < 6; ++q) { const float D = w->w_D()[6 * e + q], j = (wjar)[6 * e + q]; cc += 0.5f * D * j * j; }        \
      }                                                                                                                            \
    if (PV(lsg_) != 0.f) { const float j = PV(lsg_) * PV(xv_) - PV(lar_); if (j < 0.f) cc += 0.5f * PV(lD_) * j * j; }            \
    PV(dst) = cc;                                                                                                                  \
  REGS_END                                                                                                                         \
  FE_WSUM(dst);

  FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_SETUP)
  // ---- the two starting candidates: the unconstrained (smooth) acceleration and the warm start; the cheaper one is kept
  COMP_MULJ(w->as(), jv_, w->w_jv(), true)  // smooth candidate rows in jv_ / w_jv
  COMP_COST(jv_, w->w_jv(), as_, a_)
  const float cost_smooth = FE_UNI(a_);
  COMP_MULJ(w->x(), jar_, w->w_jar(), true) // warm candidate rows in jar_ / w_jar
  LANES_BEGIN if (PV(z_) >= 0) w->search()[PV(z_)] = PV(x_) - PV(as_); LANES_END
  COMP_MULM(w->search(), r_)
  COMP_COST(jar_, w->w_jar(), x_, a_)
  REGS_BEGIN PV(b_) = 0.5f * (PV(x_) - PV(as_)) * PV(r_); REGS_END
  FE_WSUM(b_);
  const float cost_warm = FE_UNI(a_) + FE_UNI(b_);
  if (cost_smooth < cost_warm || !(cost_warm == cost_warm)) {
    LANES_BEGIN
      PV(x_) = PV(as_); PV(r_) = 0.f;
#pragma unroll
      for (int q = 0; q < 3; ++q) PV(jar_)[q] = PV(jv_)[q];
      if (anyweld) for (int e = lane; e < 6 * ne; e += 32) w->w_jar()[e] = w->w_jv()[e];
    LANES_END
  }

  FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_START)
  // ---------------------------------------------------------------- Newton iterations
  int iter = 0;
  float impr = 0.f;
  FE_PRIVA(float, row_, NMAX);
  FE_PRIVA(float, kq_, 21); FE_PRIVA(float, d_, 6); FE_PRIVA(float, u_, 6);
  FE_PRIV(float, ks_); FE_PRIV(float, kf_);
  FE_PRIV(int, bad_);
  for (;;) {
    // cone zone, force and cost of every contact; its share K = G^T W G of the pair's 6x6 matrix; world-frame force staged
    // for the link gather (c_f holds world-frame forces inside the loop, frame-local ones after it)
    LANES_BEGIN
      float cc = 0.f;
      const int c = PV(c_);
#pragma unroll
      for (int q = 0; q < 21; ++q) PV(kq_)[q] = 0.f;
      PV(st_) = 0;
      if (c >= 0) {
        float W[6], F[9];
        float f3[3];
        const int st = fe_cone_t<true>(PV(jar_)[0], PV(jar_)[1], PV(jar_)[2], PV(par_)[2], PV(par_)[3], PV(par_)[0], PV(par_)[1], f3, &cc, W);
        PV(st_) = st;
        PV(f_)[0] = f3[0]; PV(f_)[1] = f3[1]; PV(f_)[2] = f3[2];
        float fw[3] = {0.f, 0.f, 0.f};
        if (st != 0) {
          fe_frame_load(w, c, F);
          const float* f = f3;
          fw[0] = F[0] * f[0] + F[3] * f[1] + F[6] * f[2]; fw[1] = F[1] * f[0] + F[4] * f[1] + F[7] * f[2]; fw[2] = F[2] * f[0] + F[5] * f[1] + F[8] * f[2];
          float G[18], WG[18];
          const float r[3] = {PV(px_) - PV(ox_), PV(py_) - PV(oy_), PV(pz_) - PV(oz_)};
#pragma unroll
          for (int q = 0; q < 3; ++q) { v3cross(G + 6 * q, r, F + 3 * q); G[6 * q + 3] = F[3 * q]; G[6 * q + 4] = F[3 * q + 1]; G[6 * q + 5] = F[3 * q + 2]; }
#pragma unroll
          for (int i = 0; i < 6; ++i) { // W: xx yy zz xy xz yz
            WG[i] = W[0] * G[i] + W[3] * G[6 + i] + W[4] * G[12 + i];
            WG[6 + i] = W[3] * G[i] + W[1] * G[6 + i] + W[5] * G[12 + i];
            WG[12 + i] = W[4] * G[i] + W[5] * G[6 + i] + W[2] * G[12 + i];
          }
#pragma unroll
          for (int i = 0; i < 6; ++i)
#pragma unroll
            for (int j = 0; j <= i; ++j) PV(kq_)[i * (i + 1) / 2 + j] = G[i] * WG[j] + G[6 + i] * WG[6 + j] + G[12 + i] * WG[12 + j];
        }
        w->c_f()[3 * c] = fw[0]; w->c_f()[3 * c + 1] = fw[1]; w->c_f()[3 * c + 2] = fw[2];
      }
      if (anyweld)
        for (int e = lane; e < ne; e += 32) {
          if (!w->eq_active()[e]) continue;
          for (int q = 0; q < 6; ++q) { const float D = w->w_D()[6 * e + q], j = w->w_jar()[6 * e + q]; w->w_f()[6 * e + q] = -D * j; cc += 0.5f * D * j * j; }
        }
      PV(t_) = 0.f; // limit force of this lane's dof
      if (PV(lsg_) != 0.f) { const float j = PV(lsg_) * PV(x_) - PV(lar_); if (j < 0.f) { PV(t_) = -PV(lD_) * j; cc += 0.5f * PV(lD_) * j * j; } }
      PV(a_) = cc + 0.5f * PV(r_) * (PV(x_) - PV(as_));
    LANES_END
    // J^T f: constraint wrench of every component link from its contact list (and welds), then the dof forces
    LANES_BEGIN
      const int l = lane;
      if (l < nl && COMP_INLINK(l)) {
        float P[3], Wr[6] = {0, 0, 0, 0, 0, 0};
        fe_link_ref(w, l, P);
        for (int k = lptr[l]; k < lptr[l + 1]; ++k) {
          const int c = lidx[k] & 255;
          const float sg = (lidx[k] & 256) ? 1.f : -1.f;
          const float* fw = w->c_f() + 3 * c;
          float r[3], t[3];
          v3sub(r, w->c_pos() + 3 * c, P);
          v3cross(t, r, fw);
          Wr[0] += sg * t[0]; Wr[1] += sg * t[1]; Wr[2] += sg * t[2]; Wr[3] += sg * fw[0]; Wr[4] += sg * fw[1]; Wr[5] += sg * fw[2];
        }
        if (anyweld && l >= nrl)
          for (int e = 0; e < ne; ++e)
            if (w->eq_active()[e]) fe_weld_wrench(w, e, l, Wr);
        for (int q = 0; q < 6; ++q) w->lacc2()[6 * l + q] = Wr[q];
      }
    LANES_END
    LANES_BEGIN
      const int z = PV(z_);
      float fc = 0.f;
      if (z >= 0 && z < nr) {
        fc = PV(lsg_) * PV(t_);
        for (int l = z; l < nrl; ++l)
          if ((PV(sub_) >> l) & 1) fc += dot6(w->S() + 6 * z, w->lacc2() + 6 * l);
      } else if (z >= nr) fc = w->lacc2()[6 * (nrl + (z - nr) / 6) + (z - nr) % 6];
      PV(fc_) = fc;
      const float g = z >= 0 ? PV(r_) - fc : 0.f;
      PV(s_) = g; // gradient (becomes the right-hand side below)
      PV(b_) = g * g;
    LANES_END
    FE_WSUM(a_); FE_WSUM(b_);
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_GRAD)
    const float cost = FE_UNI(a_), gnorm = sqrtf(FE_UNI(b_));
    if (!(cost == cost)) { LANES_BEGIN if (lane == 0) w->u()[FE_U_FLAGS] |= FE_FLAG_NUMERIC; LANES_END break; }
    if (fe_newton_stop(iter, maxit, scale, impr, gnorm, tol)) break;

    // ---- Newton direction: H rows in registers
    REGS_BEGIN
      const int i = lane, zi = PV(z_);
      const float* Hi = Hm + fe_tri(zi >= 0 ? i : 0);
#pragma unroll
      for (int j = 0; j < NMAX; ++j) {
        float v = (j == i) ? 1.f : 0.f;
        if (j <= i && i < nA) v = Hi[j];
        PV(row_)[j] = v;
      }
      if (PV(lsg_) != 0.f && PV(lsg_) * PV(x_) - PV(lar_) < 0.f) { // active joint-limit row: D on the diagonal
#pragma unroll
        for (int j = 0; j < NMAX; ++j) if (j == i) PV(row_)[j] += PV(lD_);
      }
      PV(b_) = zi >= 0 ? -PV(s_) : 0.f;
    REGS_END
    {
      unsigned todo = pairs;
      while (todo) {
        int g = 0;
        while (!((todo >> g) & 1u)) ++g;
        todo &= todo - 1u;
        REGS_BEGIN PV(kf_) = (float)PV(key_); PV(any_) = (PV(lead_) == g && PV(c_) >= 0 && PV(st_) != 0) ? 1 : 0; REGS_END
        if (!FE_ANY(any_)) continue; // no contact of this pair is active
        FE_SHFL(ks_, PV_ALL(px_), g); const float p0x = FE_UNI(ks_);
        FE_SHFL(ks_, PV_ALL(py_), g); const float p0y = FE_UNI(ks_);
        FE_SHFL(ks_, PV_ALL(pz_), g); const float p0z = FE_UNI(ks_);
        FE_SHFL(ks_, PV_ALL(kf_), g);
        const int gkey = (int)FE_UNI(ks_), A = (gkey & 255) - 1, B = (gkey >> 8) - 1;
        const int mA = (A >= 0 && A < nrl) ? m->link_ancmask[A] : 0, mB = (B >= 0 && B < nrl) ? m->link_ancmask[B] : 0;
        const float p0[3] = {p0x, p0y, p0z};
        REGS_BEGIN // this lane's dof: its unit contribution to the relative twist of the pair (B side minus A side), at p0
          fe_unit_twist(w, PV(z_), A, B, mA, mB, p0, Pr, PV(d_));
#pragma unroll
          for (int q = 0; q < 6; ++q) PV(u_)[q] = 0.f;
        REGS_END
        // u_i = K d_i, K[a][b] = sum of the members' terms
#pragma unroll
        for (int a = 0; a < 6; ++a) {
#pragma unroll
          for (int b = 0; b <= a; ++b) {
            REGS_BEGIN PV(ks_) = (PV(lead_) == g && PV(c_) >= 0) ? PV(kq_)[a * (a + 1) / 2 + b] : 0.f; REGS_END
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
          for (int q = 0; q < 6; ++q) {
            FE_SHFLA(ks_, d_, q, j);
            REGS_BEGIN PV(row_)[j] += PV(u_)[q] * PV(ks_); REGS_END
          }
        }
      }
    }
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_HESSIAN)
    FE_REG_CHOL_SOLVE(NMAX, row_, b_, bad_)
    LANES_BEGIN
      PV(s_) = PV(z_) >= 0 ? PV(b_) : 0.f;
      if (PV(z_) >= 0) w->search()[PV(z_)] = PV(s_);
      if (PV(bad_) && lane == 0) w->u()[FE_U_FLAGS] |= FE_FLAG_NEWTON_PIVOT;
    LANES_END
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_CHOL)
    // products with the search direction
    COMP_MULM(w->search(), Ms_)
    COMP_MULJ(w->search(), jv_, w->w_jv(), false)
    REGS_BEGIN PV(a_) = PV(s_) * PV(r_); PV(b_) = 0.5f * PV(s_) * PV(Ms_); REGS_END
    FE_WSUM(a_); FE_WSUM(b_);
    const float g1 = FE_UNI(a_), g2 = FE_UNI(b_);
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_PRODUCTS)
    FeLineSearch ls; // evaluation -1 is at alpha = 0
    for (int k = -1; k < maxls; ++k) {
      const float alpha = ls.alpha;
      REGS_BEGIN
        float q1 = 0.f, q2 = 0.f;
        if (PV(c_) >= 0) FE_CONE_LS(PV(jar_), PV(jv_), alpha, PV(par_)[2], PV(par_)[3], PV(par_)[0], PV(par_)[1], q1, =, q2)
        if (anyweld)
          for (int e = lane; e < ne; e += 32) {
            if (!w->eq_active()[e]) continue;
            for (int q = 0; q < 6; ++q) {
              const float D = w->w_D()[6 * e + q], v = w->w_jv()[6 * e + q], x = w->w_jar()[6 * e + q] + alpha * v;
              q1 += D * x * v; q2 += D * v * v;
            }
          }
        if (PV(lsg_) != 0.f) {
          const float v = PV(lsg_) * PV(s_), x = PV(lsg_) * PV(x_) - PV(lar_) + alpha * v;
          if (x < 0.f) { q1 += PV(lD_) * x * v; q2 += PV(lD_) * v * v; }
        }
        PV(a_) = q1; PV(b_) = q2;
      REGS_END
      FE_WSUM(a_); FE_WSUM(b_);
      const float p1 = FE_UNI(a_) + g1 + 2.f * alpha * g2, p2 = FE_UNI(b_) + 2.f * g2;
      if (!(k < 0 ? ls.start(p1, p2) : ls.step(p1, p2))) break;
    }
    FE_TICK(w->u() + FE_U_STAT, FE_STAT_NEWTON_LS)
    const float alpha = ls.alpha;
    if (!(alpha > 0.f)) break;
    impr = ls.impr();
    LANES_BEGIN
      PV(x_) += alpha * PV(s_); PV(r_) += alpha * PV(Ms_);
#pragma unroll
      for (int q = 0; q < 3; ++q) PV(jar_)[q] += alpha * PV(jv_)[q];
      if (anyweld) for (int e = lane; e < 6 * ne; e += 32) w->w_jar()[e] += alpha * w->w_jv()[e];
    LANES_END
    ++iter;
  }
  // results: iterate, constraint force in solver coordinates, contact states and frame-local forces
  LANES_BEGIN
    const int z = PV(z_);
    if (z >= 0) {
      w->x()[z] = PV(x_); w->fc()[z] = PV(fc_);
      if (z < nr) { w->l_f()[z] = PV(t_); w->l_jar()[z] = PV(lsg_) * PV(x_) - PV(lar_); }
    }
    const int c = PV(c_);
    if (c >= 0) {
      w->c_state()[c] = PV(st_);
      w->c_f()[3 * c] = PV(f_)[0]; w->c_f()[3 * c + 1] = PV(f_)[1]; w->c_f()[3 * c + 2] = PV(f_)[2];
#pragma unroll
      for (int q = 0; q < 3; ++q) w->c_jar()[3 * c + q] = PV(jar_)[q];
    }
    if (lane == 0) { if (iter > w->u()[FE_U_NITER]) w->u()[FE_U_NITER] = iter; w->u()[FE_U_STAT + FE_STAT_NEWTON_ITERS] += iter; w->u()[FE_U_STAT + FE_STAT_NEWTON_SOLVES] += 1; }
  LANES_END
#undef COMP_MULJ
#undef COMP_MULM
#undef COMP_COST
#undef COMP_INLINK
#undef COMP_POS
}
