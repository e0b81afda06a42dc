// SPDX-License-Identifier: Apache-2.0
//
// sim_pair.cuh -- the physics substep with the LEFT and RIGHT leg carried as
// (left, right) pairs.
//
// The two legs of the robot run the same arithmetic on different data, so every
// per-leg scalar of sim_core.cuh becomes an f2 = (left, right) and the per-leg model
// constants are stored as adjacent pairs in SimParams. On sm_90 each pair operation
// is two scalar instructions with explicit rounding (fma2 / mul2 / add2 below). A
// negated operand (neg2) costs nothing there: FFMA and FMUL negate their inputs, and
// fma(-a, b, c) rounds exactly as fma(na, b, c) with na = -a, so no negated copies
// are kept in registers.
//
// Included by sim_core.cuh; same mathematics as the scalar functions there, which
// remain available with -DUPKIE_PAIRED_LEGS=0.
#pragma once

#include <type_traits>

namespace upkie_b200 {

UPKIE_HD f2 mk2(float a, float b) { f2 r; r.x = a; r.y = b; return r; }
UPKIE_HD f2 bc2(float a) { return mk2(a, a); }          // broadcast
UPKIE_HD f2 swp2(f2 v) { return mk2(v.y, v.x); }       // lane swap (free: .LO_HI operand modifier)
#if defined(__CUDA_ARCH__)
// sm_90 has no packed f32x2 arithmetic: each lane is one scalar instruction with round-to-nearest intrinsics, which the
// compiler may neither contract nor reassociate, so the results match a packed (FFMA2 / FMUL2 / FADD2) build bit for bit.
UPKIE_HD f2 neg2(f2 v) { return mk2(-v.x, -v.y); }
UPKIE_HD f2 fma2(f2 a, f2 b, f2 c) { return mk2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
UPKIE_HD f2 mul2(f2 a, f2 b) { return mk2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
UPKIE_HD f2 add2(f2 a, f2 b) { return mk2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
#else
UPKIE_HD f2 neg2(f2 v) { return mk2(-v.x, -v.y); }
UPKIE_HD f2 fma2(f2 a, f2 b, f2 c) { return mk2(a.x * b.x + c.x, a.y * b.y + c.y); }
UPKIE_HD f2 mul2(f2 a, f2 b) { return mk2(a.x * b.x, a.y * b.y); }
UPKIE_HD f2 add2(f2 a, f2 b) { return mk2(a.x + b.x, a.y + b.y); }
#endif
UPKIE_HD f2 sub2(f2 a, f2 b) { return add2(a, neg2(b)); }

UPKIE_HD void cross3_2(const f2 a[3], const f2 b[3], f2 c[3]) {
  c[0] = fma2(a[1], b[2], neg2(mul2(a[2], b[1])));
  c[1] = fma2(a[2], b[0], neg2(mul2(a[0], b[2])));
  c[2] = fma2(a[0], b[1], neg2(mul2(a[1], b[0])));
}

// S^T x for S = s * [0 1 0 | -oz 0 ox], both legs
UPKIE_HD f2 sdot2(f2 s, f2 ox, f2 oz, const f2 x[6]) { return mul2(s, fma2(ox, x[5], fma2(neg2(oz), x[3], x[1]))); }

struct LegCache2 {
  f2 ox[3], oz[3];  // joint origins (x, z) in the base frame
  f2 U[3][6];
  f2 invD[3];       // 1 / D
};

// two right-hand sides at once against the scalar LDL^T factors of ldl6()
UPKIE_HD void ldl6_solve2(const float A[21], f2 x[6]) {
#pragma unroll
  for (int i = 1; i < 6; ++i) {
#pragma unroll
    for (int k = 0; k < i; ++k) x[i] = fma2(bc2(-A[SI(k, i)]), x[k], x[i]);
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) x[i] = mul2(x[i], bc2(A[SI(i, i)]));
#pragma unroll
  for (int i = 4; i >= 0; --i) {
#pragma unroll
    for (int k = i + 1; k < 6; ++k) x[i] = fma2(bc2(-A[SI(i, k)]), x[k], x[i]);
  }
}

// Both legs of leg_pass12 at once.
// `locked`: every joint is held (spine mode, servos stopped: Bullet velocity motors holding 0 rad/s with 100 N m,
// BulletInterface.cpp:296-301, restated as locked joints): 1 / D -> 0, so that a joint transmits everything - no
// reduction of the articulated inertia, no joint acceleration, no joint response to impulses further down the file.
UPKIE_HD void legs_pass12(const SimParams& P, const float q[6], const float qd[6], const float tau[6], const float V0[6],
                          const float* eps, LegCache2& lc, f2 cc[3][6], f2 uu[3], float IA0[21], float pA0[6],
                          bool locked = false) {
  const f2 free2 = bc2(locked ? 0.f : 1.f);
  f2 cphi[3], sphi[3];
  f2 V[3][6];
  {
    f2 phi = bc2(0.f), cp = bc2(1.f), sp = bc2(0.f), ox = bc2(0.f), oz = bc2(0.f);
    f2 Vc[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) Vc[i] = bc2(V0[i]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const f2 s = P.sgn2[k];
      // origin of body k: parent origin + Ry(phi_parent) * joint origin
      const f2 ox_n = fma2(cp, P.jo2[k][0], fma2(sp, P.jo2[k][2], ox));
      const f2 oz_n = fma2(cp, P.jo2[k][2], fma2(neg2(sp), P.jo2[k][0], oz));
      ox = ox_n;
      oz = oz_n;
      lc.ox[k] = ox;
      lc.oz[k] = oz;
      phi = fma2(s, mk2(q[k], q[k + 3]), phi);
      if (k < 2 || !P.wheel_symmetric) {
        float sx, cx, sy, cy;
        sincosf(phi.x - 6.28318530718f * rintf(phi.x * 0.15915494309f), &sx, &cx);
        sincosf(phi.y - 6.28318530718f * rintf(phi.y * 0.15915494309f), &sy, &cy);
        sp = mk2(sx, sy);
        cp = mk2(cx, cy);
      }
      cphi[k] = cp;
      sphi[k] = sp;
      const f2 w = mul2(s, mk2(qd[k], qd[k + 3]));
      Vc[1] = add2(Vc[1], w);
      Vc[3] = fma2(neg2(oz), w, Vc[3]);
      Vc[5] = fma2(ox, w, Vc[5]);
#pragma unroll
      for (int i = 0; i < 6; ++i) V[k][i] = Vc[i];
    }
  }
  f2 IA[21], pA[6];
#pragma unroll
  for (int k = 2; k >= 0; --k) {
    const f2 s = P.sgn2[k];
    const f2 ox = lc.ox[k], oz = lc.oz[k];
    const f2 scale = eps ? mk2(1.f + eps[k], 1.f + eps[k + 3]) : bc2(1.f);
    const f2 m = mul2(P.mass2[k], scale);
    f2 C[3], Ib[6];
    if (k == 2 && P.wheel_symmetric) {
      C[0] = ox; C[1] = P.oy2[k]; C[2] = oz;
      Ib[0] = mul2(P.inertia2[k][0], scale); Ib[1] = mul2(P.inertia2[k][1], scale); Ib[2] = mul2(P.inertia2[k][2], scale);
      Ib[3] = bc2(0.f); Ib[4] = bc2(0.f); Ib[5] = bc2(0.f);
    } else {
      const f2 c = cphi[k], sn = sphi[k];
      C[0] = fma2(c, P.com2[k][0], fma2(sn, P.com2[k][2], ox));
      C[1] = add2(P.com2[k][1], P.oy2[k]);
      C[2] = fma2(c, P.com2[k][2], fma2(neg2(sn), P.com2[k][0], oz));
      const f2 a = mul2(P.inertia2[k][0], scale), bb = mul2(P.inertia2[k][1], scale), cz = mul2(P.inertia2[k][2], scale);
      const f2 d = mul2(P.inertia2[k][3], scale), e = mul2(P.inertia2[k][4], scale), f = mul2(P.inertia2[k][5], scale);
      const f2 c2 = mul2(c, c), s2 = mul2(sn, sn), cs = mul2(c, sn), cs2 = add2(cs, cs);
      Ib[0] = fma2(c2, a, fma2(cs2, e, mul2(s2, cz)));
      Ib[1] = bb;
      Ib[2] = fma2(s2, a, fma2(neg2(cs2), e, mul2(c2, cz)));
      Ib[3] = fma2(c, d, mul2(sn, f));
      Ib[4] = fma2(cs, sub2(cz, a), mul2(sub2(c2, s2), e));
      Ib[5] = fma2(c, f, neg2(mul2(sn, d)));
    }
    // spatial inertia about the base origin
    f2 I[21];
    {
      const f2 cc2 = fma2(C[0], C[0], fma2(C[1], C[1], mul2(C[2], C[2])));
      I[SI(0, 0)] = fma2(m, sub2(cc2, mul2(C[0], C[0])), Ib[0]);
      I[SI(1, 1)] = fma2(m, sub2(cc2, mul2(C[1], C[1])), Ib[1]);
      I[SI(2, 2)] = fma2(m, sub2(cc2, mul2(C[2], C[2])), Ib[2]);
      const f2 hx = mul2(m, C[0]), hy = mul2(m, C[1]), hz = mul2(m, C[2]);
      I[SI(0, 1)] = fma2(neg2(hx), C[1], Ib[3]);
      I[SI(0, 2)] = fma2(neg2(hx), C[2], Ib[4]);
      I[SI(1, 2)] = fma2(neg2(hy), C[2], Ib[5]);
      I[SI(0, 3)] = bc2(0.f); I[SI(0, 4)] = neg2(hz); I[SI(0, 5)] = hy;
      I[SI(1, 3)] = hz;       I[SI(1, 4)] = bc2(0.f); I[SI(1, 5)] = neg2(hx);
      I[SI(2, 3)] = neg2(hy); I[SI(2, 4)] = hx;       I[SI(2, 5)] = bc2(0.f);
      I[SI(3, 3)] = m; I[SI(4, 4)] = m; I[SI(5, 5)] = m;
      I[SI(3, 4)] = bc2(0.f); I[SI(3, 5)] = bc2(0.f); I[SI(4, 5)] = bc2(0.f);
    }
    // momentum, bias force p = V x* (I V) - damping wrench
    f2 p[6];
    f2 spin_damp = bc2(0.f);  // damping moment about the body's own y axis (closed-form wheel leaf below)
    {
      const f2* om = &V[k][0];
      const f2* v = &V[k][3];
      f2 t[3], vC[3];
      cross3_2(om, C, t);
      vC[0] = add2(v[0], t[0]); vC[1] = add2(v[1], t[1]); vC[2] = add2(v[2], t[2]);
      const f2 f[3] = {mul2(m, vC[0]), mul2(m, vC[1]), mul2(m, vC[2])};
      const f2 nC[3] = {fma2(Ib[0], om[0], fma2(Ib[3], om[1], mul2(Ib[4], om[2]))),
                        fma2(Ib[3], om[0], fma2(Ib[1], om[1], mul2(Ib[5], om[2]))),
                        fma2(Ib[4], om[0], fma2(Ib[5], om[1], mul2(Ib[2], om[2])))};
      f2 n[3];
      cross3_2(C, f, n);
      n[0] = add2(n[0], nC[0]); n[1] = add2(n[1], nC[1]); n[2] = add2(n[2], nC[2]);
      f2 a1[3], a2[3], a3[3];
      cross3_2(om, n, a1);
      cross3_2(v, f, a2);
      cross3_2(om, f, a3);
      // Bullet-style damping: F = -m vC (k + k|vC|), N = -Ic om (k + k|om|)
      const f2 v2 = fma2(vC[0], vC[0], fma2(vC[1], vC[1], mul2(vC[2], vC[2])));
      const f2 o2 = fma2(om[0], om[0], fma2(om[1], om[1], mul2(om[2], om[2])));
      const f2 gl = fma2(bc2(P.lin_damp), mk2(sqrtf(v2.x), sqrtf(v2.y)), bc2(P.lin_damp));
      const f2 ga = fma2(bc2(P.ang_damp), mk2(sqrtf(o2.x), sqrtf(o2.y)), bc2(P.ang_damp));
      const f2 F[3] = {mul2(f[0], gl), mul2(f[1], gl), mul2(f[2], gl)};  // = -damping force
      f2 cF[3];
      cross3_2(C, F, cF);
      p[0] = add2(add2(a1[0], a2[0]), fma2(nC[0], ga, cF[0]));
      p[1] = add2(add2(a1[1], a2[1]), fma2(nC[1], ga, cF[1]));
      p[2] = add2(add2(a1[2], a2[2]), fma2(nC[2], ga, cF[2]));
      p[3] = add2(a3[0], F[0]);
      p[4] = add2(a3[1], F[1]);
      p[5] = add2(a3[2], F[2]);
      spin_damp = mul2(nC[1], ga);
    }
    if (k == 2) {
#pragma unroll
      for (int i = 0; i < 21; ++i) IA[i] = I[i];
#pragma unroll
      for (int i = 0; i < 6; ++i) pA[i] = p[i];
    } else {
#pragma unroll
      for (int i = 0; i < 21; ++i) IA[i] = add2(IA[i], I[i]);
#pragma unroll
      for (int i = 0; i < 6; ++i) pA[i] = add2(pA[i], p[i]);
    }
    // velocity-product acceleration c = V x (S qd)
    {
      const f2 w = mul2(s, mk2(qd[k], qd[k + 3]));
      const f2* om = &V[k][0];
      const f2* v = &V[k][3];
      cc[k][0] = neg2(mul2(om[2], w));
      cc[k][1] = bc2(0.f);
      cc[k][2] = mul2(om[0], w);
      cc[k][3] = mul2(fma2(om[1], ox, neg2(v[2])), w);
      cc[k][4] = neg2(mul2(fma2(om[2], oz, mul2(om[0], ox)), w));
      cc[k][5] = mul2(fma2(om[1], oz, v[0]), w);
    }
    // U = IA S, D = S^T U, u = tau - S^T pA
    f2 U[6], invD, u;
    if (k == 2 && P.wheel_symmetric) {
      // The wheel is a leaf whose centre of mass lies on its joint axis, with Ixx = Izz: spinning it moves no
      // mass, so U = (0, s Iyy, 0 | 0, 0, 0), D = Iyy, and S^T pA is the damping moment about the axis alone
      // (the gyroscopic term om x Ic om has no y component). Taking these closed forms instead of S^T IA S
      // about the base origin avoids the m |o|^2 / Iyy ~ 150x cancellation that otherwise dominates the fp32
      // error of the wheel rates (DESIGN.md section 5, "fp32 budget").
      const f2 Iyy = Ib[1];
#pragma unroll
      for (int r = 0; r < 6; ++r) U[r] = bc2(0.f);
      U[1] = mul2(s, Iyy);
      invD = mul2(free2, mk2(1.f / Iyy.x, 1.f / Iyy.y));
      u = sub2(mk2(tau[k], tau[k + 3]), mul2(s, spin_damp));
      // Ia = IA - U U^T / D: the rotor stops resisting rotation about its own axis; pa = pA + Ia c + S u
      IA[SI(1, 1)] = fma2(neg2(free2), Iyy, IA[SI(1, 1)]);
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        f2 acc = pA[r];
#pragma unroll
        for (int c2 = 0; c2 < 6; ++c2) {
          if (c2 != 1) acc = fma2(IA[SI(r, c2)], cc[k][c2], acc);  // cc[k][1] = 0
        }
        p[r] = acc;
      }
      p[1] = fma2(mul2(s, free2), u, p[1]);
    } else {
#pragma unroll
      for (int r = 0; r < 6; ++r) U[r] = mul2(s, fma2(ox, IA[SI(r, 5)], fma2(neg2(oz), IA[SI(r, 3)], IA[SI(r, 1)])));
      const f2 D = sdot2(s, ox, oz, U);
      invD = mul2(free2, mk2(1.f / D.x, 1.f / D.y));
      u = sub2(mk2(tau[k], tau[k + 3]), sdot2(s, ox, oz, pA));
      // Ia = IA - U U^T / D ; pa = pA + Ia c + U u / D
      f2 nUd[6];
#pragma unroll
      for (int r = 0; r < 6; ++r) nUd[r] = mul2(U[r], neg2(invD));
#pragma unroll
      for (int r = 0; r < 6; ++r) {
#pragma unroll
        for (int c2 = r; c2 < 6; ++c2) IA[SI(r, c2)] = fma2(nUd[r], U[c2], IA[SI(r, c2)]);
      }
      const f2 ud = mul2(u, invD);
#pragma unroll
      for (int r = 0; r < 6; ++r) {
        f2 acc = fma2(U[r], ud, pA[r]);
#pragma unroll
        for (int c2 = 0; c2 < 6; ++c2) acc = fma2(IA[SI(r, c2)], cc[k][c2], acc);
        p[r] = acc;
      }
    }
#pragma unroll
    for (int r = 0; r < 6; ++r) lc.U[k][r] = U[r];
    lc.invD[k] = invD;
    uu[k] = u;
#pragma unroll
    for (int r = 0; r < 6; ++r) pA[r] = p[r];
  }
#pragma unroll
  for (int i = 0; i < 21; ++i) IA0[i] += IA[i].x + IA[i].y;
#pragma unroll
  for (int i = 0; i < 6; ++i) pA0[i] += pA[i].x + pA[i].y;
}

// joint accelerations down both legs given the base acceleration
UPKIE_HD void legs_pass3(const SimParams& P, const LegCache2& lc, const f2 cc[3][6], const f2 uu[3], const float a0[6],
                         float qdd[6]) {
  f2 a[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) a[i] = bc2(a0[i]);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    f2 dot = bc2(0.f);
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      a[i] = add2(a[i], cc[k][i]);
      dot = fma2(lc.U[k][i], a[i], dot);
    }
    const f2 dd = fma2(dot, neg2(lc.invD[k]), mul2(uu[k], lc.invD[k]));  // (u - U.a) / D
    qdd[k] = dd.x;
    qdd[k + 3] = dd.y;
    const f2 w = mul2(P.sgn2[k], dd);
    a[1] = add2(a[1], w);
    a[3] = fma2(neg2(lc.oz[k]), w, a[3]);
    a[5] = fma2(lc.ox[k], w, a[5]);
  }
}

// lane x: impulse f.x on the LEFT wheel up the left leg; lane y: f.y on the RIGHT wheel up the right leg
// Carries q = -p (so q starts as +f): u_k = -S^T p = S^T q, q <- q - U u / D. Returns nptop = -ptop, the force the
// base feels with its sign flipped, i.e. the right-hand side of IA0 a0 = -ptop as is.
UPKIE_HD void legs_impulse_up(const SimParams& P, const LegCache2& lc, const f2 f[6], f2 uu[3], f2 nptop[6]) {
  f2 q[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) q[i] = f[i];
#pragma unroll
  for (int k = 2; k >= 0; --k) {
    const f2 u = sdot2(P.sgn2[k], lc.ox[k], lc.oz[k], q);
    uu[k] = u;
    const f2 nud = mul2(u, neg2(lc.invD[k]));
#pragma unroll
    for (int i = 0; i < 6; ++i) q[i] = fma2(lc.U[k][i], nud, q[i]);
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) nptop[i] = q[i];
}

// Velocity changes down the legs. SWAP = false: lane x walks the left leg, lane y the right leg (with the
// per-joint u's of legs_impulse_up). SWAP = true: lane x walks the RIGHT leg, lane y the LEFT leg with u = 0
// (the leg the impulse was not applied to); the leg constants are read lane-swapped, which is free in SASS.
template <bool SWAP>
UPKIE_HD void legs_impulse_down(const SimParams& P, const LegCache2& lc, const f2 uu[3], const f2 a0[6], f2 aw[6],
                                f2 dqd[3]) {
#pragma unroll
  for (int i = 0; i < 6; ++i) aw[i] = a0[i];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    f2 dot = bc2(0.f);
#pragma unroll
    for (int i = 0; i < 6; ++i) dot = fma2(SWAP ? swp2(lc.U[k][i]) : lc.U[k][i], aw[i], dot);
    const f2 invD = SWAP ? swp2(lc.invD[k]) : lc.invD[k];
    const f2 dd = SWAP ? mul2(dot, neg2(invD)) : fma2(dot, neg2(invD), mul2(uu[k], invD));
    dqd[k] = dd;
    const f2 w = mul2(SWAP ? swp2(P.sgn2[k]) : P.sgn2[k], dd);
    aw[1] = add2(aw[1], w);
    aw[3] = fma2(neg2(SWAP ? swp2(lc.oz[k]) : lc.oz[k]), w, aw[3]);
    aw[5] = fma2(SWAP ? swp2(lc.ox[k]) : lc.ox[k], w, aw[5]);
  }
}

// ---- joint-limit rows: the slow path ------------------------------------------------------------------------------
// PyBullet's URDF importer hangs a btMultiBodyJointLimitConstraint on every revolute joint with limits (hips and
// knees). While such a joint sits at or beyond a bound, one unilateral row along its coordinate joins the contact rows
// of the substep's PGS solve. That is rare (position commands are clamped to the limits upstream), so a robot with
// an active limit row solves ALL of its rows here - scalar, looped, local-memory arrays - and stays out of the packed
// six-row solver below, whose registers and instruction count are what the roofline is quoted on.
// Restated from Bullet 3.24 (third-party, absent from the reference tree; DESIGN.md): rows only while
// `penetration <= 0`, rhs = (-penetration * erp / h - rel_vel) / W_kk, impulse in [0, m_maxAppliedImpulse], limit rows
// before the contact normals and walked backwards on even sweeps, forwards on odd ones.
struct LimitRows {
  int n;
  int joint[4];
  float dir[4], pen[4];
};

UPKIE_HD float lane(const f2& v, int leg) { return leg == 0 ? v.x : v.y; }

UPKIE_HD int active_joint_limits(const SimParams& P, const float q[6], LimitRows& L) {
  L.n = 0;
  for (int j = 0; j < 6; ++j) {
    // wheels carry infinite bounds: both tests fail for them
    const float pen_lo = q[j] - P.q_lower[j], pen_hi = P.q_upper[j] - q[j];
    if (pen_lo <= 0.f && L.n < 4) { L.joint[L.n] = j; L.dir[L.n] = 1.f; L.pen[L.n] = pen_lo; ++L.n; }
    if (pen_hi <= 0.f && L.n < 4) { L.joint[L.n] = j; L.dir[L.n] = -1.f; L.pen[L.n] = pen_hi; ++L.n; }
  }
  return L.n;
}

// Velocity change for spatial impulses fw[side] on the two wheels (about the base origin, base coordinates) plus
// generalized impulses g[j] on the joint coordinates: da0 (base), dqd (joints), aw[side] (wheel bodies).
UPKIE_HD void impulse_response_generic(const SimParams& P, const LegCache2& lc, const float IA0[21], const float fw[2][6],
                                       const float g[6], float da0[6], float dqd[6], float aw[2][6]) {
  float u[6];
  for (int i = 0; i < 6; ++i) da0[i] = 0.f;
  for (int leg = 0; leg < 2; ++leg) {
    float q[6];  // q = -p
    for (int i = 0; i < 6; ++i) q[i] = fw[leg][i];
    for (int k = 2; k >= 0; --k) {
      const float s = lane(P.sgn2[k], leg), ox = lane(lc.ox[k], leg), oz = lane(lc.oz[k], leg);
      const float uj = s * (q[1] - oz * q[3] + ox * q[5]) + g[3 * leg + k];
      u[3 * leg + k] = uj;
      const float c = uj * lane(lc.invD[k], leg);
      for (int i = 0; i < 6; ++i) q[i] -= lane(lc.U[k][i], leg) * c;
    }
    for (int i = 0; i < 6; ++i) da0[i] += q[i];
  }
  ldl6_solve(IA0, da0);
  for (int leg = 0; leg < 2; ++leg) {
    float a[6];
    for (int i = 0; i < 6; ++i) a[i] = da0[i];
    for (int k = 0; k < 3; ++k) {
      float dot = 0.f;
      for (int i = 0; i < 6; ++i) dot += lane(lc.U[k][i], leg) * a[i];
      const float dd = (u[3 * leg + k] - dot) * lane(lc.invD[k], leg);
      dqd[3 * leg + k] = dd;
      const float w = lane(P.sgn2[k], leg) * dd;
      a[1] += w;
      a[3] -= lane(lc.oz[k], leg) * w;
      a[5] += lane(lc.ox[k], leg) * w;
    }
    for (int i = 0; i < 6; ++i) aw[leg][i] = a[i];
  }
}

// All constraint rows of one robot with at least one active joint limit: limit rows, then nL nR, then t1 t2 per wheel
// in contact. Updates the velocities and the cached normal impulses of S.
UPKIE_HD void limit_contact_solve(const SimParams& P, RobotState& S, const LegCache2& lc, const float IA0[21],
                                  const float R[9], const float zb[3], float inv_n, const f2 Pc[3], const f2& dist,
                                  bool actL, bool actR, float mu, const LimitRows& L, const float lam_prev[2]) {
  constexpr int kMaxRows = 10;
  int kind[kMaxRows], side[kMaxRows], joint[kMaxRows], partner[kMaxRows];  // kind 0 normal, 1 friction, 2 limit
  float dirj[kMaxRows], J[kMaxRows][6];
  int n = 0;
  for (int l = 0; l < L.n; ++l) {
    kind[n] = 2; side[n] = -1; joint[n] = L.joint[l]; dirj[n] = L.dir[l]; partner[n] = -1;
    for (int i = 0; i < 6; ++i) J[n][i] = 0.f;
    ++n;
  }
  const int nlimit = n;
  const float t1[3] = {zb[2] * inv_n, 0.f, -zb[0] * inv_n};
  float t2[3];
  cross3(zb, t1, t2);
  const bool act[2] = {actL, actR};
  int normal_of[2] = {-1, -1};
  auto add_contact_row = [&](int sd, int d) {
    const float sw = lane(P.sgn2[2], sd);
    const float pc[3] = {lane(Pc[0], sd), lane(Pc[1], sd), lane(Pc[2], sd)};
    float dir[3];
    for (int i = 0; i < 3; ++i) dir[i] = d == 0 ? zb[i] : sw * (d == 1 ? t1[i] : t2[i]);
    cross3(pc, dir, &J[n][0]);
    J[n][3] = dir[0]; J[n][4] = dir[1]; J[n][5] = dir[2];
    kind[n] = d == 0 ? 0 : 1; side[n] = sd; joint[n] = -1; dirj[n] = 0.f;
    partner[n] = d == 0 ? -1 : normal_of[sd];
    if (d == 0) normal_of[sd] = n;
    ++n;
  };
  for (int sd = 0; sd < 2; ++sd)
    if (act[sd]) add_contact_row(sd, 0);
  for (int sd = 0; sd < 2; ++sd)
    if (act[sd]) { add_contact_row(sd, 1); add_contact_row(sd, 2); }

  // wheel spatial velocities at the predicted generalized velocity
  float Vw[2][6];
  {
    float Vb[6];
    rot_tmul(R, S.angvel, &Vb[0]);
    rot_tmul(R, S.linvel, &Vb[3]);
    for (int sd = 0; sd < 2; ++sd) {
      for (int i = 0; i < 6; ++i) Vw[sd][i] = Vb[i];
      for (int k = 0; k < 3; ++k) {
        const float w = lane(P.sgn2[k], sd) * S.qd[3 * sd + k];
        Vw[sd][1] += w;
        Vw[sd][3] -= lane(lc.oz[k], sd) * w;
        Vw[sd][5] += lane(lc.ox[k], sd) * w;
      }
    }
  }
  // Delassus matrix, one generic response per row
  float W[kMaxRows][kMaxRows];
  for (int l = 0; l < n; ++l) {
    float fw[2][6], g[6], da0[6], dqd[6], aw[2][6];
    for (int i = 0; i < 6; ++i) { fw[0][i] = 0.f; fw[1][i] = 0.f; g[i] = 0.f; }
    if (kind[l] == 2) g[joint[l]] = dirj[l];
    else for (int i = 0; i < 6; ++i) fw[side[l]][i] = J[l][i];
    impulse_response_generic(P, lc, IA0, fw, g, da0, dqd, aw);
    for (int k = 0; k < n; ++k) {
      float wkl;
      if (kind[k] == 2) {
        wkl = dirj[k] * dqd[joint[k]];
      } else {
        wkl = 0.f;
        for (int i = 0; i < 6; ++i) wkl += J[k][i] * aw[side[k]][i];
      }
      W[k][l] = wkl;
    }
  }
  float rhs[kMaxRows], jdi[kMaxRows], cfmrow[kMaxRows], lam[kMaxRows];
  for (int k = 0; k < n; ++k) {
    lam[k] = 0.f;
    if (kind[k] == 2) {
      const float rel = dirj[k] * S.qd[joint[k]];
      jdi[k] = W[k][k] > 1.1920929e-7f ? 1.f / W[k][k] : 0.f;
      rhs[k] = (-L.pen[k] * P.limit_erp * P.inv_h - rel) * jdi[k];
      cfmrow[k] = 0.f;
      continue;
    }
    float rel = 0.f;
    for (int i = 0; i < 6; ++i) rel += J[k][i] * Vw[side[k]][i];
    if (kind[k] == 0) {
      lam[k] = P.warm * lam_prev[side[k]];
      const float pen = lane(dist, side[k]);
      jdi[k] = 1.f / (W[k][k] + P.cfm);
      float pos_err = 0.f, vel_err = -rel;
      if (pen > 0.f) vel_err -= pen * P.inv_h;
      else pos_err = -pen * P.erp * P.inv_h;
      rhs[k] = (pos_err + vel_err) * jdi[k];
      cfmrow[k] = P.cfm * jdi[k];
    } else {
      jdi[k] = W[k][k] > 0.f ? 1.f / W[k][k] : 0.f;
      rhs[k] = -rel * jdi[k];
      cfmrow[k] = 0.f;
    }
  }
  for (int it = 0; it < P.pgs_iterations; ++it) {
    float res = 0.f;  // largest velocity-level row change of the sweep (Bullet's residual, see pgs_solve())
    for (int pos = 0; pos < n; ++pos) {
      const int k = pos < nlimit ? ((it & 1) ? pos : nlimit - 1 - pos) : pos;
      float jdv = 0.f;
      for (int l = 0; l < n; ++l) jdv += W[k][l] * lam[l];
      const float sum = lam[k] + (rhs[k] - lam[k] * cfmrow[k] - jdv * jdi[k]);
      float lo, hi;
      if (kind[k] == 0) { lo = 0.f; hi = 1e10f; }
      else if (kind[k] == 2) { lo = 0.f; hi = P.limit_max_impulse; }
      else { hi = mu * lam[partner[k]]; lo = -hi; }
      const float nl = fminf(fmaxf(sum, lo), hi);
      if (jdi[k] != 0.f) res = fmaxf(res, fabsf(nl - lam[k]) / jdi[k]);
      lam[k] = nl;
    }
    if (res * res <= P.res_thr) break;  // per robot
  }
  // apply the total impulse
  float fw[2][6], g[6], da0[6], dqd[6], aw[2][6];
  for (int i = 0; i < 6; ++i) { fw[0][i] = 0.f; fw[1][i] = 0.f; g[i] = 0.f; }
  S.lam_n[0] = 0.f;
  S.lam_n[1] = 0.f;
  for (int k = 0; k < 4; ++k) S.lam_t[k] = 0.f;
  int nfric[2] = {0, 0};
  for (int k = 0; k < n; ++k) {
    if (kind[k] == 2) {
      g[joint[k]] += dirj[k] * lam[k];
    } else {
      for (int i = 0; i < 6; ++i) fw[side[k]][i] += J[k][i] * lam[k];
      if (kind[k] == 0) S.lam_n[side[k]] = lam[k];
      else S.lam_t[2 * side[k] + nfric[side[k]]++] = lam[k];  // rolling row first, then lateral (add_contact_row order)
    }
  }
  impulse_response_generic(P, lc, IA0, fw, g, da0, dqd, aw);
  float dw[3], dv[3];
  rot_mul(R, &da0[0], dw);
  rot_mul(R, &da0[3], dv);
  for (int i = 0; i < 3; ++i) {
    S.angvel[i] = clampf(S.angvel[i] + dw[i], -P.vmax, P.vmax);
    S.linvel[i] = clampf(S.linvel[i] + dv[i], -P.vmax, P.vmax);
  }
  for (int j = 0; j < 6; ++j) S.qd[j] = clampf(S.qd[j] + dqd[j], -P.vmax, P.vmax);
}

// ---- joint-limit rows: the packed ten-row solver ------------------------------------------------------------------
// Round-2 candidate for the joint-limit instantiations: instead of diverting robots with an active limit row to the
// scalar slow path above, every robot solves a ten-row system - one slot per limited joint (left hip, left knee, right
// hip, right knee; a joint cannot sit at both bounds) and the six contact rows - with the rows that do not exist zeroed,
// so that a warp stays converged. Rows pair across the legs like the contact rows:
//   pair 0 (nL, nR)  pair 1 (t1L, t1R)  pair 2 (t2L, t2R)  pair 3 (hipL, hipR)  pair 4 (kneeL, kneeR)
// Bullet's order within a sweep is: limit rows (in joint order hipL kneeL hipR kneeR on odd sweeps, reversed on even
// ones), then nL nR, then t1L t2L t1R t2R. The Delassus matrix uses the same telescoped form as the contact rows, which
// holds for any generalized impulse: a joint impulse enters the up-pass as u_k at its own level instead of a wheel force.
UPKIE_HD constexpr int pair_of_row10(int row) {  // rows: 0 hipL, 1 kneeL, 2 hipR, 3 kneeR, 4 nL, 5 nR, 6 t1L, 7 t2L, 8 t1R, 9 t2R
  return row == 0 || row == 2 ? 3 : row == 1 || row == 3 ? 4 : row == 4 || row == 5 ? 0 : row == 6 || row == 8 ? 1 : 2;
}
UPKIE_HD constexpr int lane_of_row10(int row) { return (row == 2 || row == 3 || row == 5 || row == 8 || row == 9) ? 1 : 0; }
UPKIE_HD constexpr int row10_of(int pair, int lane) {
  return pair == 3 ? 2 * lane : pair == 4 ? 1 + 2 * lane : pair == 0 ? 4 + lane : pair == 1 ? 6 + 2 * lane : 7 + 2 * lane;
}

// up-pass of a pair of generalized impulses: wheel forces f (or null) plus joint impulses at the hips (gh) and knees (gk)
UPKIE_HD void legs_impulse_up_general(const SimParams& P, const LegCache2& lc, const f2* f, f2 gh, f2 gk, f2 uu[3],
                                      f2 nptop[6]) {
  f2 q[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) q[i] = f ? f[i] : bc2(0.f);
#pragma unroll
  for (int k = 2; k >= 0; --k) {
    f2 u = sdot2(P.sgn2[k], lc.ox[k], lc.oz[k], q);  // zero above the level a joint impulse enters at
    if (k == 1) u = add2(u, gk);
    if (k == 0) u = add2(u, gh);
    uu[k] = u;
    const f2 nud = mul2(u, neg2(lc.invD[k]));
#pragma unroll
    for (int i = 0; i < 6; ++i) q[i] = fma2(lc.U[k][i], nud, q[i]);
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) nptop[i] = q[i];
}

// Two rewrites that cut ~280 instructions per substep out of this function - closed-form up-passes for the joint-limit
// directions, the Delassus matrix stored as paired columns and scaled in place - were measured slower: they lengthen
// live ranges in a kernel that already spills, and ptxas' schedule matters more than the instruction count here.
template <typename AnyFn, typename SyncFn>
UPKIE_HD void contact_solve_ten_rows(const SimParams& P, RobotState& S, const LegCache2& lc, const float IA0[21],
                                     const float R[9], const float zb[3], float inv_n,
                                     const f2 Pc[3], const f2& dist, bool actL, bool actR, float mu, AnyFn warp_any,
                                     SyncFn phase_sync) {
  // limit slots: dir = +1 at the lower bound, -1 at the upper one, 0 when the joint is inside its range
  f2 dirH, dirK, penH, penK;
  {
    float d[4], pn[4];
    const int js[4] = {0, 1, 3, 4};
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int j = js[a];
      const float lo = S.q[j] - P.q_lower[j], hi = P.q_upper[j] - S.q[j];
      d[a] = lo <= 0.f ? 1.f : (hi <= 0.f ? -1.f : 0.f);
      pn[a] = lo <= 0.f ? lo : (hi <= 0.f ? hi : 0.f);
    }
    dirH = mk2(d[0], d[2]); dirK = mk2(d[1], d[3]);
    penH = mk2(pn[0], pn[2]); penK = mk2(pn[1], pn[3]);
  }
  const bool any_limit = dirH.x != 0.f || dirH.y != 0.f || dirK.x != 0.f || dirK.y != 0.f;
  if (!warp_any(actL || actR || any_limit)) {
    S.lam_n[0] = 0.f;
    S.lam_n[1] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) S.lam_t[k] = 0.f;
    phase_sync();  // 3
    phase_sync();  // 4
    phase_sync();  // 5
    phase_sync();  // 6
    return;
  }
  const float t1[3] = {zb[2] * inv_n, 0.f, -zb[0] * inv_n};
  float t2[3];
  cross3(zb, t1, t2);
  const f2 sw = P.sgn2[2];
  f2 J[3][6];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    f2 dir[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) dir[i] = d == 0 ? bc2(zb[i]) : mul2(sw, bc2(d == 1 ? t1[i] : t2[i]));
    cross3_2(Pc, dir, &J[d][0]);
    J[d][3] = dir[0]; J[d][4] = dir[1]; J[d][5] = dir[2];
  }
  f2 Vw[6];
  {
    float Vb[6];
    rot_tmul(R, S.angvel, &Vb[0]);
    rot_tmul(R, S.linvel, &Vb[3]);
#pragma unroll
    for (int i = 0; i < 6; ++i) Vw[i] = bc2(Vb[i]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const f2 w = mul2(P.sgn2[k], mk2(S.qd[k], S.qd[k + 3]));
      Vw[1] = add2(Vw[1], w);
      Vw[3] = fma2(neg2(lc.oz[k]), w, Vw[3]);
      Vw[5] = fma2(lc.ox[k], w, Vw[5]);
    }
  }
  // Delassus matrix over the five direction pairs (normal, t1, t2, hip, knee)
  float W[10][10];
  {
    f2 uu_[5][3], pt_[5][6];
#pragma unroll
    for (int d = 0; d < 5; ++d) {
      if (d < 3) legs_impulse_up_general(P, lc, J[d], bc2(0.f), bc2(0.f), uu_[d], pt_[d]);
      else legs_impulse_up_general(P, lc, nullptr, d == 3 ? dirH : bc2(0.f), d == 4 ? dirK : bc2(0.f), uu_[d], pt_[d]);
      f2 da0[6];
#pragma unroll
      for (int i = 0; i < 6; ++i) da0[i] = pt_[d][i];
      ldl6_solve2(IA0, da0);
#pragma unroll
      for (int e = 0; e <= d; ++e) {
        f2 wo = bc2(0.f), wc = bc2(0.f);
#pragma unroll
        for (int k = 0; k < 3; ++k) wo = fma2(mul2(uu_[e][k], lc.invD[k]), uu_[d][k], wo);
#pragma unroll
        for (int i = 0; i < 6; ++i) {
          wo = fma2(pt_[e][i], da0[i], wo);
          wc = fma2(swp2(pt_[e][i]), da0[i], wc);
        }
        W[row10_of(e, 0)][row10_of(d, 0)] = wo.x;
        W[row10_of(e, 1)][row10_of(d, 1)] = wo.y;
        W[row10_of(e, 1)][row10_of(d, 0)] = wc.x;
        W[row10_of(e, 0)][row10_of(d, 1)] = wc.y;
        if (e != d) {
          W[row10_of(d, 0)][row10_of(e, 0)] = wo.x;
          W[row10_of(d, 1)][row10_of(e, 1)] = wo.y;
          W[row10_of(d, 0)][row10_of(e, 1)] = wc.x;
          W[row10_of(d, 1)][row10_of(e, 0)] = wc.y;
        }
      }
      if (d < 3) phase_sync();  // 3, 4, 5
    }
  }
  float rhs[10], jdi[10], lam[10];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    f2 rel = bc2(0.f);
#pragma unroll
    for (int i = 0; i < 6; ++i) rel = fma2(J[d][i], Vw[i], rel);
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      const int k = row10_of(d, side);
      const float r = side == 0 ? rel.x : rel.y;
      lam[k] = d == 0 ? ((side == 0 ? actL : actR) ? P.warm * S.lam_n[side] : 0.f) : 0.f;
      if (d == 0) {
        const float pen = side == 0 ? dist.x : dist.y;
        jdi[k] = 1.f / (W[k][k] + P.cfm);
        float pos_err = 0.f, vel_err = -r;
        if (pen > 0.f) vel_err -= pen * P.inv_h;
        else pos_err = -pen * P.erp * P.inv_h;
        rhs[k] = (pos_err + vel_err) * jdi[k];
      } else {
        jdi[k] = W[k][k] > 0.f ? 1.f / W[k][k] : 0.f;
        rhs[k] = -r * jdi[k];
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {  // limit rows 0 hipL, 1 kneeL, 2 hipR, 3 kneeR
    const int j = a == 0 ? 0 : a == 1 ? 1 : a == 2 ? 3 : 4;
    const float dir = a == 0 ? dirH.x : a == 1 ? dirK.x : a == 2 ? dirH.y : dirK.y;
    const float pen = a == 0 ? penH.x : a == 1 ? penK.x : a == 2 ? penH.y : penK.y;
    lam[a] = 0.f;
    jdi[a] = W[a][a] > 1.1920929e-7f ? 1.f / W[a][a] : 0.f;
    rhs[a] = (-pen * P.limit_erp * P.inv_h - dir * S.qd[j]) * jdi[a];
  }
  const float cfmrow = P.cfm;
  float dinv[10];  // 1 / jacDiagABInv per row: impulse change -> velocity change (Bullet's residual, see pgs_solve())
#pragma unroll
  for (int k = 0; k < 10; ++k) dinv[k] = W[k][k] + ((k == 4 || k == 5) ? P.cfm : 0.f);
  f2 Gc[10][5];
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    float g[10];
#pragma unroll
    for (int m = 0; m < 10; ++m)
      g[m] = -jdi[m] * W[m][k] + (m == k ? 1.f - ((k == 4 || k == 5) ? cfmrow * jdi[k] : 0.f) : 0.f);
#pragma unroll
    for (int p = 0; p < 5; ++p) Gc[k][p] = mk2(g[row10_of(p, 0)], g[row10_of(p, 1)]);
  }
  if (!actL) {
    rhs[4] = 0.f;
#pragma unroll
    for (int k = 0; k < 10; ++k) Gc[k][0].x = 0.f;
  }
  if (!actR) {
    rhs[5] = 0.f;
#pragma unroll
    for (int k = 0; k < 10; ++k) Gc[k][0].y = 0.f;
  }
  f2 r2[5];
#pragma unroll
  for (int p = 0; p < 5; ++p) r2[p] = mk2(rhs[row10_of(p, 0)], rhs[row10_of(p, 1)]);
#pragma unroll
  for (int l = 4; l < 6; ++l)  // warm-started normals
#pragma unroll
    for (int p = 0; p < 5; ++p) r2[p] = fma2(Gc[l][p], bc2(lam[l]), r2[p]);
  bool frozen = false;  // this lane has met Bullet's residual threshold: its updates are no-ops from here on
  auto update = [&](int k, float& res) {
    const f2 rp = r2[pair_of_row10(k)];
    const float rk = lane_of_row10(k) == 0 ? rp.x : rp.y;
    float nl;
    if (k < 4) {
      nl = fminf(fmaxf(rk, 0.f), P.limit_max_impulse);
    } else if (k < 6) {
      nl = fmaxf(rk, 0.f);
    } else {
      const float hi = mu * lam[(k < 8) ? 4 : 5];
      nl = fminf(fmaxf(rk, -hi), hi);
    }
    if (frozen) nl = lam[k];
    const float delta = nl - lam[k];
    const f2 d2 = bc2(delta);
#pragma unroll
    for (int p = 0; p < 5; ++p) r2[p] = fma2(Gc[k][p], d2, r2[p]);
    res = fmaxf(res, fabsf(delta) * dinv[k]);
    lam[k] = nl;
  };
  auto sweep = [&](bool forward) -> float {
    float res = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) update(forward ? a : 3 - a, res);
#pragma unroll
    for (int k = 4; k < 10; ++k) update(k, res);
    return res;
  };
  // two sweeps per trip, each followed by the per-lane residual test (the lane freezes exactly where Bullet would stop);
  // the warp votes once per trip - at most one no-op sweep more than needed, half the votes and branches
  auto after_sweep = [&](float res, int it) {
    const bool was_frozen = frozen;
    frozen = frozen || (res * res <= P.res_thr);
#ifdef UPKIE_PGS_STATS
    if (frozen && !was_frozen) upkie_pgs_stats(100 + it + 1);
    else if (!frozen && it + 1 == P.pgs_iterations) upkie_pgs_stats(100 + it + 1);
#else
    (void)was_frozen;
    (void)it;
#endif
  };
#ifndef UPKIE_SWEEPS_PER_TRIP
#define UPKIE_SWEEPS_PER_TRIP 2  // sweeps between two warp votes on the exit test
#endif
  for (int it = 0; it < P.pgs_iterations; it += UPKIE_SWEEPS_PER_TRIP) {
    after_sweep(sweep(false), it);  // even iteration: the non-contact rows are walked backwards
    if (it + 1 < P.pgs_iterations) after_sweep(sweep(true), it + 1);
#if UPKIE_SWEEPS_PER_TRIP == 4
    if (it + 2 < P.pgs_iterations) after_sweep(sweep(false), it + 2);
    if (it + 3 < P.pgs_iterations) after_sweep(sweep(true), it + 3);
#endif
    if (!warp_any(!frozen)) break;
  }
  S.lam_n[0] = lam[4];
  S.lam_n[1] = lam[5];
#pragma unroll
  for (int k = 0; k < 4; ++k) S.lam_t[k] = lam[6 + k];
  f2 F[6];
  {
    // F = sum_d lam_d J_d = (Pc x w, w) with w the wheels' total impulse: J itself need not outlive the Delassus matrix
    const f2 ln = mk2(lam[4], lam[5]), l1 = mk2(lam[6], lam[8]), l2 = mk2(lam[7], lam[9]);
    f2 w[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) w[i] = fma2(ln, bc2(zb[i]), mul2(sw, fma2(l1, bc2(t1[i]), mul2(l2, bc2(t2[i])))));
    cross3_2(Pc, w, &F[0]);
    F[3] = w[0]; F[4] = w[1]; F[5] = w[2];
  }
  f2 u[3], nptop[6];
  legs_impulse_up_general(P, lc, F, mul2(dirH, mk2(lam[0], lam[2])), mul2(dirK, mk2(lam[1], lam[3])), u, nptop);
  float da0[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) da0[i] = nptop[i].x + nptop[i].y;
  ldl6_solve(IA0, da0);
  f2 da2[6], aw[6], dq[3];
#pragma unroll
  for (int i = 0; i < 6; ++i) da2[i] = bc2(da0[i]);
  legs_impulse_down<false>(P, lc, u, da2, aw, dq);
  float dw[3], dv[3];
  rot_mul(R, &da0[0], dw);
  rot_mul(R, &da0[3], dv);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    S.angvel[i] = clampf(S.angvel[i] + dw[i], -P.vmax, P.vmax);
    S.linvel[i] = clampf(S.linvel[i] + dv[i], -P.vmax, P.vmax);
    S.qd[i] = clampf(S.qd[i] + dq[i].x, -P.vmax, P.vmax);
    S.qd[3 + i] = clampf(S.qd[3 + i] + dq[i].y, -P.vmax, P.vmax);
  }
  phase_sync();  // 6
}

// ---- body-ground contacts: gate and general solver ------------------------------------------------------------------
// Bullet collides every link that has a <collision> shape with plane.urdf (pybullet_backend.py:115,121,306), so a
// fallen robot rests on its torso. Here the shapes are reduced to collision points (UpkieModel.collision_*); while one
// of them is closer to the ground than the breaking threshold it holds a normal row and two friction rows. That is rare
// on the workloads the kernels are tuned for (the envs terminate on a fall), and the row count is open-ended, so such
// robots do not go through the packed solvers: once per substep a warp asks whether ANY of its robots has a collision
// point near the ground (body_points_near_ground: a dozen FMAs), and only then solves ALL rows of its robots - joint
// limits, tires, body points - in general_contact_solve(): scalar, looped, local-memory arrays, compiled as a real
// function (not inlined) so that its stack frame and registers stay out of the kernels' fast path.
// Restated from Bullet 3.24 (third-party, absent from the reference tree: parity unpinned): rigid contact for links
// without <contact> stiffness (cfm 0, erp = m_erp2), friction directions btPlaneSpace1(normal), at most four manifold
// points per pair, rows ordered limits / normals / frictions as in btMultiBodyConstraintSolver::solveSingleIteration.
// 0 in the step units whose kernel families have no body-contact rows (their SASS is what it was before the rows
// existed), 1 in those of the families with the `body` trait (step_family.h; launch_step checks it at compile time),
// in upkie_b200.cu (reset kernels) and in the host build
#ifndef UPKIE_BODY_CONTACTS_BUILD
#define UPKIE_BODY_CONTACTS_BUILD 1
#endif
#if defined(__CUDACC__)
#define UPKIE_NOINLINE __host__ __device__ __noinline__
#else
#define UPKIE_NOINLINE __attribute__((noinline))
#endif

// where the record of the last substep's body contacts goes (upkie_b200_get_body_contacts): element k at p[k * stride]
struct BodyRecOut {
  float* p;
  size_t stride;
};

// conservative per-robot test: exact for the points of the base body, through a bounding radius for the leg bodies
UPKIE_HD bool body_points_near_ground(const SimParams& P, float posz, const LegCache2& lc, const float zb[3]) {
  bool near = false;
#pragma unroll 1
  for (int p = 0; p < P.n_gate_base; ++p) {
    const float d = posz + zb[0] * P.gate_base[p][0] + zb[1] * P.gate_base[p][1] + zb[2] * P.gate_base[p][2] - P.gate_base[p][3];
    near = near || (d < P.breaking_threshold);
  }
  if (P.n_gate_base < P.n_bp) {  // collision points on leg bodies
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const f2 h = fma2(bc2(zb[0]), lc.ox[k], fma2(bc2(zb[1]), P.oy2[k], fma2(bc2(zb[2]), lc.oz[k], bc2(posz))));
      near = near || (h.x - P.gate_leg_bound[k].x < P.breaking_threshold) || (h.y - P.gate_leg_bound[k].y < P.breaking_threshold);
    }
  }
  return near;
}

struct BodySolveIO {
  // in
  float R[9];        // base -> world rotation
  float posz, inv_n, mu;
  float q[6];
  LegCache2 lc;
  float IA0[21];     // LDL^T factors of the base's articulated inertia (ldl6)
  f2 Pc[3], dist;    // tire contact points (base coordinates) and their distances to the ground
  int inL, inR;      // tire closer than the breaking threshold
  int limits;        // joint-limit rows on
  // in / out
  float angvel[3], linvel[3], qd[6];
  float lam_n[2];
  // out
  float lam_t[4];
  float rec[UPKIE_BODY_REC_DIM];
};

// Velocity change for spatial impulses fb[b] on the bodies (0 base, 1..3 left leg, 4..6 right leg; about the base
// origin, base coordinates) plus generalized impulses g[j] on the joint coordinates: ab[b] per body, dqd per joint.
UPKIE_HD void impulse_response_bodies(const SimParams& P, const LegCache2& lc, const float IA0[21], const float fb[7][6],
                                      const float g[6], float dqd[6], float ab[7][6]) {
  float u[6], da0[6];
  for (int i = 0; i < 6; ++i) da0[i] = fb[0][i];
  for (int leg = 0; leg < 2; ++leg) {
    float qv[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // q = -p
    for (int k = 2; k >= 0; --k) {
      const int b = 1 + 3 * leg + k;
      for (int i = 0; i < 6; ++i) qv[i] += fb[b][i];
      const float s = lane(P.sgn2[k], leg), ox = lane(lc.ox[k], leg), oz = lane(lc.oz[k], leg);
      const float uj = s * (qv[1] - oz * qv[3] + ox * qv[5]) + g[3 * leg + k];
      u[3 * leg + k] = uj;
      const float c = uj * lane(lc.invD[k], leg);
      for (int i = 0; i < 6; ++i) qv[i] -= lane(lc.U[k][i], leg) * c;
    }
    for (int i = 0; i < 6; ++i) da0[i] += qv[i];
  }
  ldl6_solve(IA0, da0);
  for (int i = 0; i < 6; ++i) ab[0][i] = da0[i];
  for (int leg = 0; leg < 2; ++leg) {
    float a[6];
    for (int i = 0; i < 6; ++i) a[i] = da0[i];
    for (int k = 0; k < 3; ++k) {
      float dot = 0.f;
      for (int i = 0; i < 6; ++i) dot += lane(lc.U[k][i], leg) * a[i];
      const float dd = (u[3 * leg + k] - dot) * lane(lc.invD[k], leg);
      dqd[3 * leg + k] = dd;
      const float w = lane(P.sgn2[k], leg) * dd;
      a[1] += w;
      a[3] -= lane(lc.oz[k], leg) * w;
      a[5] += lane(lc.ox[k], leg) * w;
      for (int i = 0; i < 6; ++i) ab[1 + 3 * leg + k][i] = a[i];
    }
  }
}

// All constraint rows of one robot: joint limits, tire contacts, body-point contacts. Updates the velocities, the tire
// impulses and the body-contact record of `io`.
static UPKIE_NOINLINE void general_contact_solve(const SimParams& P, BodySolveIO& io) {
  constexpr int kMaxRows = 10 + 3 * UPKIE_MAX_BODY_CONTACTS;
  const float* R = io.R;
  const float zb[3] = {R[6], R[7], R[8]};
  const LegCache2& lc = io.lc;
  // -- collision points below the breaking threshold, the deepest UPKIE_MAX_BODY_CONTACTS of them in index order
  int cand[UPKIE_MAX_COLLISION_POINTS];
  float cdist[UPKIE_MAX_COLLISION_POINTS], cpos[UPKIE_MAX_COLLISION_POINTS][3];
  int nc = 0;
  {
    float cphi[2][3], sphi[2][3];
    bool have_trig = false;
    for (int p = 0; p < P.n_bp; ++p) {
      const int b = P.bp_body[p];
      float pb[3];
      if (b == 0) {
        for (int i = 0; i < 3; ++i) pb[i] = P.bp_pos[p][i];
      } else {
        if (!have_trig) {
          for (int leg = 0; leg < 2; ++leg) {
            float phi = 0.f;
            for (int k = 0; k < 3; ++k) {
              phi += lane(P.sgn2[k], leg) * io.q[3 * leg + k];
              const float red = phi - 6.28318530718f * rintf(phi * 0.15915494309f);
              sphi[leg][k] = sinf(red);
              cphi[leg][k] = cosf(red);
            }
          }
          have_trig = true;
        }
        const int leg = (b - 1) / 3, k = (b - 1) % 3;
        const float c = cphi[leg][k], sn = sphi[leg][k];
        pb[0] = lane(lc.ox[k], leg) + c * P.bp_pos[p][0] + sn * P.bp_pos[p][2];
        pb[1] = lane(P.oy2[k], leg) + P.bp_pos[p][1];
        pb[2] = lane(lc.oz[k], leg) - sn * P.bp_pos[p][0] + c * P.bp_pos[p][2];
      }
      const float d = io.posz + zb[0] * pb[0] + zb[1] * pb[1] + zb[2] * pb[2] - P.bp_radius[p];
      if (d >= P.breaking_threshold) continue;
      cand[nc] = p;
      cdist[nc] = d;
      for (int i = 0; i < 3; ++i) cpos[nc][i] = pb[i] - P.bp_radius[p] * zb[i];  // lowest point of the sphere
      ++nc;
    }
    while (nc > UPKIE_MAX_BODY_CONTACTS) {  // drop the shallowest (the later one on ties)
      int worst = 0;
      for (int c = 1; c < nc; ++c)
        if (cdist[c] >= cdist[worst]) worst = c;
      for (int c = worst; c + 1 < nc; ++c) {
        cand[c] = cand[c + 1];
        cdist[c] = cdist[c + 1];
        for (int i = 0; i < 3; ++i) cpos[c][i] = cpos[c + 1][i];
      }
      --nc;
    }
  }
  for (int k = 0; k < UPKIE_BODY_REC_DIM; ++k) io.rec[k] = 0.f;
  {
    unsigned mask = 0;
    for (int c = 0; c < nc; ++c) { mask |= 1u << cand[c]; io.rec[1 + 4 * c] = float(cand[c]); }
    io.rec[0] = float(mask);
  }

  // -- rows. kind 0 normal, 1 friction, 2 joint limit
  int kind[kMaxRows], body[kMaxRows], joint[kMaxRows], partner[kMaxRows], wheel[kMaxRows], slot[kMaxRows];
  float dirj[kMaxRows], pen[kMaxRows], J[kMaxRows][6];
  int n = 0;
  if (io.limits) {
    for (int j = 0; j < 6; ++j) {
      // wheels carry infinite bounds: both tests fail for them
      const float pen_lo = io.q[j] - P.q_lower[j], pen_hi = P.q_upper[j] - io.q[j];
      for (int sd = 0; sd < 2; ++sd) {
        const float pn = sd == 0 ? pen_lo : pen_hi;
        if (!(pn <= 0.f) || n >= 4) continue;
        kind[n] = 2; body[n] = -1; joint[n] = j; dirj[n] = sd == 0 ? 1.f : -1.f; pen[n] = pn; partner[n] = -1;
        wheel[n] = -1; slot[n] = -1;
        for (int i = 0; i < 6; ++i) J[n][i] = 0.f;
        ++n;
      }
    }
  }
  const int nlimit = n;
  const float t1[3] = {zb[2] * io.inv_n, 0.f, -zb[0] * io.inv_n};
  float t2[3];
  cross3(zb, t1, t2);
  const bool act[2] = {io.inL != 0, io.inR != 0};
  auto add_row = [&](int b, const float pc[3], const float dir[3], int knd, int prt, int wh, int sl, float pn) {
    cross3(pc, dir, &J[n][0]);
    J[n][3] = dir[0]; J[n][4] = dir[1]; J[n][5] = dir[2];
    kind[n] = knd; body[n] = b; joint[n] = -1; dirj[n] = 0.f; partner[n] = prt; wheel[n] = wh; slot[n] = sl; pen[n] = pn;
    return n++;
  };
  int normal_of_wheel[2] = {-1, -1}, normal_of_slot[UPKIE_MAX_BODY_CONTACTS];
  for (int sd = 0; sd < 2; ++sd)
    if (act[sd]) {
      const float pc[3] = {lane(io.Pc[0], sd), lane(io.Pc[1], sd), lane(io.Pc[2], sd)};
      normal_of_wheel[sd] = add_row(3 + 3 * sd, pc, zb, 0, -1, sd, -1, lane(io.dist, sd));
    }
  for (int c = 0; c < nc; ++c) normal_of_slot[c] = add_row(P.bp_body[cand[c]], cpos[c], zb, 0, -1, -1, c, cdist[c]);
  for (int sd = 0; sd < 2; ++sd)
    if (act[sd]) {
      const float sw = lane(P.sgn2[2], sd);
      const float pc[3] = {lane(io.Pc[0], sd), lane(io.Pc[1], sd), lane(io.Pc[2], sd)};
      const float d1[3] = {sw * t1[0], sw * t1[1], sw * t1[2]}, d2[3] = {sw * t2[0], sw * t2[1], sw * t2[2]};
      add_row(3 + 3 * sd, pc, d1, 1, normal_of_wheel[sd], sd, -1, 0.f);
      add_row(3 + 3 * sd, pc, d2, 1, normal_of_wheel[sd], sd, -1, 0.f);
    }
  {
    // btPlaneSpace1((0, 0, 1)) = (0, -1, 0), (1, 0, 0) in the world, here in base coordinates
    const float d1[3] = {-R[3], -R[4], -R[5]}, d2[3] = {R[0], R[1], R[2]};
    for (int c = 0; c < nc; ++c) {
      add_row(P.bp_body[cand[c]], cpos[c], d1, 1, normal_of_slot[c], -1, c, 0.f);
      add_row(P.bp_body[cand[c]], cpos[c], d2, 1, normal_of_slot[c], -1, c, 0.f);
    }
  }
  if (n == 0) {  // nothing to solve
    io.lam_n[0] = 0.f; io.lam_n[1] = 0.f;
    for (int k = 0; k < 4; ++k) io.lam_t[k] = 0.f;
    return;
  }

  // -- body spatial velocities at the predicted generalized velocity (about the base origin, base coordinates)
  float Vb[7][6];
  {
    rot_tmul(R, io.angvel, &Vb[0][0]);
    rot_tmul(R, io.linvel, &Vb[0][3]);
    for (int leg = 0; leg < 2; ++leg) {
      float v[6];
      for (int i = 0; i < 6; ++i) v[i] = Vb[0][i];
      for (int k = 0; k < 3; ++k) {
        const float w = lane(P.sgn2[k], leg) * io.qd[3 * leg + k];
        v[1] += w;
        v[3] -= lane(lc.oz[k], leg) * w;
        v[5] += lane(lc.ox[k], leg) * w;
        for (int i = 0; i < 6; ++i) Vb[1 + 3 * leg + k][i] = v[i];
      }
    }
  }
  // -- Delassus matrix, one response per row. Rows padded to a multiple of four columns (zeros) and 16 B aligned: the
  // row . impulse products of the sweeps below read them as 128-bit local-memory loads
  constexpr int kPad = (kMaxRows + 3) / 4 * 4;
  struct alignas(16) Quad { float x, y, z, w; };
  alignas(16) float W[kMaxRows][kPad];
  float fb[7][6], g[6], dqd[6], ab[7][6];
  for (int l = 0; l < n; ++l) {
    for (int b = 0; b < 7; ++b)
      for (int i = 0; i < 6; ++i) fb[b][i] = 0.f;
    for (int j = 0; j < 6; ++j) g[j] = 0.f;
    if (kind[l] == 2) g[joint[l]] = dirj[l];
    else for (int i = 0; i < 6; ++i) fb[body[l]][i] = J[l][i];
    impulse_response_bodies(P, lc, io.IA0, fb, g, dqd, ab);
    for (int k = 0; k < n; ++k) {
      float wkl;
      if (kind[k] == 2) {
        wkl = dirj[k] * dqd[joint[k]];
      } else {
        wkl = 0.f;
        for (int i = 0; i < 6; ++i) wkl += J[k][i] * ab[body[k]][i];
      }
      W[k][l] = wkl;
    }
  }
  float rhs[kMaxRows], jdi[kMaxRows], cfmrow[kMaxRows], dinv[kMaxRows];
  alignas(16) float lam[kPad];
  const int n4 = (n + 3) & ~3;
  for (int l = 0; l < kPad; ++l) lam[l] = 0.f;
  for (int k = 0; k < n; ++k)
    for (int l = n; l < n4; ++l) W[k][l] = 0.f;
  for (int k = 0; k < n; ++k) {
    lam[k] = 0.f;
    dinv[k] = W[k][k] + ((kind[k] == 0 && wheel[k] >= 0) ? P.cfm : 0.f);
    if (kind[k] == 2) {
      const float rel = dirj[k] * io.qd[joint[k]];
      jdi[k] = W[k][k] > 1.1920929e-7f ? 1.f / W[k][k] : 0.f;
      if (jdi[k] == 0.f) dinv[k] = 0.f;
      rhs[k] = (-pen[k] * P.limit_erp * P.inv_h - rel) * jdi[k];
      cfmrow[k] = 0.f;
      continue;
    }
    float rel = 0.f;
    for (int i = 0; i < 6; ++i) rel += J[k][i] * Vb[body[k]][i];
    if (kind[k] == 0) {
      // tires: soft contact from their <contact> stiffness / damping; other links: rigid (cfm 0, erp = m_erp2)
      const bool tire = wheel[k] >= 0;
      if (tire) lam[k] = P.warm * io.lam_n[wheel[k]];
      const float row_cfm = tire ? P.cfm : 0.f, row_erp = tire ? P.erp : P.body_erp;
      jdi[k] = 1.f / (W[k][k] + row_cfm);
      float pos_err = 0.f, vel_err = -rel;
      if (pen[k] > 0.f) vel_err -= pen[k] * P.inv_h;
      else pos_err = -pen[k] * row_erp * P.inv_h;
      rhs[k] = (pos_err + vel_err) * jdi[k];
      cfmrow[k] = row_cfm * jdi[k];
    } else {
      jdi[k] = W[k][k] > 0.f ? 1.f / W[k][k] : 0.f;
      rhs[k] = -rel * jdi[k];
      cfmrow[k] = 0.f;
    }
  }
  for (int it = 0; it < P.pgs_iterations; ++it) {
    float res = 0.f;  // largest velocity-level row change of the sweep (Bullet's residual, see pgs_solve())
    for (int pos = 0; pos < n; ++pos) {
      const int k = pos < nlimit ? ((it & 1) ? pos : nlimit - 1 - pos) : pos;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;  // four partial sums: no 22-deep dependent chain
      {
        const Quad* wr = reinterpret_cast<const Quad*>(W[k]);
        const Quad* lv = reinterpret_cast<const Quad*>(lam);
        for (int q = 0; q < n4 / 4; ++q) {
          const Quad w4 = wr[q], l4 = lv[q];
          a0 += w4.x * l4.x; a1 += w4.y * l4.y; a2 += w4.z * l4.z; a3 += w4.w * l4.w;
        }
      }
      const float jdv = (a0 + a1) + (a2 + a3);
      const float sum = lam[k] + (rhs[k] - lam[k] * cfmrow[k] - jdv * jdi[k]);
      float lo, hi;
      if (kind[k] == 0) { lo = 0.f; hi = 1e10f; }
      else if (kind[k] == 2) { lo = 0.f; hi = P.limit_max_impulse; }
      else { hi = io.mu * (wheel[k] >= 0 ? 1.f : P.body_mu_scale) * lam[partner[k]]; lo = -hi; }
      const float nl = fminf(fmaxf(sum, lo), hi);
      res = fmaxf(res, fabsf(nl - lam[k]) * dinv[k]);
      lam[k] = nl;
    }
    if (res * res <= P.res_thr) break;  // per robot
  }
  // -- apply the total impulse
  for (int b = 0; b < 7; ++b)
    for (int i = 0; i < 6; ++i) fb[b][i] = 0.f;
  for (int j = 0; j < 6; ++j) g[j] = 0.f;
  io.lam_n[0] = 0.f;
  io.lam_n[1] = 0.f;
  for (int k = 0; k < 4; ++k) io.lam_t[k] = 0.f;
  int nfric[2] = {0, 0}, nbf[UPKIE_MAX_BODY_CONTACTS] = {0, 0, 0, 0};
  for (int k = 0; k < n; ++k) {
    if (kind[k] == 2) {
      g[joint[k]] += dirj[k] * lam[k];
      continue;
    }
    for (int i = 0; i < 6; ++i) fb[body[k]][i] += J[k][i] * lam[k];
    if (wheel[k] >= 0) {
      if (kind[k] == 0) io.lam_n[wheel[k]] = lam[k];
      else io.lam_t[2 * wheel[k] + nfric[wheel[k]]++] = lam[k];  // rolling row first, then lateral
    } else {
      const int c = slot[k];
      if (kind[k] == 0) io.rec[1 + 4 * c + 1] = lam[k];
      else io.rec[1 + 4 * c + 2 + nbf[c]++] = lam[k];
    }
  }
  impulse_response_bodies(P, lc, io.IA0, fb, g, dqd, ab);
  float dw[3], dv[3];
  rot_mul(R, &ab[0][0], dw);
  rot_mul(R, &ab[0][3], dv);
  for (int i = 0; i < 3; ++i) {
    io.angvel[i] = clampf(io.angvel[i] + dw[i], -P.vmax, P.vmax);
    io.linvel[i] = clampf(io.linvel[i] + dv[i], -P.vmax, P.vmax);
  }
  for (int j = 0; j < 6; ++j) io.qd[j] = clampf(io.qd[j] + dqd[j], -P.vmax, P.vmax);
}

// row / column index of (side, direction) in Bullet's order: nL nR t1L t2L t1R t2R
UPKIE_HD constexpr int row_of(int side, int d) { return d == 0 ? side : 2 + 2 * side + (d - 1); }

template <typename AnyFn, typename SyncFn = NoSync>
UPKIE_HD void physics_substep_paired(const SimParams& P, RobotState& S, const float tau[6], const float* eps, float mu,
                                     AnyFn warp_any, SyncFn phase_sync = SyncFn(), const float* wext = nullptr,
                                     int limits = 0, bool locked = false, BodyRecOut rec = BodyRecOut{nullptr, 0}) {
  float R[9];
  quat_to_rot(S.quat, R);
  float V0[6];
  rot_tmul(R, S.angvel, &V0[0]);
  rot_tmul(R, S.linvel, &V0[3]);

  float IA0[21], pA0[6];
  base_inertia_bias(P, V0, IA0, pA0);
  LegCache2 lc;
  f2 cc[3][6], uu[3];
  legs_pass12(P, S.q, S.qd, tau, V0, eps, lc, cc, uu, IA0, pA0, locked);
  phase_sync();  // 1
  ldl6(IA0);
  float a0[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) a0[i] = wext ? wext[i] - pA0[i] : -pA0[i];
  ldl6_solve(IA0, a0);
  float qdd[6];
  legs_pass3(P, lc, cc, uu, a0, qdd);

  // gravity as a uniform frame acceleration, classical acceleration of the origin
  const float zb[3] = {R[6], R[7], R[8]};  // world z axis in base coordinates
  {
    float lin[3], wxv[3], dw[3], dv[3];
    cross3(&V0[0], &V0[3], wxv);
    lin[0] = a0[3] - P.gravity * zb[0] + wxv[0];
    lin[1] = a0[4] - P.gravity * zb[1] + wxv[1];
    lin[2] = a0[5] - P.gravity * zb[2] + wxv[2];
    rot_mul(R, &a0[0], dw);
    rot_mul(R, lin, dv);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      S.angvel[i] = clampf(S.angvel[i] + P.h * dw[i], -P.vmax, P.vmax);
      S.linvel[i] = clampf(S.linvel[i] + P.h * dv[i], -P.vmax, P.vmax);
    }
#pragma unroll
    for (int j = 0; j < 6; ++j) S.qd[j] = clampf(S.qd[j] + P.h * qdd[j], -P.vmax, P.vmax);
  }

  // -- collision detection: tire circle vs the plane z = 0 (base coordinates), both wheels
  const float nxz = sqrtf(zb[0] * zb[0] + zb[2] * zb[2]);
  const bool rim_ok = nxz > 1e-6f;
  const float inv_n = rim_ok ? 1.f / nxz : 0.f;
  const float dB0 = -zb[0] * inv_n * P.wheel_radius, dB2 = -zb[2] * inv_n * P.wheel_radius;
  const f2 Pc[3] = {add2(lc.ox[2], bc2(dB0)), P.oy2[2], add2(lc.oz[2], bc2(dB2))};
  const f2 dist = fma2(bc2(zb[0]), Pc[0], fma2(bc2(zb[1]), Pc[1], fma2(bc2(zb[2]), Pc[2], bc2(S.pos[2]))));
  const bool inL = rim_ok && (dist.x < P.breaking_threshold);
  const bool inR = rim_ok && (dist.y < P.breaking_threshold);
  S.contact = (inL || inR) ? 1.f : 0.f;
  // a robot with an active joint-limit row leaves the packed solver alone (its contact rows are switched off
  // there, which makes that solve a no-op for it) and solves all of its rows in limit_contact_solve() below
  LimitRows lim;
  lim.n = 0;
  // limits: 0 no joint-limit rows, 1 scalar slow path for the robots that have one, 2 packed ten-row solver for all
  // The scalar slow path exists in the HOST build only (the CPU test-suite's independent second implementation of the
  // limit rows): on the device the whole warp would wait for the lanes that take it, and its
  // dynamically indexed local arrays cost every FAM_LIMITS kernel a 2 KB stack frame. On the device 1 aliases to 3.
  // body-ground contacts: a warp that holds a robot with a collision point near the ground solves all rows of its
  // robots in general_contact_solve() instead of the packed solvers (warp-uniform choice)
  bool body_slow = false;
#if UPKIE_BODY_CONTACTS_BUILD
  if (limits != 0 && P.body_contacts) body_slow = warp_any(body_points_near_ground(P, S.pos[2], lc, zb));
#endif
#if defined(__CUDA_ARCH__)
  const bool slow = false;
  if (limits == 1) limits = 3;
#else
  const bool slow = !body_slow && limits == 1 && active_joint_limits(P, S.q, lim) > 0;
#endif
  const float lam_prev[2] = {S.lam_n[0], S.lam_n[1]};
  const bool actL = inL && !slow, actR = inR && !slow;
  phase_sync();  // 2

  // limits == 3: the ten-row solver only for warps that hold a robot on a bound (warp-uniform choice), the six-row
  // contact block otherwise: workloads that never reach a bound (position-controlled legs) keep the plain cost
  bool ten_rows = limits == 2;
  if (limits == 3 && !body_slow) {
    bool on_bound = false;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int j = a < 2 ? a : a + 1;
      on_bound = on_bound || (S.q[j] - P.q_lower[j] <= 0.f) || (P.q_upper[j] - S.q[j] <= 0.f);
    }
    ten_rows = warp_any(on_bound);
  }
#if UPKIE_BODY_CONTACTS_BUILD
  if (body_slow) {
    phase_sync();  // 3
    phase_sync();  // 4
    phase_sync();  // 5
    BodySolveIO io;
#pragma unroll
    for (int i = 0; i < 9; ++i) io.R[i] = R[i];
    io.posz = S.pos[2]; io.inv_n = inv_n; io.mu = mu;
#pragma unroll
    for (int j = 0; j < 6; ++j) { io.q[j] = S.q[j]; io.qd[j] = S.qd[j]; }
    io.lc = lc;
#pragma unroll
    for (int i = 0; i < 21; ++i) io.IA0[i] = IA0[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) { io.Pc[i] = Pc[i]; io.angvel[i] = S.angvel[i]; io.linvel[i] = S.linvel[i]; }
    io.dist = dist;
    io.inL = inL ? 1 : 0; io.inR = inR ? 1 : 0;
    io.limits = 1;
    io.lam_n[0] = S.lam_n[0]; io.lam_n[1] = S.lam_n[1];
    general_contact_solve(P, io);
#pragma unroll
    for (int i = 0; i < 3; ++i) { S.angvel[i] = io.angvel[i]; S.linvel[i] = io.linvel[i]; }
#pragma unroll
    for (int j = 0; j < 6; ++j) S.qd[j] = io.qd[j];
    S.lam_n[0] = io.lam_n[0]; S.lam_n[1] = io.lam_n[1];
#pragma unroll
    for (int k = 0; k < 4; ++k) S.lam_t[k] = io.lam_t[k];
    if (rec.p) {
#pragma unroll 1
      for (int k = 0; k < UPKIE_BODY_REC_DIM; ++k) rec.p[size_t(k) * rec.stride] = io.rec[k];
    }
    phase_sync();  // 6
  } else
#endif
  if (ten_rows) {
    contact_solve_ten_rows(P, S, lc, IA0, R, zb, inv_n, Pc, dist, inL, inR, mu, warp_any, phase_sync);
  } else if (!warp_any(actL || actR)) {
    S.lam_n[0] = 0.f;
    S.lam_n[1] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) S.lam_t[k] = 0.f;
    phase_sync();  // 3
    phase_sync();  // 4
    phase_sync();  // 5
    phase_sync();  // 6
  } else {
    // contact directions in base coordinates: d = 0 normal, 1 rolling (s * t1), 2 lateral (s * t2)
    const float t1[3] = {zb[2] * inv_n, 0.f, -zb[0] * inv_n};
    float t2[3];
    cross3(zb, t1, t2);
    const f2 sw = P.sgn2[2];
    // J rows as spatial forces about the base origin, (left wheel, right wheel)
    f2 J[3][6];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      f2 dir[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) dir[i] = d == 0 ? bc2(zb[i]) : mul2(sw, bc2(d == 1 ? t1[i] : t2[i]));
      cross3_2(Pc, dir, &J[d][0]);
      J[d][3] = dir[0]; J[d][4] = dir[1]; J[d][5] = dir[2];
    }
    // wheel spatial velocities at the predicted generalized velocity
    f2 Vw[6];
    {
      float Vb[6];
      rot_tmul(R, S.angvel, &Vb[0]);
      rot_tmul(R, S.linvel, &Vb[3]);
#pragma unroll
      for (int i = 0; i < 6; ++i) Vw[i] = bc2(Vb[i]);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const f2 w = mul2(P.sgn2[k], mk2(S.qd[k], S.qd[k + 3]));
        Vw[1] = add2(Vw[1], w);
        Vw[3] = fma2(neg2(lc.oz[k]), w, Vw[3]);
        Vw[5] = fma2(lc.ox[k], w, Vw[5]);
      }
    }
    // Delassus matrix W = J M^-1 J^T without walking back down the legs. With the up-pass quantities of a unit
    // impulse along direction d on a wheel (per-joint u_k(d), force left on the base ptop(d)) and the base
    // response a0(d) = -IA0^-1 ptop(d), the articulated-body recursions telescope to
    //   same wheel:   W[e][d] = sum_k u_k(e) u_k(d) / D_k - ptop(e) . a0(d)
    //   other wheel:  W[e][d] =                            - ptop_other(e) . a0(d)
    // (g_k = p_k(e)^T a_k(d) obeys g_k = g_{k-1} - u_k(e) u_k(d) / D_k). Three packed up-passes and three
    // two-right-hand-side base solves; W is symmetric, so each (e <= d) pair is computed once.
    float W[6][6];
    {
      f2 uu_[3][3], pt_[3][6];
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        legs_impulse_up(P, lc, J[d], uu_[d], pt_[d]);  // pt_ = -ptop
        f2 da0[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) da0[i] = pt_[d][i];
        ldl6_solve2(IA0, da0);  // a0(d) = -IA0^-1 ptop(d); lane x: left column, lane y: right column
#pragma unroll
        for (int e = 0; e <= d; ++e) {
          f2 wo = bc2(0.f), wc = bc2(0.f);
#pragma unroll
          for (int k = 0; k < 3; ++k) wo = fma2(mul2(uu_[e][k], lc.invD[k]), uu_[d][k], wo);
#pragma unroll
          for (int i = 0; i < 6; ++i) {
            wo = fma2(pt_[e][i], da0[i], wo);        // -ptop(e) . a0(d)
            wc = fma2(swp2(pt_[e][i]), da0[i], wc);  // -ptop_other(e) . a0(d)
          }
          W[row_of(0, e)][row_of(0, d)] = wo.x;
          W[row_of(1, e)][row_of(1, d)] = wo.y;
          W[row_of(1, e)][row_of(0, d)] = wc.x;  // right wheel row e, left wheel column d
          W[row_of(0, e)][row_of(1, d)] = wc.y;  // left wheel row e, right wheel column d
          if (e != d) {
            W[row_of(0, d)][row_of(0, e)] = wo.x;
            W[row_of(1, d)][row_of(1, e)] = wo.y;
            W[row_of(0, d)][row_of(1, e)] = wc.x;
            W[row_of(1, d)][row_of(0, e)] = wc.y;
          }
        }
        phase_sync();  // 3, 4, 5
      }
    }
    // right-hand sides (btMultiBodyConstraintSolver::setupMultiBodyContactConstraint)
    float rhs[6], jdi[6], lam[6];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      f2 rel = bc2(0.f);
#pragma unroll
      for (int i = 0; i < 6; ++i) rel = fma2(J[d][i], Vw[i], rel);
#pragma unroll
      for (int side = 0; side < 2; ++side) {
        const int k = row_of(side, d);
        const float r = side == 0 ? rel.x : rel.y;
        // warm start (Bullet SOLVER_USE_WARMSTARTING): normals from the previous substep, frictions from 0
        lam[k] = d == 0 ? ((side == 0 ? actL : actR) ? P.warm * S.lam_n[side] : 0.f) : 0.f;
        if (d == 0) {
          const float pen = side == 0 ? dist.x : dist.y;
          jdi[k] = 1.f / (W[k][k] + P.cfm);
          float pos_err = 0.f, vel_err = -r;
          if (pen > 0.f) vel_err -= pen * P.inv_h;
          else pos_err = -pen * P.erp * P.inv_h;
          rhs[k] = (pos_err + vel_err) * jdi[k];
        } else {
          jdi[k] = W[k][k] > 0.f ? 1.f / W[k][k] : 0.f;
          rhs[k] = -r * jdi[k];
        }
      }
    }
    const float cfmrow = P.cfm;  // m_cfm = cfm * jacDiagABInv
    // Projected Gauss-Seidel with Bullet's residual exit rule, see pgs_solve() (sim_core.cuh)
    float dinv[6];  // 1 / jacDiagABInv: turns an impulse change into the row's velocity change
#pragma unroll
    for (int k = 0; k < 6; ++k) dinv[k] = W[k][k] + (k < 2 ? P.cfm : 0.f);
    // residual-form sweep of pgs_solve() (sim_core.cuh) with the six residuals as three (left, right) pairs:
    // r2[0] = (nL, nR), r2[1] = (t1L, t1R), r2[2] = (t2L, t2R); column k of the scaled matrix in the same pairing
    f2 Gc[6][3];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      float g[6];
#pragma unroll
      for (int m = 0; m < 6; ++m) g[m] = -jdi[m] * W[m][k] + (m == k ? 1.f - (k < 2 ? cfmrow * jdi[k] : 0.f) : 0.f);
      Gc[k][0] = mk2(g[0], g[1]);
      Gc[k][1] = mk2(g[2], g[4]);
      Gc[k][2] = mk2(g[3], g[5]);
    }
    // a wheel out of contact: zero its normal row and right-hand side, so that its residual stays 0 and the
    // normal update is a single max(r, 0) (its friction bounds are then +-mu * 0)
    if (!actL) {
      rhs[0] = 0.f;
#pragma unroll
      for (int k = 0; k < 6; ++k) Gc[k][0].x = 0.f;
    }
    if (!actR) {
      rhs[1] = 0.f;
#pragma unroll
      for (int k = 0; k < 6; ++k) Gc[k][0].y = 0.f;
    }
    f2 r2[3] = {mk2(rhs[0], rhs[1]), mk2(rhs[2], rhs[4]), mk2(rhs[3], rhs[5])};
#pragma unroll
    for (int l = 0; l < 2; ++l)  // warm-started normals; frictions start from 0
#pragma unroll
      for (int p = 0; p < 3; ++p) r2[p] = fma2(Gc[l][p], bc2(lam[l]), r2[p]);
    // One sweep = six row updates in Bullet's order: clamp the row's residual, push the change into all six
    // residuals (three paired FMAs), keep the largest velocity-level change of the sweep. A lane whose sweep stayed at or
    // below Bullet's residual threshold is frozen (its later updates are no-ops) until the warp's last lane is done.
    bool frozen = false;
    auto sweep = [&]() -> float {
      float res = 0.f;
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        const float rk = k == 0 ? r2[0].x : k == 1 ? r2[0].y : k == 2 ? r2[1].x : k == 3 ? r2[2].x : k == 4 ? r2[1].y : r2[2].y;
        float nl;
        if (k < 2) {
          nl = fmaxf(rk, 0.f);
        } else {
          const float hi = mu * lam[(k < 4) ? 0 : 1];
          nl = fminf(fmaxf(rk, -hi), hi);
        }
        if (frozen) nl = lam[k];
        const float delta = nl - lam[k];
        const f2 d2 = bc2(delta);
#pragma unroll
        for (int p = 0; p < 3; ++p) r2[p] = fma2(Gc[k][p], d2, r2[p]);
        res = fmaxf(res, fabsf(delta) * dinv[k]);
        lam[k] = nl;
      }
      return res;
    };
    auto after_sweep = [&](float res, int it) {
      const bool was_frozen = frozen;
      frozen = frozen || (res * res <= P.res_thr);
#ifdef UPKIE_PGS_STATS
      if (frozen && !was_frozen) upkie_pgs_stats(it + 1);
      else if (!frozen && it + 1 == P.pgs_iterations) upkie_pgs_stats(it + 1);
#else
      (void)was_frozen;
      (void)it;
#endif
    };
    // two sweeps per trip, one warp vote (see contact_solve_ten_rows)
    for (int it = 0; it < P.pgs_iterations; it += 2) {
      after_sweep(sweep(), it);
      if (it + 1 < P.pgs_iterations) after_sweep(sweep(), it + 1);
      if (!warp_any(!frozen)) break;
    }
    S.lam_n[0] = lam[0];
    S.lam_n[1] = lam[1];
#pragma unroll
    for (int k = 0; k < 4; ++k) S.lam_t[k] = lam[2 + k];
    // apply the total wheel impulses: both wheels up their legs at once, one base solve, both legs down
    f2 F[6];
    {
      const f2 ln = mk2(lam[0], lam[1]), l1 = mk2(lam[2], lam[4]), l2 = mk2(lam[3], lam[5]);
      // F = (Pc x w, w) in the same order as contact_solve_ten_rows, which must give a robot without a limit row the
      // same bits as this solver
      f2 w[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) w[i] = fma2(ln, bc2(zb[i]), mul2(sw, fma2(l1, bc2(t1[i]), mul2(l2, bc2(t2[i])))));
      cross3_2(Pc, w, &F[0]);
      F[3] = w[0]; F[4] = w[1]; F[5] = w[2];
    }
    f2 u[3], nptop[6];
    legs_impulse_up(P, lc, F, u, nptop);
    float da0[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) da0[i] = nptop[i].x + nptop[i].y;
    ldl6_solve(IA0, da0);
    f2 da2[6], aw[6], dq[3];
#pragma unroll
    for (int i = 0; i < 6; ++i) da2[i] = bc2(da0[i]);
    legs_impulse_down<false>(P, lc, u, da2, aw, dq);
    float dw[3], dv[3];
    rot_mul(R, &da0[0], dw);
    rot_mul(R, &da0[3], dv);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      S.angvel[i] = clampf(S.angvel[i] + dw[i], -P.vmax, P.vmax);
      S.linvel[i] = clampf(S.linvel[i] + dv[i], -P.vmax, P.vmax);
      S.qd[i] = clampf(S.qd[i] + dq[i].x, -P.vmax, P.vmax);
      S.qd[3 + i] = clampf(S.qd[3 + i] + dq[i].y, -P.vmax, P.vmax);
    }
    phase_sync();  // 6
  }
#if !defined(__CUDA_ARCH__)
  if (slow) limit_contact_solve(P, S, lc, IA0, R, zb, inv_n, Pc, dist, inL, inR, mu, lim, lam_prev);
#else
  (void)lam_prev;
#endif
#if UPKIE_BODY_CONTACTS_BUILD
  if (rec.p && !body_slow) rec.p[0] = 0.f;  // no body contact held rows in this substep
#else
  (void)rec;
  (void)body_slow;
#endif

  // -- position integration with the new velocities (as physics_substep)
#pragma unroll
  for (int i = 0; i < 3; ++i) S.pos[i] += P.h * S.linvel[i];
  {
    // rotation increment exp(w h / 2): the even Taylor polynomials of sin(x) / x and cos(x) to degree 6, x = |w| h / 2.
    // make_sim_params bounds h * max_coordinate_velocity by 0.6, so x <= 0.52 and the truncation stays below 1.4e-7
    // (defaults, h = 1 ms and the clamp at 100: x <= 0.087, ~1e-14). Not sinf / cosf: under --use_fast_math they
    // carry an absolute error of up to 3.6e-7, as large as the increment itself at slow rates
    const float* om = S.angvel;
    const float hh = 0.5f * P.h;
    const float x2 = (om[0] * om[0] + om[1] * om[1] + om[2] * om[2]) * hh * hh;
    const float sc = hh * (1.f + x2 * (-1.f / 6.f + x2 * (1.f / 120.f - x2 * (1.f / 5040.f))));
    const float ax = om[0] * sc, ay = om[1] * sc, az = om[2] * sc;
    const float dqw = 1.f + x2 * (-0.5f + x2 * (1.f / 24.f - x2 * (1.f / 720.f)));
    const float qw = S.quat[0], qx = S.quat[1], qy = S.quat[2], qz = S.quat[3];
    const float nw = dqw * qw - ax * qx - ay * qy - az * qz;
    const float nx = dqw * qx + ax * qw + ay * qz - az * qy;
    const float ny = dqw * qy - ax * qz + ay * qw + az * qx;
    const float nz = dqw * qz + ax * qy - ay * qx + az * qw;
    const float inv = 1.f / sqrtf(nw * nw + nx * nx + ny * ny + nz * nz);
    S.quat[0] = nw * inv; S.quat[1] = nx * inv; S.quat[2] = ny * inv; S.quat[3] = nz * inv;
  }
#pragma unroll
  for (int j = 0; j < 6; ++j) S.q[j] += P.h * S.qd[j];
}

}  // namespace upkie_b200
