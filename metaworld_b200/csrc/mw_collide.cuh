// Narrowphase for the step kernel.
//
// Conventions follow the reference physics (MuJoCo mj_collision [3P], reached from
// metaworld/sawyer_xyz_env.py:595,620): geom1 has the lower type id, the normal points from
// geom1 to geom2, dist < 0 is penetration, pos is the midpoint between the two surfaces.
//
// * analytic pairs (plane-*, sphere/capsule pairs, sphere-box, capsule-box, box-box) are
//   evaluated ONE PAIR PER LANE;
// * general convex pairs (cylinder-*, mesh-*) run GJK + EPA with lane 0 as the leader that owns
//   the simplex / polytope (kept in the warp's shared-memory workspace) while every support
//   query is evaluated by the whole warp (mesh hull vertices are split across lanes).
#pragma once
#include "mw_math.cuh"

#ifndef MW_WARP
#define MW_WARP 32          // lanes cooperating on one environment (1 only in the host emulation used by tests/)
#endif

enum { G_PLANE = 0, G_HFIELD, G_SPHERE, G_CAPSULE, G_ELLIPSOID, G_CYLINDER, G_BOX, G_MESH };

struct RawCon { creal dist, pos[3], normal[3]; };

struct DShape {   // pos / mat point at the geom's world pose (shared memory in the kernel): nothing is copied into the thread's stack
  int type; const creal* pos; const creal* mat; creal size[3]; const float4* vert; int nvert;   // hull vertices packed xyz_ (16-byte loads)
};

// ------------------------------------------------------------------ plane pairs
DEV int plane_sphere_raw(const creal* pn, const creal* pp, const creal* c, creal r, creal margin, RawCon* o) {
  creal t[3]; v3sub(t, c, pp);
  creal dist = v3dot(t, pn) - r;
  if (dist > margin) return 0;
  o->dist = dist; v3copy(o->normal, pn);
  v3addscl(o->pos, c, pn, -(r + (creal)0.5 * dist));
  return 1;
}
DEV int plane_capsule(const DShape& a, const DShape& b, creal margin, RawCon* o) {
  creal n[3], ax[3], c[3]; mat_col(n, a.mat, 2); mat_col(ax, b.mat, 2);
  int cnt = 0;
  v3addscl(c, b.pos, ax, b.size[1]); cnt += plane_sphere_raw(n, a.pos, c, b.size[0], margin, o + cnt);
  v3addscl(c, b.pos, ax, -b.size[1]); cnt += plane_sphere_raw(n, a.pos, c, b.size[0], margin, o + cnt);
  return cnt;
}
DEV int plane_cylinder(const DShape& a, const DShape& b, creal margin, RawCon* o) {
  creal n[3], axis[3], vec[3], t[3];
  mat_col(n, a.mat, 2); mat_col(axis, b.mat, 2);
  v3sub(t, b.pos, a.pos);
  creal dist0 = v3dot(t, n), prjaxis = v3dot(n, axis);
  if (prjaxis > 0) { v3scl(axis, axis, -1); prjaxis = -prjaxis; }
  for (int i = 0; i < 3; i++) vec[i] = prjaxis * axis[i] - n[i];
  creal len = v3norm(vec);
  if (len >= (creal)1e-12) v3scl(vec, vec, b.size[0] / len);
  else { mat_col(vec, b.mat, 0); v3scl(vec, vec, b.size[0]); }
  creal prjvec = v3dot(vec, n);
  v3scl(axis, axis, b.size[1]); prjaxis *= b.size[1];
  int cnt = 0;
  if (dist0 + prjaxis + prjvec > margin) return 0;
  creal dd = dist0 + prjaxis + prjvec;
  o[cnt].dist = dd; v3copy(o[cnt].normal, n);
  for (int i = 0; i < 3; i++) o[cnt].pos[i] = b.pos[i] + vec[i] + axis[i] - n[i] * dd * (creal)0.5;
  cnt++;
  if (dist0 - prjaxis + prjvec <= margin) {
    dd = dist0 - prjaxis + prjvec;
    o[cnt].dist = dd; v3copy(o[cnt].normal, n);
    for (int i = 0; i < 3; i++) o[cnt].pos[i] = b.pos[i] + vec[i] - axis[i] - n[i] * dd * (creal)0.5;
    cnt++;
  }
  creal prjvec1 = -prjvec * (creal)0.5;
  if (dist0 + prjaxis + prjvec1 <= margin) {
    creal vec1[3]; v3cross(vec1, vec, axis); v3normalize(vec1); v3scl(vec1, vec1, b.size[0] * (creal)0.8660254037844386);
    dd = dist0 + prjaxis + prjvec1;
    for (int s = -1; s <= 1; s += 2) {
      o[cnt].dist = dd; v3copy(o[cnt].normal, n);
      for (int i = 0; i < 3; i++) o[cnt].pos[i] = b.pos[i] + s * vec1[i] + axis[i] - vec[i] * (creal)0.5 - n[i] * dd * (creal)0.5;
      cnt++;
    }
  }
  return cnt;
}
DEV int plane_box(const DShape& a, const DShape& b, creal margin, RawCon* o) {
  creal n[3], t[3]; mat_col(n, a.mat, 2); v3sub(t, b.pos, a.pos);
  creal dist = v3dot(t, n);
  int cnt = 0;
  for (int i = 0; i < 8 && cnt < 4; i++) {
    creal v[3] = {(i & 1 ? 1 : -1) * b.size[0], (i & 2 ? 1 : -1) * b.size[1], (i & 4 ? 1 : -1) * b.size[2]}, c[3];
    mat_mulvec(c, b.mat, v);
    creal ld = v3dot(n, c);
    if (dist + ld > margin) continue;
    o[cnt].dist = dist + ld; v3copy(o[cnt].normal, n);
    for (int k = 0; k < 3; k++) o[cnt].pos[k] = b.pos[k] + c[k] - n[k] * o[cnt].dist * (creal)0.5;
    cnt++;
  }
  return cnt;
}

// ------------------------------------------------------------------ sphere / capsule pairs
DEV int sphere_sphere_raw(const creal* c1, creal r1, const creal* c2, creal r2, creal margin, RawCon* o) {
  creal dif[3]; v3sub(dif, c2, c1);
  creal len = v3norm(dif), dist = len - r1 - r2;
  if (dist > margin) return 0;
  if (len < eps_<creal>()) { dif[0] = 1; dif[1] = dif[2] = 0; } else v3scl(dif, dif, 1 / len);
  o->dist = dist; v3copy(o->normal, dif);
  v3addscl(o->pos, c1, dif, r1 + (creal)0.5 * dist);
  return 1;
}
DEV int sphere_capsule(const DShape& a, const DShape& b, creal margin, RawCon* o) {
  creal ax[3], t[3], c[3]; mat_col(ax, b.mat, 2); v3sub(t, a.pos, b.pos);
  creal x = v3dot(t, ax);
  x = fmin(fmax(x, -b.size[1]), b.size[1]);
  v3addscl(c, b.pos, ax, x);
  return sphere_sphere_raw(a.pos, a.size[0], c, b.size[0], margin, o);
}
DEV int capsule_capsule(const DShape& a, const DShape& b, creal margin, RawCon* o) {
  creal a1[3], a2[3], dif[3]; mat_col(a1, a.mat, 2); mat_col(a2, b.mat, 2); v3sub(dif, a.pos, b.pos);
  creal h1 = a.size[1], h2 = b.size[1];
  creal ma = v3dot(a1, a1), mb = -v3dot(a1, a2), mc = v3dot(a2, a2), u = -v3dot(a1, dif), v = v3dot(a2, dif);
  creal det = ma * mc - mb * mb;
  if (fabs(det) >= (creal)1e-12) {
    creal x1 = (mc * u - mb * v) / det, x2 = (ma * v - mb * u) / det;
    if (x1 > h1) { x1 = h1; x2 = (v - mb * h1) / mc; } else if (x1 < -h1) { x1 = -h1; x2 = (v + mb * h1) / mc; }
    if (x2 > h2) { x2 = h2; x1 = fmin(fmax((u - mb * h2) / ma, -h1), h1); }
    else if (x2 < -h2) { x2 = -h2; x1 = fmin(fmax((u + mb * h2) / ma, -h1), h1); }
    creal p1[3], p2[3]; v3addscl(p1, a.pos, a1, x1); v3addscl(p2, b.pos, a2, x2);
    return sphere_sphere_raw(p1, a.size[0], p2, b.size[0], margin, o);
  }
  int cnt = 0;
  for (int k = 0; k < 2; k++) {
    creal p1[3], p2[3], t[3]; v3addscl(p1, a.pos, a1, k ? -h1 : h1); v3sub(t, p1, b.pos);
    creal x2 = fmin(fmax(v3dot(t, a2), -h2), h2);
    v3addscl(p2, b.pos, a2, x2);
    cnt += sphere_sphere_raw(p1, a.size[0], p2, b.size[0], margin, o + cnt);
  }
  return cnt;
}
DEV int sphere_box_raw(const creal* c, creal r, const DShape& b, creal margin, RawCon* o) {
  creal t[3], cl[3], clamped[3]; v3sub(t, c, b.pos); mat_tmulvec(cl, b.mat, t);
  bool inside = true;
  for (int i = 0; i < 3; i++) {
    clamped[i] = cl[i];
    if (clamped[i] > b.size[i]) { clamped[i] = b.size[i]; inside = false; }
    else if (clamped[i] < -b.size[i]) { clamped[i] = -b.size[i]; inside = false; }
  }
  creal nl[3], dist, pl[3];
  if (!inside) {
    v3sub(nl, clamped, cl);
    creal len = v3normalize(nl);
    dist = len - r;
    if (dist > margin) return 0;
    v3addscl(pl, cl, nl, r + (creal)0.5 * dist);
  } else {
    int k = 0; creal best = (creal)1e30, sgn = 1;
    for (int i = 0; i < 3; i++) {
      creal dpos = b.size[i] - cl[i], dneg = b.size[i] + cl[i];
      if (dpos < best) { best = dpos; k = i; sgn = 1; }
      if (dneg < best) { best = dneg; k = i; sgn = -1; }
    }
    v3zero(nl); nl[k] = -sgn;
    dist = -(best + r);
    v3copy(pl, cl); pl[k] = cl[k] + sgn * (creal)0.5 * (best - r);
  }
  o->dist = dist;
  mat_mulvec(o->normal, b.mat, nl);
  mat_mulvec(o->pos, b.mat, pl); v3add(o->pos, o->pos, b.pos);
  return 1;
}
// minimiser interval of dist^2(p0 + t*dir, box) over t in [0,1]; exact piecewise-quadratic scan
DEV creal seg_box_min(const creal* p0, const creal* dir, const creal* size, creal* tlo, creal* thi) {
  creal bp[16]; int nb = 0;
  bp[nb++] = 0; bp[nb++] = 1;
  for (int i = 0; i < 3; i++)
    if (fabs(dir[i]) > (creal)1e-14)
      for (int s = -1; s <= 1; s += 2) { creal t = (s * size[i] - p0[i]) / dir[i]; if (t > 0 && t < 1) bp[nb++] = t; }
  for (int i = 1; i < nb; i++) { creal x = bp[i]; int j = i - 1; while (j >= 0 && bp[j] > x) { bp[j + 1] = bp[j]; j--; } bp[j + 1] = x; }
  creal best = (creal)1e30, blo = 0, bhi = 0;
  for (int k = 0; k + 1 < nb; k++) {
    creal t0 = bp[k], t1 = bp[k + 1], tm = (creal)0.5 * (t0 + t1);
    creal A = 0, B = 0, C = 0;
    for (int i = 0; i < 3; i++) {
      creal x = p0[i] + tm * dir[i];
      if (x > size[i] || x < -size[i]) { creal aa = p0[i] + (x > size[i] ? -size[i] : size[i]), bb = dir[i]; A += bb * bb; B += 2 * aa * bb; C += aa * aa; }
    }
    creal tl, th, f;
    creal f0 = A * t0 * t0 + B * t0 + C, f1 = A * t1 * t1 + B * t1 + C;
    creal ts = A > 0 ? fmin(fmax(-B / (2 * A), t0), t1) : t0;
    f = A * ts * ts + B * ts + C;
    if (f0 < 0) f0 = 0; if (f1 < 0) f1 = 0; if (f < 0) f = 0;   // a squared distance: clear negative round-off
    const creal rel = (creal)1e-9;
    if (fmax(f0, f1) - f <= rel * f + (creal)1e-18) { tl = t0; th = t1; f = fmin(fmin(f0, f1), f); }   // flat: segment parallel to the face
    else { tl = th = ts; }
    creal tol = rel * best + (creal)1e-18;
    if (f < best - tol) { best = f; blo = tl; bhi = th; }
    else if (fabs(f - best) <= tol && tl <= bhi + (creal)1e-12) { if (th > bhi) bhi = th; }
  }
  *tlo = blo; *thi = bhi;
  return best;
}
DEV int capsule_box(const DShape& a, const DShape& b, creal margin, RawCon* o) {
  creal ax[3], t[3], p0[3], p1[3], l0[3], l1[3], dir[3];
  mat_col(ax, a.mat, 2);
  v3addscl(p0, a.pos, ax, -a.size[1]); v3addscl(p1, a.pos, ax, a.size[1]);
  v3sub(t, p0, b.pos); mat_tmulvec(l0, b.mat, t);
  v3sub(t, p1, b.pos); mat_tmulvec(l1, b.mat, t);
  v3sub(dir, l1, l0);
  creal tlo, thi;
  const creal best = seg_box_min(l0, dir, b.size, &tlo, &thi);
  int cnt = 0; creal c[3];
  if (best <= (creal)1e-18) {
    // The capsule axis passes through the box: distance zero along [tlo, thi], witness direction undefined.  Rule shared
    // with the oracle: the box face of minimum depth at the interval midpoint is the contact face for both interval ends.
    creal cm[3]; const creal tm = (creal)0.5 * (tlo + thi);
    for (int i = 0; i < 3; i++) cm[i] = l0[i] + tm * dir[i];
    int k = 0; creal bd = (creal)1e300, sgn = 1;
    for (int i = 0; i < 3; i++) {
      creal dpos = b.size[i] - cm[i], dneg = b.size[i] + cm[i];
      if (dpos < bd) { bd = dpos; k = i; sgn = 1; }
      if (dneg < bd) { bd = dneg; k = i; sgn = -1; }
    }
    const int nend = thi - tlo > (creal)1e-9 ? 2 : 1;
    for (int e = 0; e < nend; e++) {
      const creal te = e ? thi : tlo; creal ce[3], nl[3] = {0, 0, 0}, pl[3];
      for (int i = 0; i < 3; i++) ce[i] = l0[i] + te * dir[i];
      creal depth = b.size[k] - sgn * ce[k]; if (depth < 0) depth = 0;
      nl[k] = -sgn;
      v3copy(pl, ce); pl[k] = ce[k] + sgn * (creal)0.5 * (depth - a.size[0]);
      RawCon* r = o + cnt++;
      r->dist = -(depth + a.size[0]);
      mat_mulvec(r->normal, b.mat, nl);
      mat_mulvec(r->pos, b.mat, pl); v3add(r->pos, r->pos, b.pos);
    }
    return cnt;
  }
  v3addscl(c, p0, ax, 2 * a.size[1] * tlo); cnt += sphere_box_raw(c, a.size[0], b, margin, o + cnt);
  if (thi - tlo > (creal)1e-9) { v3addscl(c, p0, ax, 2 * a.size[1] * thi); cnt += sphere_box_raw(c, a.size[0], b, margin, o + cnt); }
  return cnt;
}

// ------------------------------------------------------------------ box-box: separating axes + face clipping
DEV int clip_poly(creal* poly, int n, int axis, creal lim, creal sgn) {
  creal out[32]; int m = 0;
  for (int i = 0; i < n; i++) {
    const creal* p = poly + 2 * i; const creal* q = poly + 2 * ((i + 1) % n);
    creal dp = sgn * p[axis] - lim, dq = sgn * q[axis] - lim;
    if (dp <= 0) { out[2 * m] = p[0]; out[2 * m + 1] = p[1]; m++; }
    if ((dp < 0 && dq > 0) || (dp > 0 && dq < 0)) {
      creal s = dp / (dp - dq);
      out[2 * m] = p[0] + s * (q[0] - p[0]); out[2 * m + 1] = p[1] + s * (q[1] - p[1]); m++;
    }
    if (m >= 15) break;
  }
  for (int i = 0; i < 2 * m; i++) poly[i] = out[i];
  return m;
}
__device__ __noinline__ int box_box(const DShape& a, const DShape& b, creal margin, RawCon* o) {
  const creal* R1 = a.mat; const creal* R2 = b.mat;
  creal p[3], pp[3]; v3sub(p, b.pos, a.pos); mat_tmulvec(pp, R1, p);
  creal R[9], Q[9];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    creal c1[3], c2[3]; mat_col(c1, R1, i); mat_col(c2, R2, j);
    R[3 * i + j] = v3dot(c1, c2); Q[3 * i + j] = fabs(R[3 * i + j]);
  }
  const creal* A = a.size; const creal* B = b.size;
  creal s = (creal)-1e30; int code = 0; bool invert = false, haveC = false; creal normalC[3] = {0, 0, 0};
  for (int i = 0; i < 3; i++) {
    creal e = fabs(pp[i]) - (A[i] + B[0] * Q[3 * i] + B[1] * Q[3 * i + 1] + B[2] * Q[3 * i + 2]);
    if (e > margin) return 0;
    if (e > s) { s = e; code = i + 1; invert = pp[i] < 0; haveC = false; }
  }
  for (int j = 0; j < 3; j++) {
    creal c2[3]; mat_col(c2, R2, j);
    creal e1 = v3dot(c2, p);
    creal e = fabs(e1) - (A[0] * Q[j] + A[1] * Q[3 + j] + A[2] * Q[6 + j] + B[j]);
    if (e > margin) return 0;
    if (e > s) { s = e; code = j + 4; invert = e1 < 0; haveC = false; }
  }
  const creal fudge = (creal)1.05;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
    int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    creal n[3] = {0, 0, 0};
    n[i1] = -R[3 * i2 + j]; n[i2] = R[3 * i1 + j];
    creal l = sqrt(n[i1] * n[i1] + n[i2] * n[i2]);
    if (l < (creal)1e-8) continue;
    creal e1 = pp[i2] * R[3 * i1 + j] - pp[i1] * R[3 * i2 + j];
    creal e = fabs(e1) - (A[i1] * Q[3 * i2 + j] + A[i2] * Q[3 * i1 + j] + B[j1] * Q[3 * i + j2] + B[j2] * Q[3 * i + j1]);
    e /= l;
    if (e > margin) return 0;
    if ((e < 0 ? e * fudge : e) > s) {
      s = e; code = 7 + 3 * i + j; invert = e1 < 0; haveC = true;
      normalC[0] = n[0] / l; normalC[1] = n[1] / l; normalC[2] = n[2] / l;
    }
  }
  if (!code) return 0;
  creal normal[3];
  if (haveC) mat_mulvec(normal, R1, normalC);
  else if (code <= 3) mat_col(normal, R1, code - 1);
  else mat_col(normal, R2, code - 4);
  if (invert) v3scl(normal, normal, -1);
  creal depth = -s;
  if (code > 6) {
    creal pa[3], pb[3]; v3copy(pa, a.pos); v3copy(pb, b.pos);
    for (int j = 0; j < 3; j++) {
      creal c1[3], c2[3]; mat_col(c1, R1, j); mat_col(c2, R2, j);
      creal sg = v3dot(normal, c1) > 0 ? (creal)1 : (creal)-1; v3addscl(pa, pa, c1, sg * A[j]);
      sg = v3dot(normal, c2) > 0 ? (creal)-1 : (creal)1; v3addscl(pb, pb, c2, sg * B[j]);
    }
    int ia = (code - 7) / 3, ib = (code - 7) % 3;
    creal ua[3], ub[3]; mat_col(ua, R1, ia); mat_col(ub, R2, ib);
    creal d[3]; v3sub(d, pb, pa);
    creal uaub = v3dot(ua, ub), q1 = v3dot(ua, d), q2 = -v3dot(ub, d), dd = 1 - uaub * uaub;
    creal alpha = 0, beta = 0;
    if (dd > (creal)1e-4) { alpha = (q1 + uaub * q2) / dd; beta = (uaub * q1 + q2) / dd; }
    v3addscl(pa, pa, ua, alpha); v3addscl(pb, pb, ub, beta);
    o->dist = -depth; v3copy(o->normal, normal);
    for (int k = 0; k < 3; k++) o->pos[k] = (creal)0.5 * (pa[k] + pb[k]);
    return 1;
  }
  const creal *Ra, *Rb, *pa, *pb, *Sa, *Sb; creal nrm[3];
  if (code <= 3) { Ra = R1; Rb = R2; pa = a.pos; pb = b.pos; Sa = A; Sb = B; v3copy(nrm, normal); }
  else { Ra = R2; Rb = R1; pa = b.pos; pb = a.pos; Sa = B; Sb = A; v3scl(nrm, normal, -1); }
  creal nr[3], anr[3]; mat_tmulvec(nr, Rb, nrm);
  for (int k = 0; k < 3; k++) anr[k] = fabs(nr[k]);
  int lanr, a1, a2;
  if (anr[1] > anr[0]) { if (anr[1] > anr[2]) { a1 = 0; lanr = 1; a2 = 2; } else { a1 = 0; a2 = 1; lanr = 2; } }
  else { if (anr[0] > anr[2]) { lanr = 0; a1 = 1; a2 = 2; } else { a1 = 0; a2 = 1; lanr = 2; } }
  creal center[3], col[3]; mat_col(col, Rb, lanr);
  creal sg = nr[lanr] < 0 ? (creal)1 : (creal)-1;
  for (int k = 0; k < 3; k++) center[k] = pb[k] - pa[k] + sg * Sb[lanr] * col[k];
  int codeN = (code <= 3 ? code - 1 : code - 4), code1, code2;
  if (codeN == 0) { code1 = 1; code2 = 2; } else if (codeN == 1) { code1 = 0; code2 = 2; } else { code1 = 0; code2 = 1; }
  creal r1[3], r2[3], i1v[3], i2v[3];
  mat_col(r1, Ra, code1); mat_col(r2, Ra, code2); mat_col(i1v, Rb, a1); mat_col(i2v, Rb, a2);
  creal c1 = v3dot(center, r1), c2 = v3dot(center, r2);
  creal m11 = v3dot(r1, i1v), m12 = v3dot(r1, i2v), m21 = v3dot(r2, i1v), m22 = v3dot(r2, i2v);
  creal k1 = m11 * Sb[a1], k2 = m21 * Sb[a1], k3 = m12 * Sb[a2], k4 = m22 * Sb[a2];
  creal quad[32];
  quad[0] = c1 - k1 - k3; quad[1] = c2 - k2 - k4; quad[2] = c1 - k1 + k3; quad[3] = c2 - k2 + k4;
  quad[4] = c1 + k1 + k3; quad[5] = c2 + k2 + k4; quad[6] = c1 + k1 - k3; quad[7] = c2 + k2 - k4;
  int n = 4;
  n = clip_poly(quad, n, 0, Sa[code1], 1); if (n) n = clip_poly(quad, n, 0, Sa[code1], -1);
  if (n) n = clip_poly(quad, n, 1, Sa[code2], 1); if (n) n = clip_poly(quad, n, 1, Sa[code2], -1);
  if (n < 1) return 0;
  creal det1 = 1 / (m11 * m22 - m12 * m21);
  m11 *= det1; m12 *= det1; m21 *= det1; m22 *= det1;
  int cnt = 0;
  for (int j = 0; j < n && cnt < 8; j++) {
    creal kk1 = m22 * (quad[2 * j] - c1) - m12 * (quad[2 * j + 1] - c2);
    creal kk2 = -m21 * (quad[2 * j] - c1) + m11 * (quad[2 * j + 1] - c2);
    creal pt[3];
    for (int k = 0; k < 3; k++) pt[k] = center[k] + kk1 * i1v[k] + kk2 * i2v[k];
    creal dep = Sa[codeN] - v3dot(nrm, pt);
    if (dep < -margin) continue;
    creal cp[3];
    for (int k = 0; k < 3; k++) cp[k] = pt[k] + pa[k] + (creal)0.5 * dep * nrm[k];
    bool dup = false;
    for (int q = 0; q < cnt; q++) { creal dx[3]; v3sub(dx, o[q].pos, cp); if (v3dot(dx, dx) < (creal)1e-16) dup = true; }
    if (dup) continue;
    o[cnt].dist = -dep; v3copy(o[cnt].normal, normal); v3copy(o[cnt].pos, cp);
    cnt++;
  }
  return cnt;
}

// one analytic pair on the calling lane; returns #contacts (<= 8)
DEV int narrow_analytic(const DShape& a, const DShape& b, creal margin, RawCon* o) {
  int t1 = a.type, t2 = b.type;
  if (t1 == G_PLANE) {
    creal n[3]; mat_col(n, a.mat, 2);
    if (t2 == G_SPHERE) return plane_sphere_raw(n, a.pos, b.pos, b.size[0], margin, o);
    if (t2 == G_CAPSULE) return plane_capsule(a, b, margin, o);
    if (t2 == G_CYLINDER) return plane_cylinder(a, b, margin, o);
    if (t2 == G_BOX) return plane_box(a, b, margin, o);
    return 0;
  }
  if (t1 == G_SPHERE && t2 == G_SPHERE) return sphere_sphere_raw(a.pos, a.size[0], b.pos, b.size[0], margin, o);
  if (t1 == G_SPHERE && t2 == G_CAPSULE) return sphere_capsule(a, b, margin, o);
  if (t1 == G_SPHERE && t2 == G_BOX) return sphere_box_raw(a.pos, a.size[0], b, margin, o);
  if (t1 == G_CAPSULE && t2 == G_CAPSULE) return capsule_capsule(a, b, margin, o);
  if (t1 == G_CAPSULE && t2 == G_BOX) return capsule_box(a, b, margin, o);
  if (t1 == G_BOX && t2 == G_BOX) return box_box(a, b, margin, o);
  return 0;
}
DEV bool pair_is_analytic(int t1, int t2) {
  if (t1 == G_PLANE) return t2 != G_MESH;
  if (t1 == G_SPHERE) return t2 == G_SPHERE || t2 == G_CAPSULE || t2 == G_BOX;
  if (t1 == G_CAPSULE) return t2 == G_CAPSULE || t2 == G_BOX;
  return t1 == G_BOX && t2 == G_BOX;
}

// ------------------------------------------------------------------ general convex: GJK + EPA, warp-cooperative
struct SV { creal v[3], a[3], b[3]; };

// support point of one shape for a world direction; evaluated by the whole warp (uniform result)
DEV void support_shape(const DShape& s, const creal* dir, creal* out, int lane) {
  creal dl[3], l[3];
  mat_tmulvec(dl, s.mat, dir);
  if (s.type == G_MESH) {
    creal bv = (creal)-1e30; int bi = 0;
    int i = lane;
    for (; i + 3 * MW_WARP < s.nvert; i += 4 * MW_WARP) {     // four independent 16-byte loads in flight per lane
      const float4 p0 = __ldg(s.vert + i), p1 = __ldg(s.vert + i + MW_WARP), p2 = __ldg(s.vert + i + 2 * MW_WARP), p3 = __ldg(s.vert + i + 3 * MW_WARP);
      const creal x0 = dl[0] * p0.x + dl[1] * p0.y + dl[2] * p0.z, x1 = dl[0] * p1.x + dl[1] * p1.y + dl[2] * p1.z;
      const creal x2 = dl[0] * p2.x + dl[1] * p2.y + dl[2] * p2.z, x3 = dl[0] * p3.x + dl[1] * p3.y + dl[2] * p3.z;
      if (x0 > bv) { bv = x0; bi = i; }
      if (x1 > bv) { bv = x1; bi = i + MW_WARP; }
      if (x2 > bv) { bv = x2; bi = i + 2 * MW_WARP; }
      if (x3 > bv) { bv = x3; bi = i + 3 * MW_WARP; }
    }
    for (; i < s.nvert; i += MW_WARP) {
      const float4 p = __ldg(s.vert + i);
      const creal x = dl[0] * p.x + dl[1] * p.y + dl[2] * p.z;
      if (x > bv) { bv = x; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      creal ov = __shfl_xor_sync(FULLMASK, bv, o); int oi = __shfl_xor_sync(FULLMASK, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    { const float4 p = __ldg(s.vert + bi); l[0] = p.x; l[1] = p.y; l[2] = p.z; }
  } else if (s.type == G_BOX) {
    for (int i = 0; i < 3; i++) l[i] = dl[i] >= 0 ? s.size[i] : -s.size[i];
  } else if (s.type == G_CYLINDER) {
    creal n = sqrt(dl[0] * dl[0] + dl[1] * dl[1]);
    if (n > eps_<creal>()) { l[0] = dl[0] * s.size[0] / n; l[1] = dl[1] * s.size[0] / n; } else l[0] = l[1] = 0;
    l[2] = dl[2] >= 0 ? s.size[1] : -s.size[1];
  } else if (s.type == G_CAPSULE) {
    l[0] = l[1] = 0; l[2] = dl[2] >= 0 ? s.size[1] : -s.size[1];
  } else {
    l[0] = l[1] = l[2] = 0;
  }
  mat_mulvec(out, s.mat, l); v3add(out, out, s.pos);
}
DEV creal core_radius(const DShape& s) { return (s.type == G_SPHERE || s.type == G_CAPSULE) ? s.size[0] : (creal)0; }
DEV void support_pair(const DShape& A, const DShape& B, const creal* dir, SV* o, int lane) {
  creal nd[3] = {-dir[0], -dir[1], -dir[2]};
  support_shape(A, dir, o->a, lane);
  support_shape(B, nd, o->b, lane);
  v3sub(o->v, o->a, o->b);
}
// Separating-axis hint of a general convex pair: one float4 per (env, pair) in global memory, xyz = a direction from A
// towards B along which the pair was last proven apart, w = what convex_pair last concluded (below).  Bodies move about
// a millimetre per substep, so an axis that separated a pair in one pass nearly always still does in the next.
#define SEP_APART 1.f        // the last decisive "no contact" came with a separating direction
#define SEP_HIT 2.f          // the last result was a contact: do not spend a support query on the hint
// Returns 1 when the hint proves the pair apart by more than margin + 1e-4, 0 when it does not, -1 when there is no usable
// hint.  Whole warp, uniform result.  The test is GJK's own separating-axis exit, with the same slack: along a unit
// direction n, min over A - B of -n.x = -n.(support_A(n) - support_B(-n)) is a lower bound on the distance between the
// cores, for ANY direction.  GJK's upper bound fdcore never falls below the true distance (apart from rounding at the 1e-12
// level), so whenever this test rejects, GJK would either have left by its separating-axis test or skipped the contact at
// `dist <= margin + 1e-4` in convex_pair: hit = 0 and no RawCon either way.  A stale, zero or garbage hint can therefore
// only fail to reject, and nothing that is computed depends on the table's contents.
DEV int sep_hint_test(const DShape& A, const DShape& B, creal margin, const float4* hint, int lane) {
  const float4 h = *hint;                                 // one address for the whole warp: a broadcast load
  if (h.w != SEP_APART) return -1;
  creal n[3] = {h.x, h.y, h.z};
  const creal nn = v3dot(n, n);
  if (!(nn > (creal)1e-30 && nn < (creal)1e30)) return -1;   // zero or non-finite (NaN fails both comparisons)
  v3scl(n, n, 1 / sqrt(nn));
  SV w; support_pair(A, B, n, &w, lane);
  return -v3dot(n, w.v) - core_radius(A) - core_radius(B) > margin + (creal)1e-4 ? 1 : 0;
}
DEV void sep_hint_store(float4* hint, const creal* n, float flag) { *hint = float4{(float)n[0], (float)n[1], (float)n[2], flag}; }
DEV void closest_tri(const creal* a, const creal* b, const creal* c, creal* w) {
  creal ab[3], ac[3], ap[3]; v3sub(ab, b, a); v3sub(ac, c, a); v3scl(ap, a, -1);
  creal d1 = v3dot(ab, ap), d2 = v3dot(ac, ap);
  if (d1 <= 0 && d2 <= 0) { w[0] = 1; w[1] = w[2] = 0; return; }
  creal bp[3]; v3scl(bp, b, -1);
  creal d3 = v3dot(ab, bp), d4 = v3dot(ac, bp);
  if (d3 >= 0 && d4 <= d3) { w[1] = 1; w[0] = w[2] = 0; return; }
  creal vc = d1 * d4 - d3 * d2;
  if (vc <= 0 && d1 >= 0 && d3 <= 0) { creal v = d1 / (d1 - d3); w[0] = 1 - v; w[1] = v; w[2] = 0; return; }
  creal cp[3]; v3scl(cp, c, -1);
  creal d5 = v3dot(ab, cp), d6 = v3dot(ac, cp);
  if (d6 >= 0 && d5 <= d6) { w[2] = 1; w[0] = w[1] = 0; return; }
  creal vb = d5 * d2 - d1 * d6;
  if (vb <= 0 && d2 >= 0 && d6 <= 0) { creal x = d2 / (d2 - d6); w[0] = 1 - x; w[1] = 0; w[2] = x; return; }
  creal va = d3 * d6 - d5 * d4;
  if (va <= 0 && (d4 - d3) >= 0 && (d5 - d6) >= 0) { creal x = (d4 - d3) / ((d4 - d3) + (d5 - d6)); w[0] = 0; w[1] = 1 - x; w[2] = x; return; }
  creal den = 1 / (va + vb + vc);
  w[1] = vb * den; w[2] = vc * den; w[0] = 1 - w[1] - w[2];
}
// simplex reduction (leader lane only). returns true if the origin is enclosed by a tetrahedron
// Whole warp calls this (the simplex lives in shared memory); *n and v are meaningful on lane 0.  The four faces of a
// tetrahedron are examined by four lanes at once; the winner is the face with the smallest distance, lowest index on
// ties -- the same choice as a serial scan.
__device__ __noinline__ bool closest_simplex(SV* s, int* n, creal* v, int lane) {
  creal w[4] = {0, 0, 0, 0};
  const int nn = __shfl_sync(FULLMASK, *n, 0);
  if (nn == 4) {
    const int F[4][4] = {{0, 1, 2, 3}, {0, 2, 3, 1}, {0, 3, 1, 2}, {1, 3, 2, 0}};
    creal best = (creal)1e30; int bf = 4; creal btw[3] = {0, 0, 0};
    for (int f = lane; f < 4; f += MW_WARP) {
      const creal *a = s[F[f][0]].v, *b = s[F[f][1]].v, *c = s[F[f][2]].v, *dv = s[F[f][3]].v;
      creal ab[3], ac[3], nrm[3], ad[3]; v3sub(ab, b, a); v3sub(ac, c, a); v3cross(nrm, ab, ac); v3sub(ad, dv, a);
      creal sd = v3dot(nrm, ad), so = -v3dot(nrm, a);
      if (fabs(sd) < (creal)1e-300) { so = 1; sd = -1; }
      if ((sd > 0 && so > 0) || (sd < 0 && so < 0)) continue;
      creal tw[3]; closest_tri(a, b, c, tw);
      creal q[3]; for (int k = 0; k < 3; k++) q[k] = tw[0] * a[k] + tw[1] * b[k] + tw[2] * c[k];
      creal dd = v3dot(q, q);
      if (dd < best) { best = dd; bf = f; btw[0] = tw[0]; btw[1] = tw[1]; btw[2] = tw[2]; }
    }
#pragma unroll
    for (int x = 2; x > 0; x >>= 1) {
      const creal ob = __shfl_xor_sync(FULLMASK, best, x); const int of = __shfl_xor_sync(FULLMASK, bf, x);
      const creal o0 = __shfl_xor_sync(FULLMASK, btw[0], x), o1 = __shfl_xor_sync(FULLMASK, btw[1], x), o2 = __shfl_xor_sync(FULLMASK, btw[2], x);
      if (of < 4 && (bf >= 4 || ob < best || (ob == best && of < bf))) { best = ob; bf = of; btw[0] = o0; btw[1] = o1; btw[2] = o2; }
    }
    if (bf >= 4) { if (lane == 0) v3zero(v); return true; }     // no face sees the origin: enclosed
    w[F[bf][0]] = btw[0]; w[F[bf][1]] = btw[1]; w[F[bf][2]] = btw[2];
  } else if (lane == 0) {
    if (nn == 1) w[0] = 1;
    else if (nn == 2) {
      creal ab[3]; v3sub(ab, s[1].v, s[0].v);
      creal t = -v3dot(s[0].v, ab) / fmax(v3dot(ab, ab), (creal)1e-300);
      if (t <= 0) w[0] = 1; else if (t >= 1) w[1] = 1; else { w[0] = 1 - t; w[1] = t; }
    } else closest_tri(s[0].v, s[1].v, s[2].v, w);
  }
  if (lane == 0) {
    int m = 0; v3zero(v);
    for (int i = 0; i < nn; i++) if (w[i] > 0) { for (int k = 0; k < 3; k++) v[k] += w[i] * s[i].v[k]; if (m != i) s[m] = s[i]; m++; }
    *n = m;
  }
  return false;
}
DEV void simplex_weights(const SV* s, int n, creal* w) {
  w[0] = 1; w[1] = w[2] = 0;
  if (n == 2) {
    creal ab[3]; v3sub(ab, s[1].v, s[0].v);
    creal t = fmin(fmax(-v3dot(s[0].v, ab) / fmax(v3dot(ab, ab), (creal)1e-300), (creal)0), (creal)1);
    w[0] = 1 - t; w[1] = t;
  } else if (n == 3) closest_tri(s[0].v, s[1].v, s[2].v, w);
}

// EPA polytope storage.  Hot per-face scalars and the vertex positions live in the warp's shared-memory scratch (EpaSm,
// overlaid on the region that later holds the constraint Jacobian); face normals and the per-vertex witness points live
// in a per-warp global-memory block (EpaWs).  Limits and tolerance follow MuJoCo's mjOption defaults for convex
// collision (ccd_iterations 50, ccd_tolerance 1e-6) [3P].
#define EPA_MAXV 64
#define EPA_MAXF 320
#define EPA_MAXE 96
#define EPA_ITERS 50
#define EPA_TOL ((creal)1e-6)
#define GJK_TOL ((creal)1e-8)   // absolute gap between the GJK upper and lower distance bounds
struct EpaSm {
  creal fd[EPA_MAXF];            // face plane offsets
  creal vv[EPA_MAXV][3];         // Minkowski-difference vertices
  short fv[3][EPA_MAXF];         // face vertex ids
  short vis[EPA_MAXF];           // faces visible from the new vertex (ascending)
  short hz[EPA_MAXE][2];         // horizon edges (ascending (face, edge) order)
  unsigned char alive[EPA_MAXF];
};
struct EpaWs { creal fn[3][EPA_MAXF]; creal va[EPA_MAXV][3], vb[EPA_MAXV][3]; };

// plane of triangle (a,b,c) oriented away from the origin; stores face f
DEV void epa_set_face(EpaSm* E, EpaWs* W, int f, int a, int b, int c) {
  creal ab[3], ac[3], nn[3], d; v3sub(ab, E->vv[b], E->vv[a]); v3sub(ac, E->vv[c], E->vv[a]); v3cross(nn, ab, ac);
  creal l = v3norm(nn);
  if (l < (creal)1e-300) { d = 0; nn[0] = 1; nn[1] = nn[2] = 0; }
  else { v3scl(nn, nn, 1 / l); d = v3dot(nn, E->vv[a]); }
  if (d < 0) { int t = b; b = c; c = t; v3scl(nn, nn, -1); d = -d; }
  E->fv[0][f] = (short)a; E->fv[1][f] = (short)b; E->fv[2][f] = (short)c; E->alive[f] = 1; E->fd[f] = d;
  W->fn[0][f] = nn[0]; W->fn[1][f] = nn[1]; W->fn[2][f] = nn[2];
}

// Face-on contact between a cylinder and a box face (cap-on-face or generator-line-on-face): every point of the
// contact patch is a valid EPA witness, so the contact *point* is implementation-defined in the reference physics.
// We take the pressure centroid of the patch under a linear penetration profile, clipped to the overlap with the
// box face (continuous in the pose; removes rim-to-rim chatter of resting cylinders).  Other configurations are
// left as EPA/GJK produced them.
__device__ __noinline__ void refine_cyl_box(const DShape& A, const DShape& B, RawCon* o) {
  if (A.type != G_CYLINDER || B.type != G_BOX) return;
  creal nb[3]; mat_tmulvec(nb, B.mat, o->normal);
  int k = 0; for (int q = 1; q < 3; q++) if (fabs(nb[q]) > fabs(nb[k])) k = q;
  if (fabs(nb[k]) < (creal)0.99999) return;                       /* the contact normal must be a face normal of the box */
  const creal sgn = nb[k] > 0 ? (creal)1 : (creal)-1;
  const int i = (k + 1) % 3, j = (k + 2) % 3;
  const creal r = A.size[0], h = A.size[1];
  creal ax[3], a[3], t[3], cB[3];
  mat_col(ax, A.mat, 2); mat_tmulvec(a, B.mat, ax);
  v3sub(t, A.pos, B.pos); mat_tmulvec(cB, B.mat, t);
  const creal ak = a[k] * sgn;
  creal P[3], pen;
  if (fabs(ak) > (creal)0.9) {
    /* ---- cap on face */
    const creal cs = ak > 0 ? (creal)1 : (creal)-1;
    creal C[3], acap[3], g[3];
    for (int q = 0; q < 3; q++) { acap[q] = cs * a[q]; C[q] = cB[q] + cs * h * a[q]; }
    const creal pen0 = sgn * C[k] + B.size[k];
    for (int q = 0; q < 3; q++) g[q] = -(sgn * acap[k]) * acap[q];
    g[k] += sgn;
    const creal st = v3norm(g);                                   /* sin(tilt) */
    creal sbar = 0;
    if (st > (creal)1e-9) sbar = pen0 > 0 ? fmin(r, r * r * st / (4 * pen0)) : r;
    for (int q = 0; q < 3; q++) P[q] = C[q] + (st > (creal)1e-9 ? g[q] / st * sbar : (creal)0);
    const int axs[2] = {i, j};
    for (int q = 0; q < 2; q++) {
      const int u = axs[q];
      const creal lo = fmax(C[u] - r, -B.size[u]), hi = fmin(C[u] + r, B.size[u]);
      if (lo > hi) return;
      P[u] = fmin(fmax(P[u], lo), hi);
    }
    P[k] = C[k] - (acap[i] * (P[i] - C[i]) + acap[j] * (P[j] - C[j])) / acap[k];
    pen = sgn * P[k] + B.size[k];
  } else if (fabs(ak) < (creal)0.1) {
    /* ---- generator line on face */
    creal d[3], L0[3];
    for (int q = 0; q < 3; q++) d[q] = -(sgn * a[k]) * a[q];
    d[k] += sgn;
    v3normalize(d);
    for (int q = 0; q < 3; q++) L0[q] = cB[q] + r * d[q];
    creal t0 = -h, t1 = h;
    const int axs[2] = {i, j};
    for (int q = 0; q < 2; q++) {
      const int u = axs[q];
      if (fabs(a[u]) > (creal)1e-9) {
        const creal ta = (-B.size[u] - L0[u]) / a[u], tb = (B.size[u] - L0[u]) / a[u];
        t0 = fmax(t0, fmin(ta, tb)); t1 = fmin(t1, fmax(ta, tb));
      } else if (fabs(L0[u]) > B.size[u]) return;
    }
    if (t0 > t1) return;
    const creal tm = (creal)0.5 * (t0 + t1), Lh = (creal)0.5 * (t1 - t0), sl = sgn * a[k];
    const creal penm = sgn * (L0[k] + tm * a[k]) + B.size[k];
    creal off;
    if (penm > 0) off = fmin(fmax(sl * Lh * Lh / (3 * penm), -Lh), Lh);
    else off = sl > 0 ? Lh : (sl < 0 ? -Lh : (creal)0);
    const creal ts = tm + off;
    for (int q = 0; q < 3; q++) P[q] = L0[q] + ts * a[q];
    pen = sgn * P[k] + B.size[k];
  } else return;
  o->dist = -pen;
  P[k] -= sgn * (creal)0.5 * pen;
  mat_mulvec(o->pos, B.mat, P); v3add(o->pos, o->pos, B.pos);
}

// Cylinder vs box with the cylinder axis parallel to a box axis (buttons in housings, handles, a puck at rest): the
// problem separates into an interval overlap along the axis and disc-vs-rectangle across it, so distance, depth and
// normal are exact and cheap.  Evaluated one pair per lane.  Returns -1 when the axes are not parallel (GJK/EPA then).
DEV int cyl_box_aligned(const DShape& A, const DShape& B, creal margin, RawCon* o) {
  creal ax[3], a[3], t[3], c[3];
  mat_col(ax, A.mat, 2); mat_tmulvec(a, B.mat, ax);
  int k = 0; for (int q = 1; q < 3; q++) if (fabs(a[q]) > fabs(a[k])) k = q;
  if (fabs(a[k]) < 1 - (creal)1e-6) return -1;      // within ~1.4 mrad: MJCF quaternions like "0.7074 0.7068 0 0" count as parallel
  const int i = (k + 1) % 3, j = (k + 2) % 3;
  v3sub(t, A.pos, B.pos); mat_tmulvec(c, B.mat, t);
  const creal r = A.size[0], h = A.size[1]; const creal* s = B.size;
  const creal cz = c[k], sz = cz >= 0 ? (creal)1 : (creal)-1;
  const creal ga = fabs(cz) - (h + s[k]);
  const creal p[2] = {c[i], c[j]};
  const creal q[2] = {fmin(fmax(p[0], -s[i]), s[i]), fmin(fmax(p[1], -s[j]), s[j])};
  creal n2[2], gr;
  if (q[0] != p[0] || q[1] != p[1]) {
    const creal dv[2] = {p[0] - q[0], p[1] - q[1]}, dl = sqrt(dv[0] * dv[0] + dv[1] * dv[1]);
    gr = dl - r; n2[0] = dv[0] / dl; n2[1] = dv[1] / dl;
  } else {
    const creal ei = s[i] - fabs(p[0]), ej = s[j] - fabs(p[1]);
    if (ei <= ej) { gr = -ei - r; n2[0] = p[0] >= 0 ? (creal)1 : (creal)-1; n2[1] = 0; }
    else { gr = -ej - r; n2[0] = 0; n2[1] = p[1] >= 0 ? (creal)1 : (creal)-1; }
  }
  creal nB[3] = {0, 0, 0}, P[3], dist;
  if (ga > 0 && gr > 0) {
    dist = sqrt(ga * ga + gr * gr);
    nB[i] = gr * n2[0] / dist; nB[j] = gr * n2[1] / dist; nB[k] = ga * sz / dist;
    P[i] = (creal)0.5 * (p[0] - r * n2[0] + q[0]); P[j] = (creal)0.5 * (p[1] - r * n2[1] + q[1]); P[k] = (creal)0.5 * (cz - sz * h + sz * s[k]);
  } else if (ga > gr) {
    dist = ga; nB[k] = sz;
    P[i] = q[0]; P[j] = q[1]; P[k] = sz * s[k] + (creal)0.5 * ga * sz;
  } else {
    dist = gr; nB[i] = n2[0]; nB[j] = n2[1];
    const creal z0 = fmax(cz - h, -s[k]), z1 = fmin(cz + h, s[k]);
    P[i] = p[0] - (r + (creal)0.5 * gr) * n2[0]; P[j] = p[1] - (r + (creal)0.5 * gr) * n2[1]; P[k] = (creal)0.5 * (z0 + z1);
  }
  if (dist > margin + (creal)1e-4) return 0;
  o->dist = dist;
  v3scl(nB, nB, -1);
  mat_mulvec(o->normal, B.mat, nB);
  mat_mulvec(o->pos, B.mat, P); v3add(o->pos, o->pos, B.pos);
  refine_cyl_box(A, B, o);
  return o->dist <= margin ? 1 : 0;
}
// Two cylinders with parallel axes (the faucet's stacked discs): same separation of variables.
DEV int cyl_cyl_parallel(const DShape& A, const DShape& B, creal margin, RawCon* o) {
  creal a1[3], a2[3], c[3], cr[3], u[3];
  mat_col(a1, A.mat, 2); mat_col(a2, B.mat, 2);
  if (fabs(v3dot(a1, a2)) < 1 - (creal)1e-6) return -1;
  v3sub(c, B.pos, A.pos);
  const creal cz = v3dot(c, a1), sz = cz >= 0 ? (creal)1 : (creal)-1;
  v3addscl(cr, c, a1, -cz);
  const creal rho = v3norm(cr);
  if (rho > (creal)1e-12) v3scl(u, cr, 1 / rho); else mat_col(u, A.mat, 0);
  const creal r1 = A.size[0], h1 = A.size[1], r2 = B.size[0], h2 = B.size[1];
  const creal ga = fabs(cz) - (h1 + h2), gr = rho - (r1 + r2);
  creal dist, n[3], P[3];
  if (ga > 0 && gr > 0) {
    dist = sqrt(ga * ga + gr * gr);
    for (int q = 0; q < 3; q++) {
      n[q] = (gr * u[q] + ga * sz * a1[q]) / dist;
      const creal pa = A.pos[q] + r1 * u[q] + sz * h1 * a1[q], pb = B.pos[q] - r2 * u[q] - sz * h2 * a1[q];
      P[q] = (creal)0.5 * (pa + pb);
    }
  } else if (ga > gr) {
    dist = ga;
    const creal t0 = fmax(-r1, rho - r2), t1 = fmin(r1, rho + r2), tm = (creal)0.5 * (t0 + t1);
    for (int q = 0; q < 3; q++) { n[q] = sz * a1[q]; P[q] = A.pos[q] + tm * u[q] + (sz * h1 + (creal)0.5 * ga * sz) * a1[q]; }
  } else {
    dist = gr;
    const creal z0 = fmax(-h1, cz - h2), z1 = fmin(h1, cz + h2), zm = (creal)0.5 * (z0 + z1);
    for (int q = 0; q < 3; q++) { n[q] = u[q]; P[q] = A.pos[q] + (r1 + (creal)0.5 * gr) * u[q] + zm * a1[q]; }
  }
  if (dist > margin) return 0;
  o->dist = dist; v3copy(o->normal, n); v3copy(o->pos, P);
  return 1;
}

// Whole warp calls this with identical A, B.  The result (count 0/1, contact in *o) is valid on every lane.
// GJK distance query, then EPA for penetration; the same algorithm, iteration limits and tolerances as the float64 CPU
// restatement the tests compare against.  GJK and the simplex growth are leader-driven (lane 0 owns the simplex; every
// support query is evaluated by the whole warp, mesh hull vertices split across lanes):
//   leader: choose next direction or stop  ->  broadcast  ->  warp: support point  ->  leader: consume.
// The EPA expansion loop is warp-parallel: closest-face search, visibility test, horizon extraction and face creation
// are lane-strided over the polytope with deterministic (index-ordered) compaction.
#define GJK_FINISH() { /* GJK stopped without enclosing the origin: closest points from the simplex; touching cores go on to EPA */ \
    creal w4_[3]; simplex_weights(s, n, w4_); v3zero(fwa); v3zero(fwb); \
    for (int i_ = 0; i_ < n && i_ < 3; i_++) { v3addscl(fwa, fwa, s[i_].a, w4_[i_]); v3addscl(fwb, fwb, s[i_].b, w4_[i_]); } \
    creal dv_[3]; v3sub(dv_, fwb, fwa); fdcore = v3norm(dv_); \
    if (fdcore > (creal)1e-10) { outcome = 1; st = ST_DONE; } else { st = ST_G1; k = 0; } }
// `hint` (optional): the pair's separating-axis hint (sep_hint_test), updated by lane 0 when the result is decisive: the
// separating direction on a "no contact" proven by an axis or by the GJK distance, SEP_HIT on a contact; left alone
// otherwise.  It is never read here: the GJK path does not depend on it.
__device__ __noinline__ int convex_pair(const DShape& A, const DShape& B, creal margin, RawCon* o, EpaSm* E, EpaWs* W, int lane, long long* prof = nullptr,
                                        float4* hint = nullptr) {
  const creal dirs[6][3] = {{1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
  const creal ra = core_radius(A), rb = core_radius(B);
  enum { ST_GJK0 = 0, ST_GJK, ST_G1, ST_G2, ST_G3, ST_EPA, ST_DONE };
  // ---- leader state
  SV* const s = (SV*)E->fd;   // the GJK simplex (4 x 72 B, lane 0 only) lives in the not-yet-used EPA face array: shared memory, not local
  int n = 0; creal v[3];
  int st = ST_GJK0, git = 0, k = 0, sg = 0;
  int outcome = 0;          // 0 none, 1 separated result ready, 2 EPA finished (use bestf), 3 no contact
  creal ab[3] = {0, 0, 0}, gd[3] = {0, 0, 0}, nn[3] = {0, 0, 0}, vv = 0;
  creal dirl[3] = {1, 0, 0}, fwa[3] = {0, 0, 0}, fwb[3] = {0, 0, 0}, fdcore = 0;
  v3sub(v, A.pos, B.pos);
  if (v3dot(v, v) < (creal)1e-24) { v[0] = 1; v[1] = v[2] = 0; }
  for (int guard = 0; guard < 128; guard++) {
    // ---------------- leader: decide the next query (or stop)
    if (lane == 0) {
      bool query = false;
      while (!query && st != ST_DONE && st != ST_EPA) {
        if (st == ST_GJK0) { v3scl(dirl, v, -1); query = true; }
        else if (st == ST_GJK) {
          vv = v3dot(v, v);
          if (vv < (creal)1e-24) { st = ST_G1; k = 0; }                       // enclosed
          else if (git >= 64) GJK_FINISH()
          else { v3scl(dirl, v, -1); query = true; }
        } else if (st == ST_G1) {                                               // grow a point to a segment
          if (n != 1) { st = ST_G2; k = 0; sg = 0; if (n == 2) v3sub(ab, s[1].v, s[0].v); }
          else if (k >= 6) { st = ST_G2; }
          else { v3copy(dirl, dirs[k]); query = true; }
        } else if (st == ST_G2) {                                               // segment to a triangle
          if (n != 2) { st = ST_G3; sg = 0; if (n == 3) { creal ac[3], a2[3]; v3sub(a2, s[1].v, s[0].v); v3sub(ac, s[2].v, s[0].v); v3cross(nn, a2, ac); } }
          else if (k >= 6) { outcome = 3; st = ST_DONE; }
          else if (sg == 0) {
            v3cross(gd, ab, dirs[k]);
            if (v3dot(gd, gd) < (creal)1e-12 * v3dot(ab, ab)) k++;
            else { v3copy(dirl, gd); query = true; }
          } else { v3scl(dirl, gd, -1); query = true; }
        } else if (st == ST_G3) {                                               // triangle to a tetrahedron
          if (n == 4) {
            for (int i = 0; i < 4; i++) for (int q = 0; q < 3; q++) { E->vv[i][q] = s[i].v[q]; W->va[i][q] = s[i].a[q]; W->vb[i][q] = s[i].b[q]; }
            epa_set_face(E, W, 0, 0, 1, 2); epa_set_face(E, W, 1, 0, 2, 3); epa_set_face(E, W, 2, 0, 3, 1); epa_set_face(E, W, 3, 1, 3, 2);
            st = ST_EPA;
          } else if (n != 3 || sg >= 2) { outcome = 3; st = ST_DONE; }
          else { if (sg == 0) v3copy(dirl, nn); else v3scl(dirl, nn, -1); query = true; }
        }
      }
    }
    const int stb = __shfl_sync(FULLMASK, st, 0);
    if (stb == ST_DONE || stb == ST_EPA) break;
    creal dir[3] = {bcast(dirl[0], 0), bcast(dirl[1], 0), bcast(dirl[2], 0)};
    SV w; support_pair(A, B, dir, &w, lane);
    // ---------------- leader: consume the support point
    int need_cs = 0;
    if (lane == 0) {
      if (st == ST_GJK0) { s[0] = w; n = 1; v3copy(v, w.v); st = ST_GJK; git = 0; }
      else if (st == ST_GJK) {
        const creal vw = v3dot(v, w.v);
        if (vv - vw <= (creal)1e-12 * vv || vv - vw <= GJK_TOL * sqrt(vv)) GJK_FINISH()             // |v| within GJK_TOL of the lower bound: closest point found
        else if (vw > 0 && vw / sqrt(vv) - ra - rb > margin + (creal)1e-4) {                             // separating axis
          outcome = 3; st = ST_DONE;
          if (hint) sep_hint_store(hint, dirl, SEP_APART);                                                  // dirl = -v: from A towards B
        }
        else {
          bool dup = false;
          for (int i = 0; i < n; i++) { creal t[3]; v3sub(t, s[i].v, w.v); if (v3dot(t, t) < (creal)1e-24) dup = true; }
          if (dup) GJK_FINISH()
          else { s[n++] = w; need_cs = 1; }
        }
      } else if (st == ST_G1) {
        creal dd[3]; v3sub(dd, w.v, s[0].v);
        if (v3dot(dd, dd) > (creal)1e-20) s[n++] = w;
        k++;
      } else if (st == ST_G2) {
        creal aw[3], cr[3]; v3sub(aw, w.v, s[0].v); v3cross(cr, ab, aw);
        if (v3dot(cr, cr) > (creal)1e-20) s[n++] = w;
        else { sg++; if (sg == 2) { sg = 0; k++; } }
      } else if (st == ST_G3) {
        creal aw[3]; v3sub(aw, w.v, s[0].v);
        if (fabs(v3dot(aw, nn)) > (creal)1e-14 * sqrt(v3dot(nn, nn))) s[n++] = w;
        else sg++;
      }
    }
    if (__shfl_sync(FULLMASK, need_cs, 0)) {   // simplex reduction with the whole warp (tetrahedron faces in parallel)
      __syncwarp();
      const bool enc = closest_simplex(s, &n, v, lane);
      if (lane == 0) { if (enc) { st = ST_G1; k = 0; } git++; }
      __syncwarp();
    }
  }
  // ---------------- EPA expansion, warp-parallel (uniform control flow; nv, nf, bestf identical on all lanes)
  int bestf = -1, eit = 0;
  if (__shfl_sync(FULLMASK, st, 0) == ST_EPA) {
    __syncwarp();
    int nv = 4, nf = 4;
    outcome = 2;
    for (eit = 0; eit < EPA_ITERS; eit++) {
      // closest face to the origin (lowest index on ties)
      creal bd = (creal)1e300; int bf = -1;
      for (int f = lane; f < nf; f += MW_WARP) if (E->alive[f] && E->fd[f] < bd) { bd = E->fd[f]; bf = f; }
#pragma unroll
      for (int x = 16; x > 0; x >>= 1) {
        const creal od = __shfl_xor_sync(FULLMASK, bd, x); const int of = __shfl_xor_sync(FULLMASK, bf, x);
        if (of >= 0 && (bf < 0 || od < bd || (od == bd && of < bf))) { bd = od; bf = of; }
      }
      bestf = bf;
      if (bestf < 0) { outcome = 3; break; }
      creal dir[3] = {W->fn[0][bestf], W->fn[1][bestf], W->fn[2][bestf]};
      SV w; support_pair(A, B, dir, &w, lane);
      const creal dw = v3dot(w.v, dir);
      if (dw - bd < EPA_TOL || nv >= EPA_MAXV) break;
      // faces visible from w, ascending
      int nvis = 0;
      for (int base = 0; base < nf; base += MW_WARP) {
        const int f = base + lane;
        bool vsb = false;
        if (f < nf && E->alive[f]) {
          const int v0 = E->fv[0][f];
          const creal t[3] = {w.v[0] - E->vv[v0][0], w.v[1] - E->vv[v0][1], w.v[2] - E->vv[v0][2]};
          vsb = W->fn[0][f] * t[0] + W->fn[1][f] * t[1] + W->fn[2][f] * t[2] > (creal)1e-14;
        }
        const unsigned mk = __ballot_sync(FULLMASK, vsb);
        if (vsb) E->vis[nvis + __popc(mk & ((1u << lane) - 1))] = (short)f;
        nvis += __popc(mk);
      }
      __syncwarp();
      // horizon edges in (face, edge) order: an edge of a visible face whose reverse is not an edge of a visible face
      int ne = 0; bool ovf = false;
      for (int base = 0; base < 3 * nvis; base += MW_WARP) {
        const int x = base + lane;
        bool hz = false; int ea = 0, eb = 0;
        if (x < 3 * nvis) {
          const int f = E->vis[x / 3], e = x % 3;
          ea = E->fv[e][f]; eb = E->fv[(e + 1) % 3][f];
          hz = true;
          for (int y = 0; y < nvis && hz; y++) {
            const int g = E->vis[y];
            const int g0 = E->fv[0][g], g1 = E->fv[1][g], g2 = E->fv[2][g];
            if ((g0 == eb && g1 == ea) || (g1 == eb && g2 == ea) || (g2 == eb && g0 == ea)) hz = false;
          }
        }
        const unsigned mk = __ballot_sync(FULLMASK, hz);
        const int slot = ne + __popc(mk & ((1u << lane) - 1));
        if (hz) { if (slot < EPA_MAXE) { E->hz[slot][0] = (short)ea; E->hz[slot][1] = (short)eb; } }
        ne += __popc(mk);
      }
      if (ne > EPA_MAXE) ovf = true;
      for (int x = lane; x < nvis; x += MW_WARP) E->alive[E->vis[x]] = 0;
      __syncwarp();
      if (ne == 0 || ovf || nf + ne > EPA_MAXF) break;
      const int wi = nv;
      for (int c = lane; c < 3; c += MW_WARP) { E->vv[wi][c] = w.v[c]; W->va[wi][c] = w.a[c]; W->vb[wi][c] = w.b[c]; }
      nv++;
      __syncwarp();
      for (int q = lane; q < ne; q += MW_WARP) epa_set_face(E, W, nf + q, E->hz[q][0], E->hz[q][1], wi);
      nf += ne;
      __syncwarp();
    }
  }
  // ---------------- leader: build the contact
  int result = 0;
  RawCon rc; rc.dist = 0; v3zero(rc.pos); v3zero(rc.normal);
  if (lane == 0) {
    creal wa[3] = {0, 0, 0}, wb[3] = {0, 0, 0};
    bool have = false;
    if (outcome == 1) {
      const creal dist = fdcore - ra - rb;
      if (dist <= margin + (creal)1e-4) {      // slack: the analytic refinement below makes the final call
        creal dvec[3]; v3sub(dvec, fwb, fwa);
        v3scl(rc.normal, dvec, 1 / fdcore); rc.dist = dist; have = true;
        v3copy(wa, fwa); v3copy(wb, fwb);
      } else if (hint) { creal dvec[3]; v3sub(dvec, fwb, fwa); sep_hint_store(hint, dvec, SEP_APART); }
    } else if (outcome == 2 && bestf >= 0) {
      const int i0 = E->fv[0][bestf], i1 = E->fv[1][bestf], i2 = E->fv[2][bestf];
      creal w3[3]; closest_tri(E->vv[i0], E->vv[i1], E->vv[i2], w3);
      const int ids[3] = {i0, i1, i2};
      for (int q = 0; q < 3; q++) for (int c = 0; c < 3; c++) { wa[c] += W->va[ids[q]][c] * w3[q]; wb[c] += W->vb[ids[q]][c] * w3[q]; }
      const creal dist = -E->fd[bestf] - ra - rb;
      if (dist <= margin) { rc.dist = dist; rc.normal[0] = W->fn[0][bestf]; rc.normal[1] = W->fn[1][bestf]; rc.normal[2] = W->fn[2][bestf]; have = true; }
    }
    if (have) {
      for (int q = 0; q < 3; q++) rc.pos[q] = (creal)0.5 * (wa[q] + rc.normal[q] * ra + wb[q] - rc.normal[q] * rb);
      refine_cyl_box(A, B, &rc);
      result = rc.dist <= margin ? 1 : 0;
      if (hint && result) sep_hint_store(hint, rc.normal, SEP_HIT);
    }
    if (prof) { prof[10] += eit; prof[11] += git; }
  }
  __syncwarp();
  result = __shfl_sync(FULLMASK, result, 0);
  o->dist = bcast(rc.dist, 0);
  for (int q = 0; q < 3; q++) { o->pos[q] = bcast(rc.pos[q], 0); o->normal[q] = bcast(rc.normal[q], 0); }
  return result;
}
