/* ray_oracle.c -- TEST-ONLY scalar fp64 restatement of the terrain ray rules (DESIGN.md section 3), the reference the ray kernel and its host
 * emulation are compared with.  It knows nothing of the product's layouts: rays arrive in world coordinates, the static geoms as (type, world
 * position, rotation, size) in slot order, the height field as its elevations.  Built into its own library by tests/raycast_support.py.
 *
 * oracle_raycast: out[k][4] = distance (-1: none), world z of the hit (of the end point when none), slot (-1), 0.  Per geom:
 *   plane  (type 0): MuJoCo's ray_plane -- front face only, t >= 0, inside |x| <= size[0], |y| <= size[1] where those are > 0
 *   hfield (type 1): the top surface, two triangles per cell split along (r, c+1)-(r+1, c), both faces; every cell of the xy bounding box of the
 *                    segment clipped to the field is tested (no grid walk)
 *   box    (type 6): slab test; the first surface crossing at t >= 0 (from inside: the exit)
 * The nearest hit in [0, max] wins; on a tie the lower slot. */
#include <math.h>

#define TRI_EPS 1e-12

static double dot(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

/* R row-major; local = R^T (p - pos) */
static void to_local(const double *pos, const double *R, const double *p, double *l) {
  const double w[3] = {p[0] - pos[0], p[1] - pos[1], p[2] - pos[2]};
  for (int i = 0; i < 3; i++) l[i] = R[i] * w[0] + R[3 + i] * w[1] + R[6 + i] * w[2];
}
static void to_local_dir(const double *R, const double *d, double *l) {
  for (int i = 0; i < 3; i++) l[i] = R[i] * d[0] + R[3 + i] * d[1] + R[6 + i] * d[2];
}

static double plane(const double *pos, const double *R, const double *s, const double *o, const double *d) {
  double lo[3], ld[3]; to_local(pos, R, o, lo); to_local_dir(R, d, ld);
  if (ld[2] > -1e-15) return -1;
  const double t = -lo[2] / ld[2];
  if (t < 0) return -1;
  const double x = lo[0] + t * ld[0], y = lo[1] + t * ld[1];
  if ((s[0] <= 0 || fabs(x) <= s[0]) && (s[1] <= 0 || fabs(y) <= s[1])) return t;
  return -1;
}

static double box(const double *pos, const double *R, const double *s, const double *o, const double *d) {
  double lo[3], ld[3]; to_local(pos, R, o, lo); to_local_dir(R, d, ld);
  double t0 = -1e300, t1 = 1e300;
  for (int i = 0; i < 3; i++) {
    if (ld[i] == 0) { if (fabs(lo[i]) > s[i]) return -1; continue; }
    double a = (-s[i] - lo[i]) / ld[i], b = (s[i] - lo[i]) / ld[i];
    if (a > b) { const double t = a; a = b; b = t; }
    if (a > t0) t0 = a;
    if (b < t1) t1 = b;
  }
  if (t1 < t0 || t1 < 0) return -1;
  return t0 >= 0 ? t0 : t1;
}

static double tri(const double *o, const double *d, const double *a, const double *b, const double *c) {
  const double e1[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, e2[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
  const double p[3] = {d[1] * e2[2] - d[2] * e2[1], d[2] * e2[0] - d[0] * e2[2], d[0] * e2[1] - d[1] * e2[0]};
  const double det = dot(e1, p);
  if (fabs(det) < 1e-15) return -1;
  const double sv[3] = {o[0] - a[0], o[1] - a[1], o[2] - a[2]};
  const double u = dot(sv, p) / det;
  if (u < -TRI_EPS || u > 1 + TRI_EPS) return -1;
  const double q[3] = {sv[1] * e1[2] - sv[2] * e1[1], sv[2] * e1[0] - sv[0] * e1[2], sv[0] * e1[1] - sv[1] * e1[0]};
  const double v = dot(d, q) / det;
  if (v < -TRI_EPS || u + v > 1 + TRI_EPS) return -1;
  return dot(e2, q) / det;
}

static double hfield(const double *pos, const double *hf, int nrow, int ncol, const double *hs, const double *ow, const double *d, double tmax) {
  const double o[3] = {ow[0] - pos[0], ow[1] - pos[1], ow[2] - pos[2]};
  const double sx = hs[0], sy = hs[1], sz = hs[2], dx = 2 * sx / (ncol - 1), dy = 2 * sy / (nrow - 1);
  double t0 = 0, t1 = tmax;
  for (int i = 0; i < 2; i++) {
    const double h = i ? sy : sx;
    if (d[i] == 0) { if (fabs(o[i]) > h) return -1; continue; }
    double a = (-h - o[i]) / d[i], b = (h - o[i]) / d[i];
    if (a > b) { const double t = a; a = b; b = t; }
    if (a > t0) t0 = a;
    if (b < t1) t1 = b;
  }
  if (t0 > t1) return -1;
  const double xa = o[0] + t0 * d[0], xb = o[0] + t1 * d[0], ya = o[1] + t0 * d[1], yb = o[1] + t1 * d[1];
  int c0 = (int)floor(((xa < xb ? xa : xb) + sx) / dx) - 1, c1 = (int)floor(((xa < xb ? xb : xa) + sx) / dx) + 1;
  int r0 = (int)floor(((ya < yb ? ya : yb) + sy) / dy) - 1, r1 = (int)floor(((ya < yb ? yb : ya) + sy) / dy) + 1;
  if (c0 < 0) c0 = 0;
  if (r0 < 0) r0 = 0;
  if (c1 > ncol - 2) c1 = ncol - 2;
  if (r1 > nrow - 2) r1 = nrow - 2;
  double best = -1;
  for (int r = r0; r <= r1; r++) for (int c = c0; c <= c1; c++) {
    const double x0 = -sx + c * dx, y0 = -sy + r * dy;
    const double v00[3] = {x0, y0, hf[r * ncol + c] * sz}, v10[3] = {x0 + dx, y0, hf[r * ncol + c + 1] * sz};
    const double v01[3] = {x0, y0 + dy, hf[(r + 1) * ncol + c] * sz}, v11[3] = {x0 + dx, y0 + dy, hf[(r + 1) * ncol + c + 1] * sz};
    const double ta = tri(o, d, v00, v10, v01), tb = tri(o, d, v10, v11, v01);
    if (ta >= t0 && ta <= t1 && (best < 0 || ta < best)) best = ta;
    if (tb >= t0 && tb <= t1 && (best < 0 || tb < best)) best = tb;
  }
  return best;
}

/* ng static geoms: type[ng], pos[ng][3], R[ng][9] (row-major world rotation), size[ng][3]; hf [nrow][ncol] normalised elevations (or 0), hsize[4];
 * k rays: org[k][3], dir[k][3] (unit), maxd[k] */
int oracle_raycast(int ng, const int *type, const double *pos, const double *R, const double *size, const double *hf, int nrow, int ncol, const double *hsize,
                   int k, const double *org, const double *dir, const double *maxd, double *out) {
  for (int i = 0; i < k; i++) {
    const double *o = org + 3 * i, *d = dir + 3 * i;
    double best = -1; int gb = -1;
    for (int g = 0; g < ng; g++) {
      double t = -1;
      if (type[g] == 0) t = plane(pos + 3 * g, R + 9 * g, size + 3 * g, o, d);
      else if (type[g] == 6) t = box(pos + 3 * g, R + 9 * g, size + 3 * g, o, d);
      else if (type[g] == 1 && hf) t = hfield(pos + 3 * g, hf, nrow, ncol, hsize, o, d, maxd[i]);
      if (t >= 0 && t <= maxd[i] && (gb < 0 || t < best)) { best = t; gb = g; }
    }
    out[4 * i] = gb >= 0 ? best : -1;
    out[4 * i + 1] = o[2] + (gb >= 0 ? best : maxd[i]) * d[2];
    out[4 * i + 2] = gb;
    out[4 * i + 3] = 0;
  }
  return 0;
}
