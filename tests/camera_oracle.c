/* camera_oracle.c -- TEST-ONLY scalar fp64 restatement of the depth-camera rules (DESIGN.md section 3, "Depth camera"), the reference the camera
 * kernel and its host emulation are compared with.  It extends the ray oracle (tests/ray_oracle.c, included: the static-geom rules are its own) with
 * the pixel rays, the moving geoms and the z-depth, and knows nothing of the product's layouts: the camera arrives as its world position and
 * rotation, every geom as (type, world position, rotation, size).  Built into its own library by tests/camera_support.py.
 *
 * oracle_camera: depth[H][W] and geom[H][W] (static slot g, moving geom 100 + m, -1 for nothing within zfar).  Pixel (r, c) casts the unit ray along
 * R (x, y, -1) / |(x, y, -1)|, x = (2 (c + 1/2) / W - 1) tan(fovy / 2) W / H, y = (1 - 2 (r + 1/2) / H) tan(fovy / 2); a hit at distance t has
 * z-depth t / |(x, y, -1)|; the nearest hit with t > 0 and z-depth <= zfar wins (on a tie the static geom, then the lower index), else zfar.
 *   static geoms: the ray oracle's plane, box and height-field rules, cast up to the distance of depth zfar
 *   moving geoms, seen from outside only (nothing when the ray starts inside or on the geom):
 *     sphere  (type 2): |o + t d - p| = r, the smaller root
 *     capsule (type 3): MuJoCo's ray_capsule -- the cylinder |z| <= size[1] of radius size[0], and the two hemispheres beyond its ends
 *     box     (type 6): slab test, the entry */
#include "ray_oracle.c"

static double sphere_entry(const double *c, double r, const double *o, const double *d) {
  const double w[3] = {o[0] - c[0], o[1] - c[1], o[2] - c[2]};
  const double b = dot(w, d), cc = dot(w, w) - r * r, disc = b * b - cc;   /* |d| = 1 */
  if (disc < 0) return -1;
  const double t = -b - sqrt(disc);
  return t > 0 ? t : -1;
}

static double moving(int type, const double *pos, const double *R, const double *s, const double *o, const double *d) {
  double lo[3], ld[3]; to_local(pos, R, o, lo); to_local_dir(R, d, ld);
  if (type == 2) {
    if (dot(lo, lo) <= s[0] * s[0]) return -1;
    return sphere_entry(pos, s[0], o, d);
  }
  if (type == 3) {
    const double r = s[0], h = s[1], zc = lo[2] < -h ? -h : (lo[2] > h ? h : lo[2]);
    if (lo[0] * lo[0] + lo[1] * lo[1] + (lo[2] - zc) * (lo[2] - zc) <= r * r) return -1;
    double best = -1;
    const double a = ld[0] * ld[0] + ld[1] * ld[1], b = lo[0] * ld[0] + lo[1] * ld[1], c = lo[0] * lo[0] + lo[1] * lo[1] - r * r;
    if (a > 1e-15 && b * b - a * c >= 0) {
      const double t = (-b - sqrt(b * b - a * c)) / a, z = lo[2] + t * ld[2];
      if (t > 0 && fabs(z) <= h) best = t;
    }
    for (int k = 0; k < 2; k++) {   /* hemisphere k: the sphere about the end z = +-h, hits beyond that end only */
      const double zs = k ? -h : h, cl[3] = {0, 0, zs};
      const double t = sphere_entry(cl, r, lo, ld);
      if (t > 0 && (k ? lo[2] + t * ld[2] <= -h : lo[2] + t * ld[2] >= h) && (best < 0 || t < best)) best = t;
    }
    return best;
  }
  if (type == 6) {
    if (fabs(lo[0]) < s[0] && fabs(lo[1]) < s[1] && fabs(lo[2]) < s[2]) return -1;
    return box(pos, R, s, o, d);
  }
  return -1;
}

int oracle_camera(int ng, const int *type, const double *pos, const double *R, const double *size, const double *hf, int nrow, int ncol, const double *hsize,
                  int nm, const int *mtype, const double *mpos, const double *mR, const double *msize,
                  const double *cpos, const double *cR, double fovy, int W, int H, double zfar, double *depth, int *geom) {
  const double ty = tan(fovy * 3.14159265358979323846 / 360), tx = ty * W / H;
  for (int r = 0; r < H; r++) for (int c = 0; c < W; c++) {
    const double dc[3] = {(2 * (c + 0.5) / W - 1) * tx, (1 - 2 * (r + 0.5) / H) * ty, -1};
    const double nd = sqrt(dot(dc, dc)), tmax = zfar * nd;
    double d[3];
    for (int i = 0; i < 3; i++) d[i] = (cR[3 * i] * dc[0] + cR[3 * i + 1] * dc[1] + cR[3 * i + 2] * dc[2]) / nd;
    double best = -1; int gb = -1;
    for (int g = 0; g < ng; g++) {
      double t = -1;
      if (type[g] == 0) t = plane(pos + 3 * g, R + 9 * g, size + 3 * g, cpos, d);
      else if (type[g] == 6) t = box(pos + 3 * g, R + 9 * g, size + 3 * g, cpos, d);
      else if (type[g] == 1 && hf) t = hfield(pos + 3 * g, hf, nrow, ncol, hsize, cpos, d, tmax);
      if (t > 0 && t <= tmax && (gb < 0 || t < best)) { best = t; gb = g; }
    }
    for (int m = 0; m < nm; m++) {
      const double t = moving(mtype[m], mpos + 3 * m, mR + 9 * m, msize + 3 * m, cpos, d);
      if (t > 0 && t <= tmax && (gb < 0 || t < best)) { best = t; gb = 100 + m; }
    }
    depth[r * W + c] = gb >= 0 ? best / nd : zfar;
    geom[r * W + c] = gb;
  }
  return 0;
}
