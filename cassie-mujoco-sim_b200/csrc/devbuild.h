// devbuild.h -- host code that turns a HostModel into the DevModel<real> constant block, and the initial per-env state rows.
#pragma once
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <vector>
#include "devmodel.h"
#include "model.h"
#include "cassie_tree_gen.inc"

namespace cassie {

namespace detail {
inline void q2m_d(double *m, const double *q) {
  double w = q[0], x = q[1], y = q[2], z = q[3];
  m[0] = w * w + x * x - y * y - z * z; m[1] = 2 * (x * y - w * z); m[2] = 2 * (x * z + w * y);
  m[3] = 2 * (x * y + w * z); m[4] = w * w - x * x + y * y - z * z; m[5] = 2 * (y * z - w * x);
  m[6] = 2 * (x * z - w * y); m[7] = 2 * (y * z + w * x); m[8] = w * w - x * x - y * y + z * z;
}
}  // namespace detail

// world pose of geom g on a static body (the world or a body welded to it) with its frame in the body given by pos / quat (MuJoCo's geom_pos /
// geom_quat), in the layout the collision stage reads: position, then the z, x and y axes of the geom frame.  The chain of static bodies is constant.
inline void static_geom_wpose(const HostModel &m, int g, const double *pos, const double *quat, double *w) {
  double R[9]; detail::q2m_d(R, quat);
  double bp[3] = {0, 0, 0}, bq[4] = {1, 0, 0, 0};
  { std::vector<int> chain; for (int bb = m.geom_bodyid[g]; bb > 0; bb = m.body_parentid[bb]) chain.push_back(bb);
    for (int i = (int)chain.size() - 1; i >= 0; i--) { const int bb = chain[i]; double Rb[9], v[3]; detail::q2m_d(Rb, bq);
      for (int r = 0; r < 3; r++) v[r] = Rb[3 * r] * m.body_pos[3 * bb] + Rb[3 * r + 1] * m.body_pos[3 * bb + 1] + Rb[3 * r + 2] * m.body_pos[3 * bb + 2];
      for (int r = 0; r < 3; r++) bp[r] += v[r];
      const double *q2 = &m.body_quat[4 * bb]; const double t[4] = {bq[0] * q2[0] - bq[1] * q2[1] - bq[2] * q2[2] - bq[3] * q2[3], bq[0] * q2[1] + bq[1] * q2[0] + bq[2] * q2[3] - bq[3] * q2[2],
                                                                    bq[0] * q2[2] - bq[1] * q2[3] + bq[2] * q2[0] + bq[3] * q2[1], bq[0] * q2[3] + bq[1] * q2[2] - bq[2] * q2[1] + bq[3] * q2[0]};
      for (int r = 0; r < 4; r++) bq[r] = t[r]; } }
  double Rb[9], W[9], wp[3]; detail::q2m_d(Rb, bq);
  for (int r = 0; r < 3; r++) { wp[r] = bp[r] + Rb[3 * r] * pos[0] + Rb[3 * r + 1] * pos[1] + Rb[3 * r + 2] * pos[2];
    for (int c = 0; c < 3; c++) W[3 * r + c] = Rb[3 * r] * R[c] + Rb[3 * r + 1] * R[3 + c] + Rb[3 * r + 2] * R[6 + c]; }
  for (int r = 0; r < 3; r++) { w[r] = wp[r]; w[3 + r] = W[3 * r + 2]; w[6 + r] = W[3 * r]; w[9 + r] = W[3 * r + 1]; }   // position, z, x, y axes
}

// one slot of a per-environment static-geom row (GEOM_ENV_W): geom g placed at pos / quat (in its body frame) with size `size`.  A box's bounding radius
// is recomputed as |size| so that a box enlarged beyond its file size is not culled by a stale bound; a plane keeps the model's (0)
template <typename real> void env_geom_slot(const HostModel &m, int g, const double *pos, const double *quat, const double *size, real *slot) {
  double w[12]; static_geom_wpose(m, g, pos, quat, w);
  for (int c = 0; c < 12; c++) slot[GE_POSE + c] = (real)w[c];
  for (int c = 0; c < 3; c++) slot[GE_SIZE + c] = (real)size[c];
  slot[GE_RBOUND] = m.geom_type[g] == GEOM_BOX ? (real)std::sqrt(size[0] * size[0] + size[1] * size[1] + size[2] * size[2]) : (real)m.geom_rbound[g];
}
// a row holding the model block's own placement of every static slot
template <typename real> void init_genv_row(const DevModel<real> &d, real *row) {
  for (int k = 0; k < MGS; k++) { real *s = row + GE_SLOT * k;
    for (int c = 0; c < 12; c++) s[GE_POSE + c] = d.geom_wpose[k][c];
    for (int c = 0; c < 3; c++) s[GE_SIZE + c] = d.geom_size[MG + k][c];
    s[GE_RBOUND] = d.geom_rbound[MG + k]; }
}
// the host geom of the model's height field (-1: none)
inline int hfield_geom(const HostModel &m) { for (int g = 0; g < m.ngeom; g++) if (m.geom_type[g] == GEOM_HFIELD) return g; return -1; }
// a height-field size [x half-extent, y half-extent, elevation scale, base thickness] the verbs accept: an empty reason, else what is wrong with it
inline std::string hfield_size_check(const double *s) {
  for (int c = 0; c < 4; c++) if (!std::isfinite(s[c])) return "size[" + std::to_string(c) + "] is not finite";
  if (!(s[0] > 0) || !(s[1] > 0)) return "the half-extents size[0], size[1] must be > 0";
  if (s[2] < 0 || s[3] < 0) return "the elevation scale size[2] and base thickness size[3] must be >= 0";
  return std::string();
}
// the height field's slot of a per-environment row (F_TR instances): geom g at pos (in its body frame, the model's orientation) with size hs[4]: GE_SIZE
// holds the half-extents and the elevation scale, GE_RBOUND the model compiler's bound |(x, y, max(elevation, base))|
template <typename real> void env_hfield_slot(const HostModel &m, int g, const double *pos, const double *hs, real *slot) {
  env_geom_slot(m, g, pos, &m.geom_quat[4 * g], hs, slot);
  const double z = std::fmax(hs[2], hs[3]);
  slot[GE_RBOUND] = (real)std::sqrt(hs[0] * hs[0] + hs[1] * hs[1] + z * z);
}
// the static collision slot (0 .. MGS-1) of host geom g, or a reason why it has none that a per-environment placement could move
inline int env_geom_check(const HostModel &m, const int *geom_dev, int g, std::string &err) {
  if (g < 0 || g >= m.ngeom) { err = "unknown geom"; return -1; }
  if (m.body_weldid[m.geom_bodyid[g]] != 0) { err = "the geom is on a moving body"; return -1; }
  if (m.geom_type[g] == GEOM_HFIELD) { err = "the height field's placement is shared by the batch"; return -1; }
  if (geom_dev[g] < MG) { err = "the geom has no collision slot (visual only)"; return -1; }
  if (m.geom_type[g] != GEOM_PLANE && m.geom_type[g] != GEOM_BOX) { err = "only planes and boxes can be placed per environment"; return -1; }
  return geom_dev[g] - MG;
}

// the obstacle broad phase's robot bound (DevModel::robot_reach, before its slack) for body offsets bp [nbody][3]: build_dev_model's rule -- the
// farthest any collision geom of the robot reaches from the root body's origin along the offset chain -- over the geoms that have a moving slot
inline double robot_reach_of(const HostModel &m, const double *bp, int root, int xb, const int *geom_dev) {
  std::vector<double> reach(m.nbody, 0.0);
  for (int b = 1; b < m.nbody; b++) if (m.body_weldid[b] != 0 && b != root && b != xb) {
    const double *p = bp + 3 * b; reach[b] = reach[m.body_parentid[b]] + std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]); }
  double r = 0;
  for (int g = 0; g < m.ngeom && g < 256; g++) {
    const int b = m.geom_bodyid[g];
    if (geom_dev[g] < 0 || geom_dev[g] >= MG || b == xb) continue;
    const double *gp = &m.geom_pos[3 * g]; r = std::max(r, reach[b] + std::sqrt(gp[0] * gp[0] + gp[1] * gp[1] + gp[2] * gp[2]) + m.geom_rbound[g]);
  }
  return r;
}
// a body offset the per-environment verb may change: an empty reason, else why not (the world body, a body welded to the world -- its geoms are static
// and placed per environment by the static-geom verbs -- and the extra free body, whose pose is qpos)
inline std::string env_body_pos_check(const HostModel &m, int b, int xb) {
  if (b == 0) return "the world body";
  if (m.body_weldid[b] == 0) return "a body welded to the world (place its geoms with cassie_batch_set_env_geom_pose / set_env_hfield)";
  if (b == xb) return "the extra free body (its pose is qpos)";
  return std::string();
}

// cassie_batch_set_env_actuators' check of every masked value, before anything changes: an empty reason, else the first refusal (a non-finite value,
// lo >= hi, rpm <= 0, a delay outside 0..AC_MAXDELAY), naming the environment and the actuator.  ctrlrange [n][nu][2], rpm [n][nu], delay [n][nu]; null
// parts are not checked (kept)
inline std::string env_actuators_check(int n, int nu, const double *ctrlrange, const double *rpm, const int *delay, const unsigned char *mask) {
  for (int e = 0; e < n; e++) {
    if (mask && !mask[e]) continue;
    for (int i = 0; i < nu; i++) {
      const std::string at = "environment " + std::to_string(e) + ", actuator " + std::to_string(i) + ": ";
      const size_t k = (size_t)e * nu + i;
      if (ctrlrange) {
        const double lo = ctrlrange[2 * k], hi = ctrlrange[2 * k + 1];
        if (!std::isfinite(lo) || !std::isfinite(hi)) return at + "ctrlrange is not finite";
        if (!(lo < hi)) return at + "ctrlrange needs lo < hi";
      }
      if (rpm && !(std::isfinite(rpm[k]) && rpm[k] > 0)) return at + "rpm must be finite and positive";
      if (delay && (delay[k] < 0 || delay[k] > AC_MAXDELAY)) return at + "delay must be in 0.." + std::to_string(AC_MAXDELAY);
    }
  }
  return std::string();
}

// cassie_batch_set_env_mechanics' check of every masked value, before anything changes: an empty reason, else the first refusal, naming the environment,
// the body / dof / joint and the field.  Refused: a non-finite value; a negative inertia moment, armature or stiffness; moments that break MuJoCo's
// compiler rule A + B >= C for some order; a change (against the shared block m, which is what get reports there) to the inertia of the world body, a
// body welded to the world or the extra free body xb, to the armature of the extra free body's dofs (>= nv_main), or to the stiffness or qpos_spring of a
// slide, ball or free joint.  inertia [n][nbody][3], armature [n][nv], stiffness and springref [n][njnt]; null parts are not checked (kept)
inline std::string env_mechanics_check(const HostModel &m, int n, int xb, int nv_main, const double *inertia, const double *armature, const double *stiffness,
                                       const double *springref, const unsigned char *mask) {
  const int nb = m.nbody, nv = m.nv, nj = m.njnt;
  auto joint = [&](int j) { return (size_t)j < m.names_joint.size() && !m.names_joint[j].empty() ? m.names_joint[j] : std::to_string(j); };   // unnamed: the index
  for (int e = 0; e < n; e++) {
    if (mask && !mask[e]) continue;
    const std::string env = "environment " + std::to_string(e) + ", ";
    if (inertia) for (int b = 0; b < nb; b++) {
      const double *I = inertia + ((size_t)e * nb + b) * 3, *I0 = &m.body_inertia[3 * b];
      const std::string at = env + "body " + m.names_body[b] + ": body_inertia ";
      for (int k = 0; k < 3; k++) {
        if (!std::isfinite(I[k])) return at + "is not finite";
        if (I[k] < 0) return at + "must be >= 0";
      }
      if (I[0] + I[1] < I[2] || I[1] + I[2] < I[0] || I[2] + I[0] < I[1]) return at + "must satisfy A + B >= C for every order of the three moments";
      if (I[0] == I0[0] && I[1] == I0[1] && I[2] == I0[2]) continue;
      const std::string w = env_body_pos_check(m, b, xb);
      if (!w.empty()) return at + "of " + w + " cannot change";
    }
    if (armature) for (int i = 0; i < nv; i++) {
      const double a = armature[(size_t)e * nv + i];
      const std::string at = env + "dof " + std::to_string(i) + " (joint " + joint(m.dof_jntid[i]) + "): dof_armature ";
      if (!std::isfinite(a)) return at + "is not finite";
      if (a < 0) return at + "must be >= 0";
      if (i >= nv_main && a != m.dof_armature[i]) return at + "of the extra free body cannot change";
    }
    for (int j = 0; j < nj; j++) {
      const std::string at = env + "joint " + joint(j) + ": ";
      const bool hinge = m.jnt_type[j] == JNT_HINGE;
      if (stiffness) {
        const double k = stiffness[(size_t)e * nj + j];
        if (!std::isfinite(k)) return at + "jnt_stiffness is not finite";
        if (k < 0) return at + "jnt_stiffness must be >= 0";
        if (!hinge && k != m.jnt_stiffness[j]) return at + "jnt_stiffness of a slide, ball or free joint cannot change";
      }
      if (springref) {
        const double q = springref[(size_t)e * nj + j];
        if (!std::isfinite(q)) return at + "qpos_spring is not finite";
        if (!hinge && q != m.qpos_spring[m.jnt_qposadr[j]]) return at + "qpos_spring of a slide, ball or free joint cannot change";
      }
    }
  }
  return std::string();
}

// cassie_batch_set_env_contact's check of every masked value, before anything changes: an empty reason, else the first refusal, naming the environment,
// the geom and the field.  Refused: a non-finite value; a solref in neither MuJoCo form -- standard (timeconst > 0, dampratio > 0) or direct (stiffness
// <= 0, damping <= 0); a solimp outside MuJoCo's documented ranges 0 < dmin < 1, 0 < dmax < 1, width >= 0, 0 < midpoint < 1, power >= 1 (inside them the
// impedance and R = (1 - imp) dA / imp stay finite); a negative solmix.  Geoms without a collision slot (geom_dev < 0) never make contact: their entries
// are not looked at.  solref [n][ngeom][2], solimp [n][ngeom][5], solmix [n][ngeom]; null parts are not checked (kept)
inline std::string env_contact_check(const HostModel &m, int n, const int *geom_dev, const double *solref, const double *solimp, const double *solmix,
                                     const unsigned char *mask) {
  static const char *imp_name[5] = {"dmin", "dmax", "width", "midpoint", "power"};
  const int ng = m.ngeom;
  auto geom = [&](int g) { return (size_t)g < m.names_geom.size() && !m.names_geom[g].empty() ? m.names_geom[g] : std::to_string(g); };   // unnamed: the index
  for (int e = 0; e < n; e++) {
    if (mask && !mask[e]) continue;
    for (int g = 0; g < ng; g++) {
      if (g >= 256 || geom_dev[g] < 0 || geom_dev[g] >= MGT) continue;
      const std::string at = "environment " + std::to_string(e) + ", geom " + geom(g) + ": ";
      if (solref) {
        const double *r = solref + ((size_t)e * ng + g) * 2;
        if (!std::isfinite(r[0]) || !std::isfinite(r[1])) return at + "geom_solref is not finite";
        if (!((r[0] > 0 && r[1] > 0) || (r[0] <= 0 && r[1] <= 0)))
          return at + "geom_solref must be standard (timeconst > 0, dampratio > 0) or direct (stiffness <= 0, damping <= 0), not mixed";
      }
      if (solimp) {
        const double *s = solimp + ((size_t)e * ng + g) * 5;
        for (int k = 0; k < 5; k++) if (!std::isfinite(s[k])) return at + "geom_solimp[" + std::to_string(k) + "] (" + imp_name[k] + ") is not finite";
        for (int k : {0, 1, 3}) if (!(s[k] > 0 && s[k] < 1)) return at + "geom_solimp[" + std::to_string(k) + "] (" + imp_name[k] + ") must be in (0, 1)";
        if (!(s[2] >= 0)) return at + "geom_solimp[2] (width) must be >= 0";
        if (!(s[4] >= 1)) return at + "geom_solimp[4] (power) must be >= 1";
      }
      if (solmix) {
        const double x = solmix[(size_t)e * ng + g];
        if (!std::isfinite(x)) return at + "geom_solmix is not finite";
        if (x < 0) return at + "geom_solmix must be >= 0";
      }
    }
  }
  return std::string();
}

// one row of a batch's frame table (FT_W) for body (kind 0) or site (kind 1) `name`; its id, or -1 with a reason for an unknown name or kind
template <typename real> int frame_table_row(const HostModel &m, const char *name, int kind, real *row, std::string &err) {
  for (int c = 0; c < FT_W; c++) row[c] = 0;
  row[FT_QUAT] = 1;
  if (!name) { err = "frame name missing"; return -1; }
  if (kind == 0) {
    const int b = m.body_id(name);
    if (b < 0) { err = std::string("unknown body ") + name; return -1; }
    row[FT_BODY] = (real)b;
    return b;
  }
  if (kind == 1) {
    const int s = m.site_id(name);
    if (s < 0) { err = std::string("unknown site ") + name; return -1; }
    row[FT_BODY] = (real)m.site_bodyid[s]; row[FT_KIND] = 1;
    for (int c = 0; c < 3; c++) row[FT_POS + c] = (real)m.site_pos[3 * s + c];
    for (int c = 0; c < 4; c++) row[FT_QUAT + c] = (real)m.site_quat[4 * s + c];
    return s;
  }
  err = "unknown frame kind " + std::to_string(kind) + " (0 body, 1 site)";
  return -1;
}

struct BuildInfo { int unsupported_pairs = 0; int collision_geoms = 0; int geom_dev[256]; BuildInfo() { for (int i = 0; i < 256; i++) geom_dev[i] = -1; } };   // geom_dev: host geom id -> collision geom slot of the device block

template <typename real>
bool build_dev_model(const HostModel &m, DevModel<real> &d, std::string &err, BuildInfo *info = nullptr) {
  std::memset(&d, 0, sizeof d);
  // at most one extra free body (cassie_tray_box.xml's cup): it must be the last joint / last 6 dofs, a child of the world, with its inertial
  // frame equal to its body frame; its dofs live beside the main tree's (one lane per main-tree dof)
  int xb = -1;
  for (int j = 0; j < m.njnt; j++) if (m.jnt_type[j] == JNT_FREE) {
    int b = m.jnt_bodyid[j];
    if (xb >= 0 || j != m.njnt - 1 || m.jnt_dofadr[j] != m.nv - 6 || m.body_parentid[b] != 0 || b != m.nbody - 1) { err = "only one free body, defined last and attached to the world, is supported"; return false; }
    if (std::fabs(m.body_ipos[3 * b]) + std::fabs(m.body_ipos[3 * b + 1]) + std::fabs(m.body_ipos[3 * b + 2]) > 1e-12 || std::fabs(m.body_iquat[4 * b]) < 1 - 1e-12) { err = "the free body's inertial frame must coincide with its body frame"; return false; }
    xb = b;
  }
  const int nvm = m.nv - (xb >= 0 ? 6 : 0);   // dofs of the main tree
  if (nvm > MV || m.nbody > MB || m.njnt > MJ || m.nM > NM_MAX + 21 || m.neq > ME || m.nu != MU) { err = "model exceeds the one-warp-per-env limits (main-tree nv<=32, nbody<=32, neq<=4, nu==10)"; return false; }
  { int root = -1;   // one moving tree; other bodies must be static (welded to the world, e.g. the 'floor' body of cassie_hfield.xml)
    for (int b = 1; b < m.nbody; b++) { if (m.body_weldid[b] == 0 || b == xb) continue; if (root < 0) root = m.body_rootid[b]; if (m.body_rootid[b] != root) { err = "a single articulated tree (plus at most one free body) is required"; return false; } } }
  if (m.nhfield > 1) { err = "at most one height field is supported"; return false; }
  if (m.nhfield == 1) { d.hf_nrow = m.hfield_nrow[0]; d.hf_ncol = m.hfield_ncol[0]; for (int k = 0; k < 4; k++) d.hf_size[k] = (real)m.hfield_size[k]; }
  d.nq = m.nq; d.nv = nvm; d.nbody = m.nbody; d.njnt = m.njnt; d.neq = m.neq; d.nu = m.nu; d.iterations = m.iterations;
  d.nM = 0; for (int i = 0; i < nvm; i++) d.nM = m.dof_Madr[i] + 1; { int last = nvm - 1, dep = 0; for (int k = m.dof_parentid[last]; k >= 0; k = m.dof_parentid[k]) dep++; d.nM = m.dof_Madr[last] + dep + 1; }
  d.xb = xb; d.qpos_w = xb >= 0 ? QPOS_W_XB : QPOS_W_MAIN; d.qvel_w = xb >= 0 ? QVEL_W_XB : QVEL_W_MAIN; d.ystride = xb >= 0 ? YSTRIDE_MAX : YSTRIDE_MAIN;
  if (xb >= 0) {
    d.xb_jnt = m.njnt - 1; d.xb_qadr = m.jnt_qposadr[d.xb_jnt]; d.xb_dadr = m.jnt_dofadr[d.xb_jnt];
    d.xb_mass = (real)m.body_mass[xb]; for (int k = 0; k < 3; k++) { d.xb_inertia[k] = (real)m.body_inertia[3 * xb + k]; d.xb_dsqi[k] = (real)(1.0 / std::sqrt(m.body_mass[xb])); d.xb_dsqi[3 + k] = (real)(1.0 / std::sqrt(m.body_inertia[3 * xb + k])); }
  }
  d.timestep = (real)m.timestep; d.tolerance = (real)m.tolerance; d.pgs_scale = (real)(1.0 / (m.meaninertia * std::max(1, m.nv)));
  d.nsub = (int)std::lround(5e-4 / m.timestep); if (d.nsub < 1) d.nsub = 1;
  d.euler_eps = (real)(4 * std::numeric_limits<real>::epsilon());
  d.force_zpath = std::getenv("CASSIE_B200_ZPATH") ? 1 : 0;   // test hook: force the reduction-based solver path used when nefc > 32
  double mass = 0; for (int b = 1; b < m.nbody; b++) if (b != xb) mass += m.body_mass[b];
  d.root_mass_inv = (real)(1.0 / mass);
  for (int k = 0; k < 3; k++) { d.gravity[k] = (real)m.gravity[k]; d.magnetic[k] = (real)m.magnetic[k]; }
  for (int k = 0; k < 44; k++) d.qpos0[k] = k < m.nq ? (real)m.qpos0[k] : real(0);
  if (std::fabs(m.impratio - 1.0) > 1e-12) { err = "impratio != 1 is not supported"; return false; }
  // bodies
  for (int b = 0; b < m.nbody; b++) {
    d.body_parent[b] = m.body_parentid[b]; d.body_depth[b] = b ? d.body_depth[m.body_parentid[b]] + 1 : 0;
    if (d.body_depth[b] > d.maxdepth) d.maxdepth = d.body_depth[b];
    d.body_jntadr[b] = m.body_jntadr[b]; d.body_jntnum[b] = m.body_jntnum[b];
    int p = b; while (p > 0 && m.body_dofnum[p] == 0) p = m.body_parentid[p];
    d.body_lastdof[b] = (p > 0 && b != xb) ? m.body_dofadr[p] + m.body_dofnum[p] - 1 : -1;
    uint32_t mask = 0; for (int k = d.body_lastdof[b]; k >= 0; k = m.dof_parentid[k]) mask |= 1u << k;
    d.body_dofmask[b] = mask;
    int end = b + 1; while (end < m.nbody) { int a = end; while (a > b) a = m.body_parentid[a]; if (a != b) break; end++; }
    d.body_subtree_end[b] = b == 0 ? m.nbody : end;
    double R[9]; detail::q2m_d(R, &m.body_iquat[4 * b]);
    for (int k = 0; k < 3; k++) { d.body_pos[b][k] = (real)m.body_pos[3 * b + k]; d.body_ipos[b][k] = (real)m.body_ipos[3 * b + k]; d.body_inertia[b][k] = (real)m.body_inertia[3 * b + k]; }
    for (int k = 0; k < 4; k++) d.body_quat[b][k] = (real)m.body_quat[4 * b + k];
    for (int k = 0; k < 9; k++) d.body_imat[b][k] = (real)R[k];
    d.body_mass[b] = (real)m.body_mass[b]; d.body_invw[b] = (real)m.body_invweight0[2 * b];
  }
  // joints
  for (int j = 0; j < m.njnt; j++) {
    d.jnt_type[j] = m.jnt_type[j]; d.jnt_qposadr[j] = m.jnt_qposadr[j]; d.jnt_dofadr[j] = m.jnt_dofadr[j]; d.jnt_body[j] = m.jnt_bodyid[j];
    d.jnt_limited[j] = (m.jnt_limited[j] && (m.jnt_type[j] == JNT_HINGE || m.jnt_type[j] == JNT_SLIDE)) ? 1 : 0;
    for (int k = 0; k < 3; k++) { d.jnt_pos[j][k] = (real)m.jnt_pos[3 * j + k]; d.jnt_axis[j][k] = (real)m.jnt_axis[3 * j + k]; }
    d.jnt_stiffness[j] = (real)m.jnt_stiffness[j]; d.jnt_range[j][0] = (real)m.jnt_range[2 * j]; d.jnt_range[j][1] = (real)m.jnt_range[2 * j + 1];
    d.jnt_qpos0[j] = (real)m.qpos0[m.jnt_qposadr[j]]; d.jnt_qspring[j] = (real)m.qpos_spring[m.jnt_qposadr[j]];
    for (int k = 0; k < 2; k++) d.jnt_solref[j][k] = (real)m.jnt_solref[2 * j + k];
    for (int k = 0; k < 5; k++) d.jnt_solimp[j][k] = (real)m.jnt_solimp[5 * j + k];
    if (m.jnt_margin[j] != 0) { err = "joint margins are not supported"; return false; }
    if (std::fabs(m.jnt_pos[3 * j]) + std::fabs(m.jnt_pos[3 * j + 1]) + std::fabs(m.jnt_pos[3 * j + 2]) > 0) d.any_jnt_pos = 1;
  }
  // joint arrangement the kinematics stage relies on: per body, slides first, then at most one hinge or ball joint
  for (int b = 1; b < m.nbody; b++) { int rot = 0; for (int jj = 0; jj < m.body_jntnum[b]; jj++) { int t = m.jnt_type[m.body_jntadr[b] + jj];
      if (t == JNT_SLIDE && rot) { err = "a slide joint after a rotational joint in the same body is not supported"; return false; } if (t == JNT_HINGE || t == JNT_BALL) rot++; }
    if (rot > 1) { err = "more than one rotational joint per body is not supported"; return false; } }
  // dofs
  d.ntri = 0;
  for (int i = 0; i < nvm; i++) {
    d.dof_body[i] = m.dof_bodyid[i]; d.dof_jnt[i] = m.dof_jntid[i]; d.dof_parent[i] = m.dof_parentid[i]; d.dof_Madr[i] = m.dof_Madr[i];
    d.dof_armature[i] = (real)m.dof_armature[i]; d.dof_damping[i] = (real)m.dof_damping[i]; d.dof_invweight0[i] = (real)m.dof_invweight0[i];
    uint32_t mask = 0; int depth = 0; for (int k = m.dof_parentid[i]; k >= 0; k = m.dof_parentid[k]) { mask |= 1u << k; depth++; }
    d.dof_ancmask[i] = mask; d.dof_depth[i] = depth; d.dof_Mrow[i] = m.dof_Madr[i] + depth;
    if (depth > 15) { err = "dof tree deeper than 15"; return false; }
    { int t = 1; for (int k = m.dof_parentid[i]; k >= 0; k = m.dof_parentid[k]) d.dof_anc[i][t++] = (unsigned char)k; }
    { int end = i + 1; while (end < nvm) { int a = end; while (a > i) a = m.dof_parentid[a]; if (a != i) break; end++; } d.dof_subtree_end[i] = end; }
    if (m.dof_damping[i] > 0) d.has_damping = 1;
    int j = m.dof_jntid[i];
    d.dof_cvelsrc[i] = (m.jnt_type[j] == JNT_BALL) ? m.dof_parentid[m.jnt_dofadr[j]] : m.dof_parentid[i];
  }
  for (int i = nvm - 1; i >= 0; i--) { int a = m.dof_Madr[i] + 1; for (int j = m.dof_parentid[i]; j >= 0; j = m.dof_parentid[j]) { if (d.ntri >= NTRI_MAX) { err = "too many factor entries"; return false; } d.tri[d.ntri++] = ((uint32_t)i << 24) | ((uint32_t)j << 16) | (uint32_t)a; a++; } }
  // two-level subtree sums: a body whose subtree has more than 13 bodies (the pelvis) takes its own term plus the finished sums of its direct children,
  // provided there are at most 4 of them, each carries a dof (its first dof's lane holds the child's sum in the bias stage) and none is large itself
  d.any_big = 0;
  for (int b = 0; b < MB; b++) d.body_kid_dofs[b] = 0;
  if (!std::getenv("CASSIE_B200_NOKIDS")) for (int b = 1; b < m.nbody; b++) {
    if (d.body_subtree_end[b] - b <= 13 || b == xb) continue;
    uint32_t packed = 0; int nk = 0; bool ok = true;
    for (int c = b + 1; c < d.body_subtree_end[b] && ok; c++) {
      if (m.body_parentid[c] != b) continue;
      if (m.body_dofnum[c] == 0 || nk == 4 || d.body_subtree_end[c] - c > 13 || m.body_dofadr[c] >= nvm) { ok = false; break; }
      packed |= (uint32_t)(m.body_dofadr[c] + 1) << (8 * nk++);
    }
    if (ok && nk > 0) { d.body_kid_dofs[b] = packed; d.any_big = 1; }
  }
  // balanced factorisation schedule (falls back to the per-ancestor loop when the table would not fit)
  { int total = 0; for (int k = 0; k < nvm; k++) total += d.dof_depth[k] * (d.dof_depth[k] + 1) / 2;
    d.nfac = 0;
    if (total <= NFAC_MAX) {
      int n = 0;
      for (int k = 0; k < nvm; k++) {
        d.fac_start[k] = n; int dk = d.dof_depth[k], kk = m.dof_Madr[k];
        for (int t = 1; t <= dk; t++) { int i = d.dof_anc[k][t], ia = m.dof_Madr[i]; for (int c = 0; c <= dk - t; c++) d.fac_pairs[n++] = ((uint32_t)t << 24) | ((uint32_t)(kk + t + c) << 12) | (uint32_t)(ia + c); }
      }
      d.fac_start[nvm] = n; d.nfac = n;
    } }
  // IMU site and its sensors
  int imu = m.site_id("imu");
  if (imu < 0) { err = "site 'imu' not found"; return false; }
  d.imu_body = m.site_bodyid[imu];
  { int n = 0; int pb = d.imu_body; while (pb > 0 && m.body_dofnum[pb] == 0) pb = m.body_parentid[pb]; for (int k = pb > 0 ? m.body_dofadr[pb] + m.body_dofnum[pb] - 1 : -1; k >= 0; k = m.dof_parentid[k]) n++;
    if (n > 7) { err = "the IMU body must have at most 7 dofs in its chain"; return false; } }
  double Rs[9]; detail::q2m_d(Rs, &m.site_quat[4 * imu]);
  for (int k = 0; k < 3; k++) d.imu_pos[k] = (real)m.site_pos[3 * imu + k];
  for (int k = 0; k < 4; k++) d.imu_quat[k] = (real)m.site_quat[4 * imu + k];
  for (int k = 0; k < 9; k++) d.imu_mat[k] = (real)Rs[k];
  // sensor layout must be the Cassie one: 16 encoders, framequat, gyro, accelerometer, magnetometer (model/cassie.xml:272-292)
  if (m.nsensor < 20) { err = "unexpected sensor layout"; return false; }
  for (int s = 0; s < 16; s++) {
    if (m.sensor_type[s] == SENS_ACTUATORPOS) { int a = m.sensor_objid[s], j = m.actuator_jntid[a]; d.enc_qposadr[s] = m.jnt_qposadr[j]; d.enc_scale[s] = (real)m.actuator_gear[a]; }
    else if (m.sensor_type[s] == SENS_JOINTPOS) { d.enc_qposadr[s] = m.jnt_qposadr[m.sensor_objid[s]]; d.enc_scale[s] = 1; }
    else { err = "unexpected sensor layout"; return false; }
    d.enc_bits[s] = (int)m.sensor_user[s];
  }
  if (m.sensor_type[16] != SENS_FRAMEQUAT || m.sensor_type[17] != SENS_GYRO || m.sensor_type[18] != SENS_ACCEL || m.sensor_type[19] != SENS_MAG) { err = "unexpected sensor layout"; return false; }
  d.gyro_cutoff = (real)m.sensor_cutoff[17]; d.accel_cutoff = (real)m.sensor_cutoff[18];
  // motors
  static const double torque_limit[5] = {140.63, 140.63, 216.16, 216.16, 45.14};  // elmo torqueLimit, src/cassiemujoco.c:687-691
  for (int i = 0; i < m.nu; i++) {
    int j = m.actuator_jntid[i];
    d.act_dof[i] = m.jnt_dofadr[j]; d.act_qposadr[i] = m.jnt_qposadr[j]; d.act_gear[i] = (real)m.actuator_gear[i];
    bool lim = m.actuator_ctrllimited[i] != 0;
    d.act_ctrl_lo[i] = lim ? (real)m.actuator_ctrlrange[2 * i] : -std::numeric_limits<real>::max();
    d.act_ctrl_hi[i] = lim ? (real)m.actuator_ctrlrange[2 * i + 1] : std::numeric_limits<real>::max();
    d.act_wmax[i] = (real)(m.actuator_user[i] * 2 * M_PI / 60); d.act_torque_limit[i] = (real)torque_limit[i % 5];
  }
  // equality
  for (int e = 0; e < m.neq; e++) {
    d.eq_b1[e] = m.eq_obj1id[e]; d.eq_b2[e] = m.eq_obj2id[e];
    for (int k = 0; k < 6; k++) d.eq_data[e][k] = (real)m.eq_data[6 * e + k];
    for (int k = 0; k < 2; k++) d.eq_solref[e][k] = (real)m.eq_solref[2 * e + k];
    for (int k = 0; k < 5; k++) d.eq_solimp[e][k] = (real)m.eq_solimp[5 * e + k];
  }
  // candidate pairs in MuJoCo's order: body pairs ascending, geoms in id order; then type-sorted.  Collision geoms get device ids: on moving
  // bodies 0 .. MG-1 (world pose recomputed every step), static ones (world body and bodies welded to it) MG .. MG+MGS-1 with their world pose here
  int gmap[256]; for (int g = 0; g < 256; g++) gmap[g] = -1;
  int n_dyn = 0, n_stat = 0, n_pc = 0;
  std::vector<double> reach(m.nbody, 0.0);   // bound on the distance of a body's origin from the root body's origin, whatever the joint angles
  { int root = -1; for (int b = 1; b < m.nbody; b++) if (m.body_weldid[b] != 0 && b != xb) { root = b; break; }
    d.root_body = root < 0 ? 0 : root;
    for (int b = 1; b < m.nbody; b++) if (m.body_weldid[b] != 0 && b != d.root_body && b != xb) {
      const double *bp = &m.body_pos[3 * b]; reach[b] = reach[m.body_parentid[b]] + std::sqrt(bp[0] * bp[0] + bp[1] * bp[1] + bp[2] * bp[2]); } }
  double robot_reach = 0;
  auto dev_geom = [&](int g) -> int {
    if (gmap[g] >= 0) return gmap[g];
    const int b = m.geom_bodyid[g]; const bool stat = m.body_weldid[b] == 0;
    if ((stat && n_stat >= MGS) || (!stat && n_dyn >= MG)) return -1;
    const int k = stat ? MG + n_stat++ : n_dyn++; gmap[g] = k; d.geom_body[k] = b; d.geom_type[k] = m.geom_type[g];
    double R[9]; detail::q2m_d(R, &m.geom_quat[4 * g]);
    for (int c = 0; c < 3; c++) d.geom_size[k][c] = (real)m.geom_size[3 * g + c];
    d.geom_rbound[k] = (real)m.geom_rbound[g];
    if (!stat) {
      for (int c = 0; c < 3; c++) d.geom_pos[k][c] = (real)m.geom_pos[3 * g + c];
      for (int c = 0; c < 9; c++) d.geom_mat[k][c] = (real)R[c];
      if (b != xb) { const double *gp = &m.geom_pos[3 * g]; robot_reach = std::max(robot_reach, reach[b] + std::sqrt(gp[0] * gp[0] + gp[1] * gp[1] + gp[2] * gp[2]) + m.geom_rbound[g]); }
    } else {   // world pose: compose the (constant) chain of static bodies
      double w[12]; static_geom_wpose(m, g, &m.geom_pos[3 * g], &m.geom_quat[4 * g], w);
      for (int c = 0; c < 12; c++) d.geom_wpose[k - MG][c] = (real)w[c];
    }
    return k;
  };
  int unsupported = 0;
  for (int b1 = 0; b1 < m.nbody; b1++) for (int b2 = b1 + 1; b2 < m.nbody; b2++) {
    int w1 = m.body_weldid[b1], w2 = m.body_weldid[b2];
    if (w1 == w2) continue;
    if (w1 && w2 && (m.body_weldid[m.body_parentid[w1]] == w2 || m.body_weldid[m.body_parentid[w2]] == w1)) continue;
    for (int ga = 0; ga < m.ngeom; ga++) if (m.geom_bodyid[ga] == b1) for (int gb = 0; gb < m.ngeom; gb++) if (m.geom_bodyid[gb] == b2) {
      int g1 = ga, g2 = gb; if (m.geom_type[g1] > m.geom_type[g2]) std::swap(g1, g2);
      if (!((m.geom_contype[g1] & m.geom_conaffinity[g2]) || (m.geom_contype[g2] & m.geom_conaffinity[g1]))) continue;
      int t1 = m.geom_type[g1], t2 = m.geom_type[g2], kind;
      if (t1 == GEOM_PLANE && t2 == GEOM_SPHERE) kind = PAIR_PLANE_SPHERE;
      else if (t1 == GEOM_PLANE && t2 == GEOM_CAPSULE) kind = PAIR_PLANE_CAPSULE;
      else if (t1 == GEOM_CAPSULE && t2 == GEOM_CAPSULE) kind = PAIR_CAPSULE_CAPSULE;
      else if (t1 == GEOM_HFIELD && t2 == GEOM_SPHERE) kind = PAIR_HFIELD_SPHERE;
      else if (t1 == GEOM_HFIELD && t2 == GEOM_CAPSULE) kind = PAIR_HFIELD_CAPSULE;
      else if (t1 == GEOM_PLANE && t2 == GEOM_BOX) kind = PAIR_PLANE_BOX;
      else if (t1 == GEOM_SPHERE && t2 == GEOM_BOX) kind = PAIR_SPHERE_BOX;
      else if (t1 == GEOM_CAPSULE && t2 == GEOM_BOX) kind = PAIR_CAPSULE_BOX;
      else if (t1 == GEOM_BOX && t2 == GEOM_BOX) kind = PAIR_BOX_BOX;
      else { unsupported++; continue; }
      if (d.npair >= MPAIR) { err = "too many candidate geom pairs"; return false; }
      if (t1 == GEOM_HFIELD) { const double *q = &m.geom_quat[4 * g1], *bq = &m.body_quat[4 * m.geom_bodyid[g1]];
        if (std::fabs(q[0]) < 1 - 1e-12 || std::fabs(bq[0]) < 1 - 1e-12 || m.body_weldid[m.geom_bodyid[g1]] != 0) { err = "the height field must be axis aligned and static"; return false; } }
      int k1 = dev_geom(g1), k2 = dev_geom(g2); if (k1 < 0 || k2 < 0) { err = "too many collision geoms (16 on moving bodies, 16 static)"; return false; }
      int fl = 0;
      { const int u1 = m.geom_user[g1], u2 = m.geom_user[g2], r1 = m.geom_group[g1], r2 = m.geom_group[g2];
        if (u1 == 1 || u2 == 1) fl |= 1;
        if (u1 == 2 && u2 == 2) fl |= 2;
        if (r1 == 1 && r2 >= 0 && r2 < 16) fl |= 256 << r2;
        if (r2 == 1 && r1 >= 0 && r1 < 16) fl |= 256 << r1; }
      // contact parameter mixing (mj_contactParam)
      double fr, solref[2], solimp[5]; int dim;
      if (m.geom_priority[g1] != m.geom_priority[g2]) {
        int g = m.geom_priority[g1] > m.geom_priority[g2] ? g1 : g2; dim = m.geom_condim[g]; fr = m.geom_friction[3 * g];
        for (int k = 0; k < 2; k++) solref[k] = m.geom_solref[2 * g + k]; for (int k = 0; k < 5; k++) solimp[k] = m.geom_solimp[5 * g + k];
      } else {
        dim = std::max(m.geom_condim[g1], m.geom_condim[g2]); fr = std::max(m.geom_friction[3 * g1], m.geom_friction[3 * g2]);
        double s1 = m.geom_solmix[g1], s2 = m.geom_solmix[g2], mix;
        if (s1 >= 1e-15 && s2 >= 1e-15) mix = s1 / (s1 + s2); else if (s1 < 1e-15 && s2 < 1e-15) mix = 0.5; else mix = s1 < 1e-15 ? 0.0 : 1.0;
        if (m.geom_solref[2 * g1] > 0 && m.geom_solref[2 * g2] > 0) for (int k = 0; k < 2; k++) solref[k] = mix * m.geom_solref[2 * g1 + k] + (1 - mix) * m.geom_solref[2 * g2 + k];
        else for (int k = 0; k < 2; k++) solref[k] = std::min(m.geom_solref[2 * g1 + k], m.geom_solref[2 * g2 + k]);
        for (int k = 0; k < 5; k++) solimp[k] = mix * m.geom_solimp[5 * g1 + k] + (1 - mix) * m.geom_solimp[5 * g2 + k];
      }
      if (dim != 1 && dim != 3) { err = "only condim 1 and 3 contacts are supported"; return false; }
      // the pair's parameter record: shared with every pair that mixes to the same values (all 135 box x robot pairs of cassie.xml share one)
      const real mu = (real)(fr / std::sqrt(m.impratio)), mg = (real)std::max(m.geom_margin[g1], m.geom_margin[g2]), gp = (real)std::max(m.geom_gap[g1], m.geom_gap[g2]);
      const int msrc = m.geom_priority[g1] == m.geom_priority[g2] ? 0 : (m.geom_priority[g1] > m.geom_priority[g2] ? 1 : 2);
      int pc = -1;
      for (int c = 0; c < n_pc && pc < 0; c++) {
        bool same = d.pc_condim[c] == dim && d.pc_mu_src[c] == msrc && d.pc_flags[c] == fl && d.pc_mu[c] == mu && d.pc_margin[c] == mg && d.pc_gap[c] == gp;
        for (int k = 0; k < 2; k++) same = same && d.pc_solref[c][k] == (real)solref[k];
        for (int k = 0; k < 5; k++) same = same && d.pc_solimp[c][k] == (real)solimp[k];
        if (same) pc = c;
      }
      if (pc < 0) {
        if (n_pc >= NPC) { err = "too many distinct contact-parameter records"; return false; }
        pc = n_pc++; d.pc_condim[pc] = dim; d.pc_mu_src[pc] = msrc; d.pc_flags[pc] = fl; d.pc_mu[pc] = mu; d.pc_margin[pc] = mg; d.pc_gap[pc] = gp;
        for (int k = 0; k < 2; k++) d.pc_solref[pc][k] = (real)solref[k];
        for (int k = 0; k < 5; k++) d.pc_solimp[pc][k] = (real)solimp[k];
      }
      d.pair_code[d.npair++] = (uint32_t)k1 | ((uint32_t)k2 << 6) | ((uint32_t)kind << 12) | ((uint32_t)pc << 16);
    }
  }
  d.ngeom = n_dyn; d.ngeom_static = n_stat; d.robot_reach = (real)(robot_reach * 1.05 + 0.05);
  { // two runs: pairs without a static box first, static-box pairs after them; each keeps MuJoCo's relative order and its rank in the full order
    std::vector<uint32_t> a, bx; d.static_box_mask = 0;
    for (int g = MG; g < MGT; g++) if (g - MG < n_stat && d.geom_type[g] == GEOM_BOX) d.static_box_mask |= 1 << (g - MG);
    for (int p = 0; p < d.npair; p++) {
      const uint32_t c = d.pair_code[p] | ((uint32_t)p << 20); const int g1 = pair_g1(c), g2 = pair_g2(c);
      const bool sb = (g1 >= MG && ((d.static_box_mask >> (g1 - MG)) & 1)) || (g2 >= MG && ((d.static_box_mask >> (g2 - MG)) & 1));
      (sb ? bx : a).push_back(c);
    }
    d.npair_a = (int)a.size();
    for (size_t i = 0; i < a.size(); i++) d.pair_code[i] = a[i];
    for (size_t i = 0; i < bx.size(); i++) d.pair_code[a.size() + i] = bx[i];
    if (d.npair > 255) { err = "too many candidate geom pairs"; return false; } }
  // mirror symmetry of the dof tree: a base chain 0..f-1, then two blocks of n dofs with identical relative structure hanging off dof f-1
  d.sym_on = 0;
  { const int nv2 = d.nv;
    for (int j = 2; j < nv2 && !d.sym_on; j++) {   // candidate root of the second leg: a dof whose parent p is not its predecessor
      const int p = m.dof_parentid[j]; if (p < 0 || p >= j - 1) continue;
      const int first = p + 1, n = j - first; if (n < 1 || j + n != nv2) continue;
      bool ok = m.dof_parentid[first] == p;
      for (int i = 1; i < first && ok; i++) ok = m.dof_parentid[i] == i - 1;                       // the base is a chain
      for (int r = 1; r < n && ok; r++) { const int pa = m.dof_parentid[first + r], pb = m.dof_parentid[j + r]; ok = pa >= first && pb == pa + n; }
      if (ok && first == 6 && n == 13 && !std::getenv("CASSIE_B200_NOSYM")) { d.sym_on = 1; d.sym_first = first; d.sym_n = n; d.sym_madr = m.dof_Madr[j] - m.dof_Madr[first]; }   // the unrolled products are written for the Cassie tree (6 + 13 + 13)
    }
    { static const int sigp[32] = CT19_SIG_PARENT, sigm[32] = CT19_SIG_MADR;   // the tree the straight-line row transform was generated for
      bool same = d.sym_on && nv2 == 32 && d.sym_first == 6 && d.sym_n == 13;
      for (int i = 0; i < 32 && same; i++) same = m.dof_parentid[i] == sigp[i] && m.dof_Madr[i] == sigm[i];
      d.spec19 = (same && !std::getenv("CASSIE_B200_NOSPEC")) ? 1 : 0; }
    for (int b = 0; b < m.nbody; b++) { int sd = 0; const int ld = d.body_lastdof[b];
      if (d.sym_on && ld >= d.sym_first) sd = ld < d.sym_first + d.sym_n ? 1 : 2;
      d.body_side[b] = (unsigned char)sd; }
  }
  // feet: bodies `left-foot` / `right-foot`; toe and heel points = the named sites when the model has them (model/cassie.xml:153-154,
  // 219-220), else the end points of the foot capsule (where cassie.xml puts those sites; cassie_hfield.xml / cassie_tray_box.xml lack them)
  d.foot_offset = (real)std::sqrt(0.01762 * 0.01762 + 0.05219 * 0.05219);   // src/cassiemujoco.c:1618
  { double mt = 0; for (int b = 1; b < m.nbody; b++) mt += m.body_mass[b]; d.total_mass_inv = (real)(mt > 0 ? 1.0 / mt : 0.0); }
  for (int s = 0; s < 2; s++) {
    const int fb = m.body_id(s ? "right-foot" : "left-foot"), toe = m.site_id(s ? "right-toe" : "left-toe"), heel = m.site_id(s ? "right-heel" : "left-heel");
    d.foot_body[s] = fb;
    for (int k = 0; k < 3; k++) { d.toe_local[s][k] = 0; d.heel_local[s][k] = 0; }
    if (fb < 0) continue;
    if (toe >= 0 && heel >= 0) { for (int k = 0; k < 3; k++) { d.toe_local[s][k] = (real)m.site_pos[3 * toe + k]; d.heel_local[s][k] = (real)m.site_pos[3 * heel + k]; } continue; }
    for (int g = 0; g < m.ngeom; g++) if (m.geom_bodyid[g] == fb && m.geom_type[g] == GEOM_CAPSULE && m.geom_contype[g]) {
      double R[9]; detail::q2m_d(R, &m.geom_quat[4 * g]);
      for (int k = 0; k < 3; k++) { d.toe_local[s][k] = (real)(m.geom_pos[3 * g + k] + R[3 * k + 2] * m.geom_size[3 * g + 1]); d.heel_local[s][k] = (real)(m.geom_pos[3 * g + k] - R[3 * k + 2] * m.geom_size[3 * g + 1]); }
    }
  }
  if (info) { info->unsupported_pairs = unsupported; info->collision_geoms = d.ngeom + d.ngeom_static; for (int g = 0; g < 256; g++) info->geom_dev[g] = gmap[g]; }
  return true;
}

// slot of entry i of a named per-env model array ("body_mass" [nbody], "body_ipos" [3 nbody], "dof_damping" [nv], "geom_friction" [3 ngeom],
// all in the host model's numbering = the reference's) inside the constant row, or -1 for entries the stepper does not use (damping of the
// extra free body, friction of non-colliding geoms, the torsional / rolling coefficients); width <- entries per env, -1 for an unknown name
inline int cenv_slot(const HostModel &hm, int nv_main, const int *geom_dev, const char *what, int i, int &width) {
  const std::string k(what);
  if (k == "body_mass") { width = hm.nbody; return CE_MASS + i; }
  if (k == "body_ipos") { width = 3 * hm.nbody; return CE_IPOS + i; }   // (the extra free body keeps its inertial frame: the setter rejects a change there)
  if (k == "dof_damping") { width = hm.nv; return i < nv_main ? CE_DAMP + i : -1; }
  if (k == "geom_friction") { width = 3 * hm.ngeom; const int g = i / 3; return (i % 3 == 0 && g < 256 && geom_dev[g] >= 0) ? CE_FRIC + geom_dev[g] : -1; }
  width = -1; return -1;
}

// default row of per-environment model constants (CE_* layout): the shared model's own values
template <typename real>
void init_cenv_row(const DevModel<real> &d, real *row, const HostModel &hm, const int *geom_dev) {
  for (int i = 0; i < CE_W; i++) row[i] = 0;
  for (int b = 0; b < d.nbody; b++) { row[CE_MASS + b] = d.body_mass[b]; for (int k = 0; k < 3; k++) row[CE_IPOS + 3 * b + k] = d.body_ipos[b][k]; row[CE_BINVW + b] = d.body_invw[b]; }
  for (int i = 0; i < d.nv; i++) { row[CE_DAMP + i] = d.dof_damping[i]; row[CE_DINVW + i] = d.dof_invweight0[i]; }
  for (int g = 0; g < hm.ngeom && g < 256; g++) if (geom_dev[g] >= 0 && geom_dev[g] < MGT) row[CE_FRIC + geom_dev[g]] = (real)hm.geom_friction[3 * g];   // collision geoms only, in the kernel's numbering
  row[CE_ROOT_MINV] = d.root_mass_inv; row[CE_TOT_MINV] = d.total_mass_inv; row[CE_PGS_SCALE] = d.pgs_scale;
}

// initial per-env rows: what cassie_sim_init leaves behind before its mj_forward (src/cassiemujoco.c:989-1027)
template <typename real>
void init_env_rows(const HostModel &m, real *qpos, real *qvel, real *qacc_ws, real *cst, int *dfilt, real *xfrc) {
  static const double qi[28] = {0.0045, 0, 0.4973, 0.9785, -0.0164, 0.01787, -0.2049, -1.1997, 0, 1.4267, 0, -1.5244, 1.5244, -1.5968,
                                -0.0045, 0, 0.4973, 0.9786, 0.00386, -0.01524, -0.2051, -1.1997, 0, 1.4267, 0, -1.5244, 1.5244, -1.5968};
  for (int i = 0; i < QPOS_W_XB; i++) qpos[i] = 0;
  for (int i = 0; i < m.nq; i++) qpos[i] = (real)m.qpos0[i];
  for (int i = 0; i < 28 && 7 + i < m.nq; i++) qpos[7 + i] = (real)qi[i];
  for (int i = 0; i < QVEL_W_XB; i++) { qvel[i] = 0; qacc_ws[i] = 0; }
  for (int i = 0; i < CST_W; i++) cst[i] = 0;
  cst[CS_STO] = 1;  // radio channel 8 = 1 (cassie_out_init, :724)
  for (int i = 0; i < DFILT_W; i++) dfilt[i] = 0;
  for (int i = 0; i < XFRC_W; i++) xfrc[i] = 0;
}

}  // namespace cassie
