// mjcf.cpp -- MJCF-subset compiler for the Cassie model family (host C++).
//
// Replaces, for this model family, what the reference gets from MuJoCo's mj_loadXML (src/cassiemujoco.c:851,930,997)
// followed by mj_setConst (:952): default-class inheritance (model/cassie.xml:14-35), xyaxes / fromto / fullinertia
// conversions, ref offsets, connect anchors at qpos0, dof tree tables, and the constants that feed constraint
// regularisation (dof_invweight0, body_invweight0, stat.meaninertia).  Supported: compiler(angle), option, default,
// asset/hfield, worldbody/body/inertial/joint/freejoint/geom/site/camera, equality/connect, actuator/motor, sensor/*.
// Everything else visual (meshes, materials, lights) is ignored -- it has no effect on the stepped state.  Cameras are recorded (pose in their body
// frame, fovy, mode) for the depth renderer; they do not touch the stepped state either.
#include "model.h"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <sstream>

namespace cassie {
namespace {

// ------------------------------------------------------------------ minimal XML reader
struct XNode {
  std::string tag;
  std::map<std::string, std::string> attr;
  std::vector<std::unique_ptr<XNode>> kids;
  const char *get(const char *k) const { auto it = attr.find(k); return it == attr.end() ? nullptr : it->second.c_str(); }
  bool has(const char *k) const { return attr.count(k) != 0; }
  const XNode *child(const char *t) const { for (auto &c : kids) if (c->tag == t) return c.get(); return nullptr; }
};

struct XParser {
  const std::string &s; size_t p = 0; std::string err;
  explicit XParser(const std::string &src) : s(src) {}
  void skip_ws() { while (p < s.size() && isspace((unsigned char)s[p])) p++; }
  bool starts(const char *t) const { return s.compare(p, strlen(t), t) == 0; }
  void skip_misc() {  // whitespace, comments, <?...?>, <!DOCTYPE ...>, text
    for (;;) {
      skip_ws();
      if (starts("<!--")) { size_t e = s.find("-->", p); p = e == std::string::npos ? s.size() : e + 3; }
      else if (starts("<?")) { size_t e = s.find("?>", p); p = e == std::string::npos ? s.size() : e + 2; }
      else if (starts("<!")) { size_t e = s.find('>', p); p = e == std::string::npos ? s.size() : e + 1; }
      else if (p < s.size() && s[p] != '<') { while (p < s.size() && s[p] != '<') p++; }
      else return;
    }
  }
  std::unique_ptr<XNode> element() {
    skip_misc();
    if (p >= s.size() || s[p] != '<') return nullptr;
    p++;
    auto n = std::make_unique<XNode>();
    while (p < s.size() && !isspace((unsigned char)s[p]) && s[p] != '>' && s[p] != '/') n->tag += s[p++];
    for (;;) {
      skip_ws();
      if (p >= s.size()) { err = "unexpected end inside <" + n->tag + ">"; return nullptr; }
      if (s[p] == '/') { p += 2; return n; }
      if (s[p] == '>') { p++; break; }
      std::string k;
      while (p < s.size() && !isspace((unsigned char)s[p]) && s[p] != '=') k += s[p++];
      skip_ws(); if (s[p] != '=') { err = "expected '=' after attribute " + k; return nullptr; }
      p++; skip_ws();
      char q = s[p++]; std::string v;
      while (p < s.size() && s[p] != q) v += s[p++];
      p++;
      n->attr[k] = v;
    }
    for (;;) {
      skip_misc();
      if (p >= s.size()) { err = "missing </" + n->tag + ">"; return nullptr; }
      if (starts("</")) { size_t e = s.find('>', p); p = e + 1; return n; }
      auto c = element();
      if (!c) return nullptr;
      n->kids.push_back(std::move(c));
    }
  }
};

// ------------------------------------------------------------------ small math
typedef std::vector<double> vec;
vec nums(const char *s) { vec v; if (!s) return v; std::istringstream is(s); double x; while (is >> x) v.push_back(x); return v; }
double norm3(const double *a) { return std::sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); }
void cross3(double *r, const double *a, const double *b) { double t[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]}; memcpy(r, t, sizeof t); }
void qmul(double *r, const double *a, const double *b) {
  double t[4] = {a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                 a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]};
  memcpy(r, t, sizeof t);
}
void q2m(double *m, const double *q) {
  double w = q[0], x = q[1], y = q[2], z = q[3];
  m[0] = w * w + x * x - y * y - z * z; m[1] = 2 * (x * y - w * z); m[2] = 2 * (x * z + w * y);
  m[3] = 2 * (x * y + w * z); m[4] = w * w - x * x + y * y - z * z; m[5] = 2 * (y * z - w * x);
  m[6] = 2 * (x * z - w * y); m[7] = 2 * (y * z + w * x); m[8] = w * w - x * x - y * y + z * z;
}
void mv3(double *r, const double *m, const double *v) { double t[3]; for (int i = 0; i < 3; i++) t[i] = m[3 * i] * v[0] + m[3 * i + 1] * v[1] + m[3 * i + 2] * v[2]; memcpy(r, t, sizeof t); }
void mtv3(double *r, const double *m, const double *v) { double t[3]; for (int i = 0; i < 3; i++) t[i] = m[i] * v[0] + m[3 + i] * v[1] + m[6 + i] * v[2]; memcpy(r, t, sizeof t); }
void m2q(double *q, const double *R) {  // R row-major
  double tr = R[0] + R[4] + R[8];
  if (tr > 0) { double s = std::sqrt(tr + 1.0) * 2; q[0] = 0.25 * s; q[1] = (R[7] - R[5]) / s; q[2] = (R[2] - R[6]) / s; q[3] = (R[3] - R[1]) / s; }
  else if (R[0] > R[4] && R[0] > R[8]) { double s = std::sqrt(1.0 + R[0] - R[4] - R[8]) * 2; q[0] = (R[7] - R[5]) / s; q[1] = 0.25 * s; q[2] = (R[1] + R[3]) / s; q[3] = (R[2] + R[6]) / s; }
  else if (R[4] > R[8]) { double s = std::sqrt(1.0 + R[4] - R[0] - R[8]) * 2; q[0] = (R[2] - R[6]) / s; q[1] = (R[1] + R[3]) / s; q[2] = 0.25 * s; q[3] = (R[5] + R[7]) / s; }
  else { double s = std::sqrt(1.0 + R[8] - R[0] - R[4]) * 2; q[0] = (R[3] - R[1]) / s; q[1] = (R[2] + R[6]) / s; q[2] = (R[5] + R[7]) / s; q[3] = 0.25 * s; }
  double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int i = 0; i < 4; i++) q[i] /= n;
  if (q[0] < 0) for (int i = 0; i < 4; i++) q[i] = -q[i];
}
void z2quat(double *q, const double *v_) {  // minimal rotation taking +z to v (fromto convention)
  double v[3] = {v_[0], v_[1], v_[2]}, n = norm3(v); for (int i = 0; i < 3; i++) v[i] /= n;
  double z[3] = {0, 0, 1}, ax[3]; cross3(ax, z, v); double s = norm3(ax);
  if (s < 1e-10) { ax[0] = 1; ax[1] = ax[2] = 0; } else for (int i = 0; i < 3; i++) ax[i] /= s;
  double ang = std::atan2(s, v[2]);
  q[0] = std::cos(ang / 2); for (int i = 0; i < 3; i++) q[1 + i] = ax[i] * std::sin(ang / 2);
}
// symmetric 3x3 eigen-decomposition by cyclic Jacobi; eigenvalues descending, V columns = eigenvectors, det(V) = +1
void eig3(const double A_[9], double w[3], double V[9]) {
  double A[9]; memcpy(A, A_, sizeof A);
  double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}; memcpy(V, I, sizeof I);
  for (int sweep = 0; sweep < 60; sweep++) {
    double off = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
    if (off < 1e-40) break;
    for (int p = 0; p < 3; p++) for (int q = p + 1; q < 3; q++) {
      double apq = A[3 * p + q]; if (std::fabs(apq) < 1e-300) continue;
      double theta = (A[3 * q + q] - A[3 * p + p]) / (2 * apq);
      double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1)), c = 1 / std::sqrt(t * t + 1), s = t * c;
      for (int k = 0; k < 3; k++) { double akp = A[3 * k + p], akq = A[3 * k + q]; A[3 * k + p] = c * akp - s * akq; A[3 * k + q] = s * akp + c * akq; }
      for (int k = 0; k < 3; k++) { double apk = A[3 * p + k], aqk = A[3 * q + k]; A[3 * p + k] = c * apk - s * aqk; A[3 * q + k] = s * apk + c * aqk; }
      for (int k = 0; k < 3; k++) { double vkp = V[3 * k + p], vkq = V[3 * k + q]; V[3 * k + p] = c * vkp - s * vkq; V[3 * k + q] = s * vkp + c * vkq; }
    }
  }
  int idx[3] = {0, 1, 2};
  for (int i = 0; i < 3; i++) for (int j = i + 1; j < 3; j++) if (A[4 * idx[j]] > A[4 * idx[i]]) std::swap(idx[i], idx[j]);
  double Vs[9];
  for (int c = 0; c < 3; c++) { w[c] = A[4 * idx[c]]; for (int r = 0; r < 3; r++) Vs[3 * r + c] = V[3 * r + idx[c]]; }
  double det = Vs[0] * (Vs[4] * Vs[8] - Vs[5] * Vs[7]) - Vs[1] * (Vs[3] * Vs[8] - Vs[5] * Vs[6]) + Vs[2] * (Vs[3] * Vs[7] - Vs[4] * Vs[6]);
  if (det < 0) for (int r = 0; r < 3; r++) Vs[3 * r + 2] = -Vs[3 * r + 2];
  memcpy(V, Vs, sizeof Vs);
}

typedef std::map<std::string, std::string> Attrs;
struct Defaults {
  std::map<std::string, std::map<std::string, Attrs>> cls;
  void walk(const XNode *n, const std::string *parent) {
    std::string name = n->get("class") ? n->get("class") : "main";
    std::map<std::string, Attrs> base;
    if (parent) base = cls[*parent];
    for (auto &c : n->kids) if (c->tag != "default") for (auto &kv : c->attr) base[c->tag][kv.first] = kv.second;
    cls[name] = base;
    for (auto &c : n->kids) if (c->tag == "default") walk(c.get(), &name);
  }
  Attrs get(const std::string &c, const char *tag) const {
    auto it = cls.find(c.empty() ? "main" : c);
    if (it == cls.end()) return Attrs();
    auto jt = it->second.find(tag);
    return jt == it->second.end() ? Attrs() : jt->second;
  }
};
Attrs merged(const Defaults &d, const std::string &cls, const char *tag, const XNode *n) { Attrs a = d.get(cls, tag); for (auto &kv : n->attr) a[kv.first] = kv.second; return a; }
const char *A(const Attrs &a, const char *k) { auto it = a.find(k); return it == a.end() ? nullptr : it->second.c_str(); }
double Ad(const Attrs &a, const char *k, double dflt) { const char *s = A(a, k); return s ? atof(s) : dflt; }
int Ai(const Attrs &a, const char *k, int dflt) { const char *s = A(a, k); return s ? atoi(s) : dflt; }
vec Av(const Attrs &a, const char *k, const char *dflt) { const char *s = A(a, k); return nums(s ? s : dflt); }
void orientation(const Attrs &a, double q[4]) {
  q[0] = 1; q[1] = q[2] = q[3] = 0;
  if (A(a, "quat")) { vec v = nums(A(a, "quat")); double n = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]); for (int i = 0; i < 4; i++) q[i] = v[i] / n; }
  else if (A(a, "xyaxes")) {
    vec v = nums(A(a, "xyaxes")); double x[3] = {v[0], v[1], v[2]}, y[3] = {v[3], v[4], v[5]}, z[3];
    double n = norm3(x); for (int i = 0; i < 3; i++) x[i] /= n;
    double d = x[0] * y[0] + x[1] * y[1] + x[2] * y[2]; for (int i = 0; i < 3; i++) y[i] -= x[i] * d;
    n = norm3(y); for (int i = 0; i < 3; i++) y[i] /= n;
    cross3(z, x, y);
    double R[9] = {x[0], y[0], z[0], x[1], y[1], z[1], x[2], y[2], z[2]}; m2q(q, R);
  } else if (A(a, "zaxis")) { vec v = nums(A(a, "zaxis")); z2quat(q, v.data()); }
}

struct Body { std::string name; int parent; double pos[3], quat[4], ipos[3], iquat[4], mass, inertia[3]; bool explicit_inertial; std::vector<int> joints, geoms; };
struct Joint { std::string name; int type, body, limited; double pos[3], axis[3], range[2], ref, springref, stiffness, damping, armature, margin, solref[2], solimp[5]; int qposadr, dofadr; };
struct Geom { std::string name; int type, body, contype, conaffinity, condim, priority, hfid, user, group; double pos[3], quat[4], size[3], rbound, friction[3], solmix, solref[2], solimp[5], margin, gap, mass; bool has_mass; };
struct Site { std::string name; int body; double pos[3], quat[4]; };
struct Camera { std::string name; int body, mode; double pos[3], quat[4], fovy; };
void solimp5(const Attrs &a, const char *key, double out[5]) { vec v = Av(a, key, "0.9 0.95 0.001"); double d[5] = {0.9, 0.95, 0.001, 0.5, 2}; for (size_t i = 0; i < v.size() && i < 5; i++) d[i] = v[i]; memcpy(out, d, sizeof d); }

struct Compiler {
  Defaults dfl; double ang = M_PI / 180;
  std::vector<Body> bodies; std::vector<Joint> joints; std::vector<Geom> geoms; std::vector<Site> sites; std::vector<Camera> cameras;
  std::vector<std::string> hf_names; std::vector<int> hf_nrow, hf_ncol; std::vector<double> hf_size;
  std::string err;

  bool add_geom(const XNode *g, int bid, const std::string &childclass) {
    std::string cls = g->get("class") ? g->get("class") : childclass;
    Attrs a = merged(dfl, cls, "geom", g);
    static const std::map<std::string, int> types = {{"plane", 0}, {"hfield", 1}, {"sphere", 2}, {"capsule", 3}, {"ellipsoid", 4}, {"cylinder", 5}, {"box", 6}, {"mesh", 7}};
    std::string ts = A(a, "type") ? A(a, "type") : "sphere";
    if (!types.count(ts)) { err = "unknown geom type " + ts; return false; }
    Geom G{}; G.type = types.at(ts); G.body = bid; G.name = A(a, "name") ? A(a, "name") : "";
    G.contype = Ai(a, "contype", 1); G.conaffinity = Ai(a, "conaffinity", 1);
    const bool mesh = G.type == GEOM_MESH;   // visual only: kept (zero size) so geom ids / per-geom arrays are numbered as in the reference's model
    if (mesh && (G.contype || G.conaffinity)) { err = "colliding mesh geoms are not supported"; return false; }
    if (G.type == 4 || G.type == 5) { err = "ellipsoid/cylinder geoms are not supported"; return false; }
    vec s = mesh ? vec() : Av(a, "size", ""), pos = Av(a, "pos", "0 0 0");
    memcpy(G.pos, pos.data(), sizeof G.pos); orientation(a, G.quat);
    if (!mesh && A(a, "fromto")) {
      vec ft = nums(A(a, "fromto")); double v[3] = {ft[0] - ft[3], ft[1] - ft[4], ft[2] - ft[5]};  // z axis points from 'to' to 'from'
      G.size[0] = s.size() ? s[0] : 0; G.size[1] = norm3(v) / 2;
      for (int i = 0; i < 3; i++) G.pos[i] = 0.5 * (ft[i] + ft[3 + i]);
      z2quat(G.quat, v);
    } else for (size_t i = 0; i < s.size() && i < 3; i++) G.size[i] = s[i];
    G.hfid = -1;
    if (G.type == GEOM_HFIELD) { const char *h = A(a, "hfield"); for (size_t i = 0; i < hf_names.size(); i++) if (h && hf_names[i] == h) G.hfid = (int)i; if (G.hfid < 0) { err = "unknown hfield"; return false; } }
    if (G.type == GEOM_SPHERE) G.rbound = G.size[0];
    else if (G.type == GEOM_CAPSULE) G.rbound = G.size[0] + G.size[1];
    else if (G.type == GEOM_BOX) G.rbound = norm3(G.size);
    else if (G.type == GEOM_HFIELD) { const double *h = &hf_size[4 * G.hfid]; double t[3] = {h[0], h[1], std::max(h[2], h[3])}; G.rbound = norm3(t); }
    else G.rbound = 0;
    G.condim = Ai(a, "condim", 3); G.priority = Ai(a, "priority", 0);
    { vec u = Av(a, "user", "0"); G.user = u.empty() ? 0 : (int)u[0]; G.group = Ai(a, "group", 0); }
    vec fr = Av(a, "friction", "1 0.005 0.0001"); double f3[3] = {1, 0.005, 0.0001}; for (size_t i = 0; i < fr.size() && i < 3; i++) f3[i] = fr[i]; memcpy(G.friction, f3, sizeof f3);
    G.solmix = Ad(a, "solmix", 1); vec sr = Av(a, "solref", "0.02 1"); G.solref[0] = sr[0]; G.solref[1] = sr[1]; solimp5(a, "solimp", G.solimp);
    G.margin = Ad(a, "margin", 0); G.gap = Ad(a, "gap", 0); G.has_mass = A(a, "mass") != nullptr; G.mass = Ad(a, "mass", 0);
    geoms.push_back(G); bodies[bid].geoms.push_back((int)geoms.size() - 1);
    return true;
  }

  bool walk(const XNode *node, int parent, const std::string &childclass) {
    for (auto &c : node->kids) if (c->tag == "geom" && !add_geom(c.get(), parent, childclass)) return false;
    for (auto &c : node->kids) if (c->tag == "site") {
      Attrs a = merged(dfl, c->get("class") ? c->get("class") : childclass, "site", c.get());
      Site S{}; S.name = A(a, "name") ? A(a, "name") : ""; S.body = parent;
      if (A(a, "fromto")) { vec ft = nums(A(a, "fromto")); double v[3] = {ft[0] - ft[3], ft[1] - ft[4], ft[2] - ft[5]}; for (int i = 0; i < 3; i++) S.pos[i] = 0.5 * (ft[i] + ft[3 + i]); z2quat(S.quat, v); }
      else { vec p = Av(a, "pos", "0 0 0"); memcpy(S.pos, p.data(), sizeof S.pos); orientation(a, S.quat); }
      sites.push_back(S);
    }
    for (auto &c : node->kids) if (c->tag == "camera") {   // numbered in document order, like MuJoCo's
      static const std::map<std::string, int> modes = {{"fixed", CAM_FIXED}, {"track", CAM_TRACK}, {"trackcom", CAM_TRACKCOM}, {"targetbody", CAM_TARGETBODY}, {"targetbodycom", CAM_TARGETBODYCOM}};
      Attrs a = merged(dfl, c->get("class") ? c->get("class") : childclass, "camera", c.get());
      Camera K{}; K.name = A(a, "name") ? A(a, "name") : ""; K.body = parent; K.fovy = Ad(a, "fovy", 45);
      const std::string ms = A(a, "mode") ? A(a, "mode") : "fixed";
      if (!modes.count(ms)) { err = "unknown camera mode " + ms; return false; }
      K.mode = modes.at(ms);
      vec p = Av(a, "pos", "0 0 0"); memcpy(K.pos, p.data(), sizeof K.pos); orientation(a, K.quat);
      cameras.push_back(K);
    }
    for (auto &c : node->kids) if (c->tag == "body") {
      const XNode *b = c.get(); int bid = (int)bodies.size();
      std::string cc = b->get("childclass") ? b->get("childclass") : childclass;
      Body B{}; B.name = b->get("name") ? b->get("name") : ""; B.parent = parent;
      vec p = nums(b->get("pos") ? b->get("pos") : "0 0 0"); memcpy(B.pos, p.data(), sizeof B.pos);
      orientation(b->attr, B.quat); B.iquat[0] = 1;
      if (const XNode *in = b->child("inertial")) {
        B.explicit_inertial = true; vec ip = nums(in->get("pos") ? in->get("pos") : "0 0 0"); ip.resize(3, 0.0); memcpy(B.ipos, ip.data(), sizeof B.ipos); B.mass = in->get("mass") ? atof(in->get("mass")) : 0.0;
        if (in->has("fullinertia")) {
          vec f = nums(in->get("fullinertia")); double I[9] = {f[0], f[3], f[4], f[3], f[1], f[5], f[4], f[5], f[2]}, V[9];
          eig3(I, B.inertia, V); m2q(B.iquat, V);
        } else { vec d = nums(in->get("diaginertia")); for (size_t i = 0; i < 3; i++) B.inertia[i] = i < d.size() ? d[i] : 0.0;   // a point mass (model/cassie_mass.xml:88) carries no inertia of its own
                 orientation(in->attr, B.iquat); }
      }
      bodies.push_back(B);
      for (auto &jn : b->kids) if (jn->tag == "joint" || jn->tag == "freejoint") {
        Attrs a = merged(dfl, jn->get("class") ? jn->get("class") : cc, "joint", jn.get());
        std::string ts = jn->tag == "freejoint" ? "free" : (A(a, "type") ? A(a, "type") : "hinge");
        Joint J{}; J.name = A(a, "name") ? A(a, "name") : ""; J.body = bid;
        J.type = ts == "free" ? JNT_FREE : ts == "ball" ? JNT_BALL : ts == "slide" ? JNT_SLIDE : JNT_HINGE;
        J.limited = (A(a, "limited") && !strcmp(A(a, "limited"), "true") && J.type != JNT_FREE) ? 1 : 0;
        vec r = Av(a, "range", "0 0"); J.range[0] = r[0]; J.range[1] = r[1]; J.ref = Ad(a, "ref", 0); J.springref = Ad(a, "springref", 0);
        if (J.type == JNT_HINGE || J.type == JNT_BALL) { J.range[0] *= ang; J.range[1] *= ang; }
        if (J.type == JNT_HINGE) { J.ref *= ang; J.springref *= ang; }
        vec ax = Av(a, "axis", "0 0 1"), jp = Av(a, "pos", "0 0 0"); double n = norm3(ax.data());
        for (int i = 0; i < 3; i++) { J.axis[i] = ax[i] / n; J.pos[i] = jp[i]; }
        J.stiffness = Ad(a, "stiffness", 0); J.damping = Ad(a, "damping", 0); J.armature = Ad(a, "armature", 0); J.margin = Ad(a, "margin", 0);
        vec sr = Av(a, "solreflimit", "0.02 1"); J.solref[0] = sr[0]; J.solref[1] = sr[1]; solimp5(a, "solimplimit", J.solimp);
        joints.push_back(J); bodies[bid].joints.push_back((int)joints.size() - 1);
      }
      if (!walk(b, bid, cc)) return false;
    }
    return true;
  }
};

// ---- kinematics at an arbitrary qpos on the intermediate representation (used for anchors and set_const)
struct Kin { std::vector<double> xpos, xquat, xmat, xipos, xanchor, xaxis; };
void host_fk(const HostModel &m, const double *qpos, Kin &k) {
  int nb = m.nbody, nj = m.njnt;
  k.xpos.assign(3 * nb, 0); k.xquat.assign(4 * nb, 0); k.xmat.assign(9 * nb, 0); k.xipos.assign(3 * nb, 0); k.xanchor.assign(3 * nj, 0); k.xaxis.assign(3 * nj, 0);
  k.xquat[0] = 1; q2m(&k.xmat[0], &k.xquat[0]);
  for (int b = 1; b < nb; b++) {
    double pos[3], quat[4]; int jadr = m.body_jntadr[b];
    if (m.body_jntnum[b] == 1 && m.jnt_type[jadr] == JNT_FREE) {
      int qa = m.jnt_qposadr[jadr]; memcpy(pos, qpos + qa, sizeof pos); memcpy(quat, qpos + qa + 3, sizeof quat);
      double n = std::sqrt(quat[0] * quat[0] + quat[1] * quat[1] + quat[2] * quat[2] + quat[3] * quat[3]); for (int i = 0; i < 4; i++) quat[i] /= n;
      memcpy(&k.xanchor[3 * jadr], pos, sizeof pos); memcpy(&k.xaxis[3 * jadr], &m.jnt_axis[3 * jadr], sizeof pos);
    } else {
      int p = m.body_parentid[b]; double v[3]; mv3(v, &k.xmat[9 * p], &m.body_pos[3 * b]);
      for (int i = 0; i < 3; i++) pos[i] = k.xpos[3 * p + i] + v[i];
      qmul(quat, &k.xquat[4 * p], &m.body_quat[4 * b]);
      for (int jj = 0; jj < m.body_jntnum[b]; jj++) {
        int j = jadr + jj, qa = m.jnt_qposadr[j]; double R[9]; q2m(R, quat);
        mv3(&k.xaxis[3 * j], R, &m.jnt_axis[3 * j]); mv3(v, R, &m.jnt_pos[3 * j]);
        for (int i = 0; i < 3; i++) k.xanchor[3 * j + i] = pos[i] + v[i];
        if (m.jnt_type[j] == JNT_SLIDE) { for (int i = 0; i < 3; i++) pos[i] += k.xaxis[3 * j + i] * (qpos[qa] - m.qpos0[qa]); }
        else {
          double ql[4];
          if (m.jnt_type[j] == JNT_BALL) { memcpy(ql, qpos + qa, sizeof ql); double n = std::sqrt(ql[0] * ql[0] + ql[1] * ql[1] + ql[2] * ql[2] + ql[3] * ql[3]); for (int i = 0; i < 4; i++) ql[i] /= n; }
          else { double a = qpos[qa] - m.qpos0[qa]; ql[0] = std::cos(a / 2); for (int i = 0; i < 3; i++) ql[1 + i] = m.jnt_axis[3 * j + i] * std::sin(a / 2); }
          qmul(quat, quat, ql); q2m(R, quat); mv3(v, R, &m.jnt_pos[3 * j]);
          for (int i = 0; i < 3; i++) pos[i] = k.xanchor[3 * j + i] - v[i];
        }
      }
    }
    double n = std::sqrt(quat[0] * quat[0] + quat[1] * quat[1] + quat[2] * quat[2] + quat[3] * quat[3]);
    for (int i = 0; i < 4; i++) k.xquat[4 * b + i] = quat[i] / n;
    memcpy(&k.xpos[3 * b], pos, sizeof pos); q2m(&k.xmat[9 * b], &k.xquat[4 * b]);
    double v[3]; mv3(v, &k.xmat[9 * b], &m.body_ipos[3 * b]); for (int i = 0; i < 3; i++) k.xipos[3 * b + i] = pos[i] + v[i];
  }
}
// dense 3 x nv translational / rotational Jacobians of a world point attached to `body`
void host_jac(const HostModel &m, const Kin &k, const double *point, int body, std::vector<double> &jp, std::vector<double> &jr) {
  int nv = m.nv; jp.assign(3 * nv, 0); jr.assign(3 * nv, 0);
  for (int b = body; b > 0; b = m.body_parentid[b]) for (int jj = m.body_jntnum[b] - 1; jj >= 0; jj--) {
    int j = m.body_jntadr[b] + jj, d = m.jnt_dofadr[j]; const double *ax = &k.xaxis[3 * j], *an = &k.xanchor[3 * j];
    double off[3] = {point[0] - an[0], point[1] - an[1], point[2] - an[2]}, c[3];
    if (m.jnt_type[j] == JNT_SLIDE) for (int i = 0; i < 3; i++) jp[i * nv + d] = ax[i];
    else if (m.jnt_type[j] == JNT_HINGE) { cross3(c, ax, off); for (int i = 0; i < 3; i++) { jr[i * nv + d] = ax[i]; jp[i * nv + d] = c[i]; } }
    else {
      int d0 = d;
      if (m.jnt_type[j] == JNT_FREE) { for (int i = 0; i < 3; i++) jp[i * nv + d + i] = 1; d0 = d + 3; for (int i = 0; i < 3; i++) off[i] = point[i] - k.xpos[3 * b + i]; }
      for (int kk = 0; kk < 3; kk++) { double a[3] = {k.xmat[9 * b + kk], k.xmat[9 * b + 3 + kk], k.xmat[9 * b + 6 + kk]}; cross3(c, a, off); for (int i = 0; i < 3; i++) { jr[i * nv + d0 + kk] = a[i]; jp[i * nv + d0 + kk] = c[i]; } }
    }
  }
}
// in-place inverse of a symmetric positive definite n x n matrix (Gauss-Jordan with partial pivoting)
void invert(std::vector<double> &Amat, int n) {
  std::vector<double> B(n * n, 0); for (int i = 0; i < n; i++) B[i * n + i] = 1;
  for (int c = 0; c < n; c++) {
    int piv = c; for (int r = c + 1; r < n; r++) if (std::fabs(Amat[r * n + c]) > std::fabs(Amat[piv * n + c])) piv = r;
    if (piv != c) for (int k = 0; k < n; k++) { std::swap(Amat[c * n + k], Amat[piv * n + k]); std::swap(B[c * n + k], B[piv * n + k]); }
    double d = Amat[c * n + c]; for (int k = 0; k < n; k++) { Amat[c * n + k] /= d; B[c * n + k] /= d; }
    for (int r = 0; r < n; r++) if (r != c) { double f = Amat[r * n + c]; if (f != 0) for (int k = 0; k < n; k++) { Amat[r * n + k] -= f * Amat[c * n + k]; B[r * n + k] -= f * B[c * n + k]; } }
  }
  Amat = B;
}
}  // namespace

void set_const(HostModel &m) {
  int nv = m.nv, nb = m.nbody; Kin k; host_fk(m, m.qpos0.data(), k);
  std::vector<double> M(nv * nv, 0), jp, jr;
  for (int d = 0; d < nv; d++) M[d * nv + d] = m.dof_armature[d];
  for (int b = 1; b < nb; b++) {
    host_jac(m, k, &k.xipos[3 * b], b, jp, jr);
    double Ri[9], R[9], Iw[9]; q2m(Ri, &m.body_iquat[4 * b]);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double s = 0; for (int t = 0; t < 3; t++) s += k.xmat[9 * b + 3 * i + t] * Ri[3 * t + j]; R[3 * i + j] = s; }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double s = 0; for (int t = 0; t < 3; t++) s += R[3 * i + t] * m.body_inertia[3 * b + t] * R[3 * j + t]; Iw[3 * i + j] = s; }
    for (int a = 0; a < nv; a++) for (int c = 0; c < nv; c++) {
      double s = 0;
      for (int i = 0; i < 3; i++) { s += m.body_mass[b] * jp[i * nv + a] * jp[i * nv + c]; for (int j = 0; j < 3; j++) s += jr[i * nv + a] * Iw[3 * i + j] * jr[j * nv + c]; }
      M[a * nv + c] += s;
    }
  }
  double tr = 0; for (int d = 0; d < nv; d++) tr += M[d * nv + d];
  m.meaninertia = tr / nv;
  std::vector<double> Minv = M; invert(Minv, nv);
  m.body_invweight0.assign(2 * nb, 0);
  for (int b = 1; b < nb; b++) {
    if (m.body_weldid[b] == 0) continue;
    host_jac(m, k, &k.xipos[3 * b], b, jp, jr);
    for (int which = 0; which < 2; which++) {
      const std::vector<double> &J = which ? jr : jp; double s = 0;
      for (int i = 0; i < 3; i++) for (int a = 0; a < nv; a++) if (J[i * nv + a] != 0) for (int c = 0; c < nv; c++) s += J[i * nv + a] * Minv[a * nv + c] * J[i * nv + c];
      m.body_invweight0[2 * b + which] = s / 3;
    }
  }
  m.dof_invweight0.assign(nv, 0);
  for (int j = 0; j < m.njnt; j++) {
    int d = m.jnt_dofadr[j];
    if (m.jnt_type[j] == JNT_SLIDE || m.jnt_type[j] == JNT_HINGE) m.dof_invweight0[d] = Minv[d * nv + d];
    else {
      int d0 = d;
      if (m.jnt_type[j] == JNT_FREE) { double s = (Minv[d * nv + d] + Minv[(d + 1) * nv + d + 1] + Minv[(d + 2) * nv + d + 2]) / 3; for (int i = 0; i < 3; i++) m.dof_invweight0[d + i] = s; d0 = d + 3; }
      double s = (Minv[d0 * nv + d0] + Minv[(d0 + 1) * nv + d0 + 1] + Minv[(d0 + 2) * nv + d0 + 2]) / 3;
      for (int i = 0; i < 3; i++) m.dof_invweight0[d0 + i] = s;
    }
  }
  m.body_subtreemass = m.body_mass;
  for (int b = nb - 1; b > 0; b--) m.body_subtreemass[m.body_parentid[b]] += m.body_subtreemass[b];
}

bool compile_mjcf(const std::string &xml_path, HostModel &m, std::string &err) {
  std::ifstream f(xml_path);
  if (!f) { err = "cannot open " + xml_path; return false; }
  std::stringstream ss; ss << f.rdbuf(); std::string src = ss.str();
  XParser xp(src); auto root = xp.element();
  if (!root || root->tag != "mujoco") { err = "XML parse error: " + xp.err; return false; }
  Compiler C;
  if (const XNode *c = root->child("compiler")) if (c->get("angle") && !strcmp(c->get("angle"), "radian")) C.ang = 1.0;
  if (const XNode *d = root->child("default")) C.dfl.walk(d, nullptr);
  m = HostModel();
  if (const XNode *o = root->child("option")) {
    if (o->get("timestep")) m.timestep = atof(o->get("timestep"));
    if (o->get("gravity")) { vec g = nums(o->get("gravity")); memcpy(m.gravity, g.data(), sizeof m.gravity); }
    if (o->get("magnetic")) { vec g = nums(o->get("magnetic")); memcpy(m.magnetic, g.data(), sizeof m.magnetic); }
    if (o->get("iterations")) m.iterations = atoi(o->get("iterations"));
    if (o->get("tolerance")) m.tolerance = atof(o->get("tolerance"));
    if (o->get("impratio")) m.impratio = atof(o->get("impratio"));
    if (!o->get("solver") || strcmp(o->get("solver"), "PGS")) { err = "only solver='PGS' is implemented (all Cassie models use it)"; return false; }
    if (o->get("cone") && strcmp(o->get("cone"), "pyramidal")) { err = "only pyramidal friction cones are implemented"; return false; }
  }
  if (const XNode *as = root->child("asset")) for (auto &h : as->kids) if (h->tag == "hfield") {
    if (!h->get("nrow") || !h->get("ncol")) { err = "hfield needs nrow/ncol (file-based hfields are not supported)"; return false; }
    C.hf_names.push_back(h->get("name") ? h->get("name") : ""); C.hf_nrow.push_back(atoi(h->get("nrow"))); C.hf_ncol.push_back(atoi(h->get("ncol")));
    vec s = nums(h->get("size")); for (int i = 0; i < 4; i++) C.hf_size.push_back(s[i]);
  }
  Body W{}; W.name = "world"; W.quat[0] = W.iquat[0] = 1; W.explicit_inertial = true; C.bodies.push_back(W);
  const XNode *wb = root->child("worldbody");
  if (!wb) { err = "no <worldbody>"; return false; }
  if (!C.walk(wb, 0, "")) { err = C.err; return false; }
  // inertia inferred from geoms (inertiafromgeom='auto'): boxes only
  for (size_t b = 1; b < C.bodies.size(); b++) if (!C.bodies[b].explicit_inertial) {
    Body &B = C.bodies[b]; double tot = 0, com[3] = {0, 0, 0};
    { bool is_static = B.joints.empty(); for (int a = B.parent; a > 0 && is_static; a = C.bodies[a].parent) if (!C.bodies[a].joints.empty()) is_static = false;
      if (is_static) { B.mass = 0; B.inertia[0] = B.inertia[1] = B.inertia[2] = 0; B.ipos[0] = B.ipos[1] = B.ipos[2] = 0; B.iquat[0] = 1; B.iquat[1] = B.iquat[2] = B.iquat[3] = 0; continue; } }
    for (int gi : B.geoms) { Geom &G = C.geoms[gi]; if (G.type != GEOM_BOX) { err = "geom-inferred inertia implemented for boxes only"; return false; }
      if (!G.has_mass) G.mass = 1000.0 * 8 * G.size[0] * G.size[1] * G.size[2]; tot += G.mass; for (int i = 0; i < 3; i++) com[i] += G.mass * G.pos[i]; }
    if (tot <= 0) { err = "body '" + B.name + "' has no inertia"; return false; }
    for (int i = 0; i < 3; i++) com[i] /= tot;
    double I[9] = {0};
    for (int gi : B.geoms) {
      Geom &G = C.geoms[gi]; double R[9]; q2m(R, G.quat);
      double bi[3] = {G.mass / 3 * (G.size[1] * G.size[1] + G.size[2] * G.size[2]), G.mass / 3 * (G.size[0] * G.size[0] + G.size[2] * G.size[2]), G.mass / 3 * (G.size[0] * G.size[0] + G.size[1] * G.size[1])};
      double d[3] = {G.pos[0] - com[0], G.pos[1] - com[1], G.pos[2] - com[2]}, dd = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
      for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double s = 0; for (int t = 0; t < 3; t++) s += R[3 * i + t] * bi[t] * R[3 * j + t]; I[3 * i + j] += s + G.mass * ((i == j ? dd : 0) - d[i] * d[j]); }
    }
    double V[9]; eig3(I, B.inertia, V); m2q(B.iquat, V); B.mass = tot; memcpy(B.ipos, com, sizeof com);
  }
  // ---- flatten
  int nb = (int)C.bodies.size(), nj = (int)C.joints.size(), ng = (int)C.geoms.size();
  int qa = 0, da = 0;
  for (auto &J : C.joints) { J.qposadr = qa; J.dofadr = da; qa += J.type == JNT_FREE ? 7 : J.type == JNT_BALL ? 4 : 1; da += J.type == JNT_FREE ? 6 : J.type == JNT_BALL ? 3 : 1; }
  m.nq = qa; m.nv = da; m.nbody = nb; m.njnt = nj; m.ngeom = ng; m.nsite = (int)C.sites.size();
  m.body_parentid.resize(nb); m.body_rootid.assign(nb, 0); m.body_weldid.assign(nb, 0); m.body_jntnum.resize(nb); m.body_jntadr.resize(nb);
  m.body_dofnum.assign(nb, 0); m.body_dofadr.assign(nb, -1);
  for (int b = 0; b < nb; b++) {
    const Body &B = C.bodies[b]; m.body_parentid[b] = B.parent; m.body_jntnum[b] = (int)B.joints.size(); m.body_jntadr[b] = B.joints.empty() ? -1 : B.joints[0];
    m.body_pos.insert(m.body_pos.end(), B.pos, B.pos + 3); m.body_quat.insert(m.body_quat.end(), B.quat, B.quat + 4);
    m.body_ipos.insert(m.body_ipos.end(), B.ipos, B.ipos + 3); m.body_iquat.insert(m.body_iquat.end(), B.iquat, B.iquat + 4);
    m.body_mass.push_back(B.mass); m.body_inertia.insert(m.body_inertia.end(), B.inertia, B.inertia + 3); m.names_body.push_back(B.name);
    if (b) { m.body_rootid[b] = B.parent == 0 ? b : m.body_rootid[B.parent]; m.body_weldid[b] = B.joints.empty() ? m.body_weldid[B.parent] : b; }
  }
  m.dof_bodyid.resize(m.nv); m.dof_jntid.resize(m.nv); m.dof_parentid.assign(m.nv, -1); m.dof_Madr.resize(m.nv); m.dof_armature.resize(m.nv); m.dof_damping.resize(m.nv);
  m.qpos0.assign(m.nq, 0); m.qpos_spring.assign(m.nq, 0);
  for (int j = 0; j < nj; j++) {
    const Joint &J = C.joints[j]; int n = J.type == JNT_FREE ? 6 : J.type == JNT_BALL ? 3 : 1;
    m.jnt_type.push_back(J.type); m.jnt_qposadr.push_back(J.qposadr); m.jnt_dofadr.push_back(J.dofadr); m.jnt_bodyid.push_back(J.body); m.jnt_limited.push_back(J.limited);
    m.jnt_pos.insert(m.jnt_pos.end(), J.pos, J.pos + 3); m.jnt_axis.insert(m.jnt_axis.end(), J.axis, J.axis + 3); m.jnt_stiffness.push_back(J.stiffness);
    m.jnt_range.insert(m.jnt_range.end(), J.range, J.range + 2); m.jnt_margin.push_back(J.margin); m.jnt_solref.insert(m.jnt_solref.end(), J.solref, J.solref + 2);
    m.jnt_solimp.insert(m.jnt_solimp.end(), J.solimp, J.solimp + 5); m.names_joint.push_back(J.name);
    if (m.body_dofadr[J.body] < 0) m.body_dofadr[J.body] = J.dofadr;
    m.body_dofnum[J.body] += n;
    for (int k = 0; k < n; k++) { m.dof_bodyid[J.dofadr + k] = J.body; m.dof_jntid[J.dofadr + k] = j; m.dof_armature[J.dofadr + k] = J.armature; m.dof_damping[J.dofadr + k] = J.damping; }
    if (J.type == JNT_FREE) { const Body &B = C.bodies[J.body]; for (int i = 0; i < 3; i++) m.qpos0[J.qposadr + i] = B.pos[i]; for (int i = 0; i < 4; i++) m.qpos0[J.qposadr + 3 + i] = B.quat[i]; for (int i = 0; i < 7; i++) m.qpos_spring[J.qposadr + i] = m.qpos0[J.qposadr + i]; }
    else if (J.type == JNT_BALL) { m.qpos0[J.qposadr] = 1; m.qpos_spring[J.qposadr] = 1; }
    else { m.qpos0[J.qposadr] = J.ref; m.qpos_spring[J.qposadr] = J.springref; }
  }
  for (int d = 0; d < m.nv; d++) {
    int b = m.dof_bodyid[d];
    if (d > m.body_dofadr[b]) m.dof_parentid[d] = d - 1;
    else { int p = m.body_parentid[b]; while (p > 0 && m.body_dofnum[p] == 0) p = m.body_parentid[p]; m.dof_parentid[d] = p > 0 ? m.body_dofadr[p] + m.body_dofnum[p] - 1 : -1; }
  }
  m.nM = 0; for (int d = 0; d < m.nv; d++) { m.dof_Madr[d] = m.nM; for (int k = d; k >= 0; k = m.dof_parentid[k]) m.nM++; }
  for (const Geom &G : C.geoms) {
    m.geom_type.push_back(G.type); m.geom_bodyid.push_back(G.body); m.geom_contype.push_back(G.contype); m.geom_conaffinity.push_back(G.conaffinity);
    m.geom_condim.push_back(G.condim); m.geom_priority.push_back(G.priority); m.geom_hfid.push_back(G.hfid); m.geom_user.push_back(G.user); m.geom_group.push_back(G.group);
    m.geom_pos.insert(m.geom_pos.end(), G.pos, G.pos + 3); m.geom_quat.insert(m.geom_quat.end(), G.quat, G.quat + 4); m.geom_size.insert(m.geom_size.end(), G.size, G.size + 3);
    m.geom_friction.insert(m.geom_friction.end(), G.friction, G.friction + 3); m.geom_solref.insert(m.geom_solref.end(), G.solref, G.solref + 2);
    m.geom_solimp.insert(m.geom_solimp.end(), G.solimp, G.solimp + 5); m.geom_rbound.push_back(G.rbound); m.geom_solmix.push_back(G.solmix);
    m.geom_margin.push_back(G.margin); m.geom_gap.push_back(G.gap); m.names_geom.push_back(G.name);
  }
  for (const Site &S : C.sites) { m.site_bodyid.push_back(S.body); m.site_pos.insert(m.site_pos.end(), S.pos, S.pos + 3); m.site_quat.insert(m.site_quat.end(), S.quat, S.quat + 4); m.names_site.push_back(S.name); }
  for (const Camera &K : C.cameras) {
    m.camera_body.push_back(K.body); m.camera_mode.push_back(K.mode); m.camera_pos.insert(m.camera_pos.end(), K.pos, K.pos + 3);
    m.camera_quat.insert(m.camera_quat.end(), K.quat, K.quat + 4); m.camera_fovy.push_back(K.fovy); m.names_camera.push_back(K.name);
  }
  m.nhfield = (int)C.hf_names.size(); m.hfield_nrow = C.hf_nrow; m.hfield_ncol = C.hf_ncol; m.hfield_size = C.hf_size;
  // equality: anchors of body2 computed in the qpos0 configuration
  Kin k; host_fk(m, m.qpos0.data(), k);
  if (const XNode *eq = root->child("equality")) for (auto &e : eq->kids) {
    if (e->tag != "connect") { err = "only <connect> equalities are implemented"; return false; }
    Attrs a = merged(C.dfl, e->get("class") ? e->get("class") : "", "equality", e.get());
    int b1 = m.body_id(A(a, "body1")), b2 = m.body_id(A(a, "body2"));
    if (b1 < 0 || b2 < 0) { err = "connect: unknown body"; return false; }
    vec an = nums(A(a, "anchor")); double gp[3], v[3], a2[3]; mv3(v, &k.xmat[9 * b1], an.data());
    for (int i = 0; i < 3; i++) gp[i] = k.xpos[3 * b1 + i] + v[i] - k.xpos[3 * b2 + i];
    mtv3(a2, &k.xmat[9 * b2], gp);
    m.eq_obj1id.push_back(b1); m.eq_obj2id.push_back(b2);
    m.eq_data.insert(m.eq_data.end(), an.begin(), an.begin() + 3); m.eq_data.insert(m.eq_data.end(), a2, a2 + 3);
    vec sr = Av(a, "solref", "0.02 1"); m.eq_solref.push_back(sr[0]); m.eq_solref.push_back(sr[1]);
    double si[5]; solimp5(a, "solimp", si); m.eq_solimp.insert(m.eq_solimp.end(), si, si + 5);
  }
  m.neq = (int)m.eq_obj1id.size();
  std::vector<std::string> actnames;
  if (const XNode *ac = root->child("actuator")) for (auto &x : ac->kids) {
    if (x->tag != "motor") { err = "only <motor> actuators are implemented"; return false; }
    Attrs a = merged(C.dfl, x->get("class") ? x->get("class") : "", "motor", x.get());
    int j = m.joint_id(A(a, "joint")); if (j < 0) { err = "motor: unknown joint"; return false; }
    actnames.push_back(A(a, "name") ? A(a, "name") : "");
    m.actuator_jntid.push_back(j); m.actuator_gear.push_back(Av(a, "gear", "1")[0]);
    vec cr = Av(a, "ctrlrange", "0 0"); m.actuator_ctrlrange.push_back(cr[0]); m.actuator_ctrlrange.push_back(cr[1]);
    m.actuator_ctrllimited.push_back(A(a, "ctrllimited") && !strcmp(A(a, "ctrllimited"), "true"));
    m.actuator_user.push_back(Av(a, "user", "0")[0]);
  }
  m.nu = (int)m.actuator_jntid.size();
  if (const XNode *sn = root->child("sensor")) for (auto &x : sn->kids) {
    int t, obj = -1;
    if (x->tag == "actuatorpos") { t = SENS_ACTUATORPOS; for (size_t i = 0; i < actnames.size(); i++) if (x->get("actuator") && actnames[i] == x->get("actuator")) obj = (int)i; }
    else if (x->tag == "jointpos") { t = SENS_JOINTPOS; obj = m.joint_id(x->get("joint") ? x->get("joint") : ""); }
    else if (x->tag == "framequat") { t = SENS_FRAMEQUAT; obj = m.site_id(x->get("objname") ? x->get("objname") : ""); }
    else if (x->tag == "gyro") { t = SENS_GYRO; obj = m.site_id(x->get("site") ? x->get("site") : ""); }
    else if (x->tag == "accelerometer") { t = SENS_ACCEL; obj = m.site_id(x->get("site") ? x->get("site") : ""); }
    else if (x->tag == "magnetometer") { t = SENS_MAG; obj = m.site_id(x->get("site") ? x->get("site") : ""); }
    else if (x->tag == "rangefinder") {   // cassie_no_grav.xml: six rangefinders after the 29 numbers the hot path reads; recorded apart (cassie_sim_read_rangefinder)
      const int site = m.site_id(x->get("site") ? x->get("site") : "");
      if (site < 0) { err = "sensor <rangefinder> refers to an unknown site"; return false; }
      m.rangefinder_site.push_back(site); m.rangefinder_cutoff.push_back(x->get("cutoff") ? atof(x->get("cutoff")) : 0);
      continue;
    }
    else { err = "unsupported sensor <" + x->tag + ">"; return false; }
    if (obj < 0) { err = "sensor <" + x->tag + "> refers to an unknown object"; return false; }
    m.sensor_type.push_back(t); m.sensor_objid.push_back(obj);
    m.sensor_user.push_back(x->get("user") ? atof(x->get("user")) : 0); m.sensor_cutoff.push_back(x->get("cutoff") ? atof(x->get("cutoff")) : 0);
  }
  m.nsensor = (int)m.sensor_type.size();
  set_const(m);
  return true;
}

// ------------------------------------------------------------------ .cmodel text tables
namespace {
template <class T> void put(std::ostream &o, const char *k, const std::vector<T> &v, char ty) { o << k << ' ' << ty << ' ' << v.size(); o.precision(17); for (auto &x : v) o << ' ' << x; o << '\n'; }
void puts_(std::ostream &o, const char *k, const std::vector<std::string> &v) { o << k << " S " << v.size(); for (auto &x : v) o << ' ' << (x.empty() ? "-" : x); o << '\n'; }
}  // namespace
bool save_cmodel(const HostModel &m, const std::string &path) {
  std::ofstream o(path); if (!o) return false;
  o << "# compiled Cassie model table (cassie-mujoco-sim_b200/csrc/mjcf.cpp); numeric constants derived from an MJCF file\n";
#define PI1(name) o << #name << " I 1 " << m.name << '\n'
#define PF1(name) o.precision(17), o << #name << " F 1 " << m.name << '\n'
#define PVI(name) put(o, #name, m.name, 'I')
#define PVF(name) put(o, #name, m.name, 'F')
  PI1(nq); PI1(nv); PI1(nu); PI1(nbody); PI1(njnt); PI1(ngeom); PI1(nsite); PI1(neq); PI1(nM); PI1(nsensor); PI1(nhfield); PI1(iterations);
  PF1(timestep); PF1(tolerance); PF1(impratio); PF1(meaninertia);
  put(o, "gravity", std::vector<double>(m.gravity, m.gravity + 3), 'F'); put(o, "magnetic", std::vector<double>(m.magnetic, m.magnetic + 3), 'F');
  PVI(body_parentid); PVI(body_rootid); PVI(body_weldid); PVI(body_jntnum); PVI(body_jntadr); PVI(body_dofnum); PVI(body_dofadr);
  PVF(body_pos); PVF(body_quat); PVF(body_ipos); PVF(body_iquat); PVF(body_mass); PVF(body_inertia); PVF(body_invweight0); PVF(body_subtreemass);
  PVI(jnt_type); PVI(jnt_qposadr); PVI(jnt_dofadr); PVI(jnt_bodyid); PVI(jnt_limited);
  PVF(jnt_pos); PVF(jnt_axis); PVF(jnt_stiffness); PVF(jnt_range); PVF(jnt_margin); PVF(jnt_solref); PVF(jnt_solimp);
  PVI(dof_bodyid); PVI(dof_jntid); PVI(dof_parentid); PVI(dof_Madr); PVF(dof_armature); PVF(dof_damping); PVF(dof_invweight0); PVF(qpos0); PVF(qpos_spring);
  PVI(geom_type); PVI(geom_bodyid); PVI(geom_contype); PVI(geom_conaffinity); PVI(geom_condim); PVI(geom_priority); PVI(geom_hfid); PVI(geom_user); PVI(geom_group);
  PVF(geom_pos); PVF(geom_quat); PVF(geom_size); PVF(geom_friction); PVF(geom_solref); PVF(geom_solimp); PVF(geom_rbound); PVF(geom_solmix); PVF(geom_margin); PVF(geom_gap);
  PVI(site_bodyid); PVF(site_pos); PVF(site_quat); PVI(eq_obj1id); PVI(eq_obj2id); PVF(eq_data); PVF(eq_solref); PVF(eq_solimp);
  PVI(actuator_jntid); PVI(actuator_ctrllimited); PVF(actuator_gear); PVF(actuator_ctrlrange); PVF(actuator_user);
  PVI(sensor_type); PVI(sensor_objid); PVF(sensor_user); PVF(sensor_cutoff); PVI(hfield_nrow); PVI(hfield_ncol); PVF(hfield_size);
  if (!m.rangefinder_site.empty()) { PVI(rangefinder_site); PVF(rangefinder_cutoff); }   // optional: tables of models without rangefinders are unchanged
  if (!m.camera_body.empty()) { PVI(camera_body); PVI(camera_mode); PVF(camera_pos); PVF(camera_quat); PVF(camera_fovy); }   // optional, like the rangefinders
  puts_(o, "names_body", m.names_body); puts_(o, "names_site", m.names_site); puts_(o, "names_geom", m.names_geom); puts_(o, "names_joint", m.names_joint);
  if (!m.names_camera.empty()) puts_(o, "names_camera", m.names_camera);
  return (bool)o;
}
bool load_cmodel(const std::string &path, HostModel &m, std::string &err) {
  std::ifstream f(path); if (!f) { err = "cannot open " + path; return false; }
  m = HostModel(); std::string line;
  while (std::getline(f, line)) {
    if (line.empty() || line[0] == '#') continue;
    std::istringstream is(line); std::string key; char ty; size_t n; is >> key >> ty >> n;
    std::vector<double> vf; std::vector<int> vi; std::vector<std::string> vs;
    if (ty == 'F') { vf.resize(n); for (auto &x : vf) is >> x; } else if (ty == 'I') { vi.resize(n); for (auto &x : vi) is >> x; } else { vs.resize(n); for (auto &x : vs) { is >> x; if (x == "-") x.clear(); } }
#define LI1(name) else if (key == #name) m.name = vi.empty() ? 0 : vi[0]
#define LF1(name) else if (key == #name) m.name = vf.empty() ? 0 : vf[0]
#define LVI(name) else if (key == #name) m.name = vi
#define LVF(name) else if (key == #name) m.name = vf
    if (false) {}
    LI1(nq); LI1(nv); LI1(nu); LI1(nbody); LI1(njnt); LI1(ngeom); LI1(nsite); LI1(neq); LI1(nM); LI1(nsensor); LI1(nhfield); LI1(iterations);
    LF1(timestep); LF1(tolerance); LF1(impratio); LF1(meaninertia);
    else if (key == "gravity") for (int i = 0; i < 3 && i < (int)vf.size(); i++) m.gravity[i] = vf[i];
    else if (key == "magnetic") for (int i = 0; i < 3 && i < (int)vf.size(); i++) m.magnetic[i] = vf[i];
    LVI(body_parentid); LVI(body_rootid); LVI(body_weldid); LVI(body_jntnum); LVI(body_jntadr); LVI(body_dofnum); LVI(body_dofadr);
    LVF(body_pos); LVF(body_quat); LVF(body_ipos); LVF(body_iquat); LVF(body_mass); LVF(body_inertia); LVF(body_invweight0); LVF(body_subtreemass);
    LVI(jnt_type); LVI(jnt_qposadr); LVI(jnt_dofadr); LVI(jnt_bodyid); LVI(jnt_limited);
    LVF(jnt_pos); LVF(jnt_axis); LVF(jnt_stiffness); LVF(jnt_range); LVF(jnt_margin); LVF(jnt_solref); LVF(jnt_solimp);
    LVI(dof_bodyid); LVI(dof_jntid); LVI(dof_parentid); LVI(dof_Madr); LVF(dof_armature); LVF(dof_damping); LVF(dof_invweight0); LVF(qpos0); LVF(qpos_spring);
    LVI(geom_type); LVI(geom_bodyid); LVI(geom_contype); LVI(geom_conaffinity); LVI(geom_condim); LVI(geom_priority); LVI(geom_hfid); LVI(geom_user); LVI(geom_group);
    LVF(geom_pos); LVF(geom_quat); LVF(geom_size); LVF(geom_friction); LVF(geom_solref); LVF(geom_solimp); LVF(geom_rbound); LVF(geom_solmix); LVF(geom_margin); LVF(geom_gap);
    LVI(site_bodyid); LVF(site_pos); LVF(site_quat); LVI(eq_obj1id); LVI(eq_obj2id); LVF(eq_data); LVF(eq_solref); LVF(eq_solimp);
    LVI(actuator_jntid); LVI(actuator_ctrllimited); LVF(actuator_gear); LVF(actuator_ctrlrange); LVF(actuator_user);
    LVI(sensor_type); LVI(sensor_objid); LVF(sensor_user); LVF(sensor_cutoff); LVI(hfield_nrow); LVI(hfield_ncol); LVF(hfield_size);
    LVI(rangefinder_site); LVF(rangefinder_cutoff);
    LVI(camera_body); LVI(camera_mode); LVF(camera_pos); LVF(camera_quat); LVF(camera_fovy);
    else if (key == "names_camera") m.names_camera = vs;
    else if (key == "names_body") m.names_body = vs; else if (key == "names_site") m.names_site = vs;
    else if (key == "names_geom") m.names_geom = vs; else if (key == "names_joint") m.names_joint = vs;
  }
  if (m.nv <= 0 || (int)m.dof_parentid.size() != m.nv || (int)m.body_parentid.size() != m.nbody) { err = "malformed model table " + path; return false; }
  m.geom_user.resize(m.ngeom, 0); m.geom_group.resize(m.ngeom, 0);   // tables written before these columns existed
  if (m.rangefinder_cutoff.size() != m.rangefinder_site.size()) { err = "malformed rangefinder entries in " + path; return false; }
  for (int s : m.rangefinder_site) if (s < 0 || s >= m.nsite) { err = "a rangefinder refers to an unknown site in " + path; return false; }
  const size_t ncam = m.camera_body.size();
  if (m.camera_mode.size() != ncam || m.camera_pos.size() != 3 * ncam || m.camera_quat.size() != 4 * ncam || m.camera_fovy.size() != ncam || m.names_camera.size() != ncam) {
    err = "malformed camera entries in " + path; return false; }
  for (int b : m.camera_body) if (b < 0 || b >= m.nbody) { err = "a camera refers to an unknown body in " + path; return false; }
  return true;
}
bool load_model_any(const std::string &path, HostModel &out, std::string &err) {
  if (path.size() > 4 && path.compare(path.size() - 4, 4, ".xml") == 0) return compile_mjcf(path, out, err);
  return load_cmodel(path, out, err);
}

}  // namespace cassie
