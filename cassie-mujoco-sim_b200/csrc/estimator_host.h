// estimator_host.h -- host-side part of the reference's estimator (state_output_step, closed source; semantics recovered by probing the
// archive, DESIGN.md): the toe / heel force of one leg (a pure function of the measured angles and the IMU quaternion) and, further down, the
// Kalman filters behind pelvis.position / translationalVelocity / externalForce and terrain.height.  Both run on the host while state_out_t
// rows are unpacked (the kernel's observation row does not carry them in this round).
//
//   toeForce = heelForce = Rz(yaw)' R(q) [f_x, 0, f_z],   (f_x, f_z) = -1/2 J^-T [k_s shin; k_h (H - H0)],   k = (1500, 1250) N m / rad
//
// H = the heel-spring angle that closes the achilles rod (length 0.5012 between (0, 0, 0.045) on the hip-pitch link and the rod end
// (0.11877, -0.01, 0) of the heel-spring frame, which rides on the tarsus as in model/cassie.xml:132); J = Jacobian (pelvis x, z) of the
// foot point w.r.t. the two spring deflections under that closure.  The archive evaluates this in single precision; agreement ~1e-4 relative.
#pragma once
#include <cmath>
#ifdef __CUDACC__
#define CASSIE_HD __host__ __device__
#else
#define CASSIE_HD
#endif

namespace cassie {

template <typename T> struct V3T { T x, y, z; };
template <typename T> CASSIE_HD inline V3T<T> operator+(V3T<T> a, V3T<T> b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <typename T> CASSIE_HD inline V3T<T> operator-(V3T<T> a, V3T<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <typename T> CASSIE_HD inline V3T<T> operator*(T s, V3T<T> a) { return {s * a.x, s * a.y, s * a.z}; }
template <typename T> CASSIE_HD inline T dot(V3T<T> a, V3T<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> CASSIE_HD inline V3T<T> crs(V3T<T> a, V3T<T> b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
template <typename T> struct M3T { V3T<T> c0, c1, c2; };   // columns
template <typename T> CASSIE_HD inline V3T<T> operator*(const M3T<T> &m, V3T<T> v) { return v.x * m.c0 + v.y * m.c1 + v.z * m.c2; }
template <typename T> CASSIE_HD inline M3T<T> operator*(const M3T<T> &a, const M3T<T> &b) { return {a * b.c0, a * b.c1, a * b.c2}; }
template <typename T> CASSIE_HD inline M3T<T> rotz(T t) { const T c = std::cos(t), s = std::sin(t); return {{c, s, 0}, {-s, c, 0}, {0, 0, 1}}; }
template <typename T> CASSIE_HD inline M3T<T> rotz_sc(T s, T c) { return {{c, s, 0}, {-s, c, 0}, {0, 0, 1}}; }   // the same rotation from a sine / cosine pair the caller already has
using V3 = V3T<double>; using M3 = M3T<double>;

// ang: hipRoll, hipYaw, hipPitch, knee (motor positions), shin, tarsus (joint encoders), foot (motor position); quat: IMU quaternion (w, x, y, z).
// T = double on the host and in fp64 batches; the fp32 kernel instance evaluates it in float, which is the archive's own precision for this block
// sc (optional): {sin, cos} pairs of hipRoll, hipYaw, hipPitch, knee, knee + shin, knee + shin + tarsus, knee + shin + tarsus + foot -- the kernel has
// them from the foot-pose stage of the same tick (same inputs, same sums), so the seven rotations below are not evaluated a second time
template <typename T>
CASSIE_HD inline void estimator_leg_force_t(int side, const T ang[7], const T quat[4], T force[3], const T *sc = nullptr) {
  typedef V3T<T> V; typedef M3T<T> M;
  T scl[14];
  if (sc) { for (int i = 0; i < 14; i++) scl[i] = sc[i]; }
  else { const T a[7] = {ang[0], ang[1], ang[2], ang[3], ang[3] + ang[4], ang[3] + ang[4] + ang[5], ang[3] + ang[4] + ang[5] + ang[6]}; for (int i = 0; i < 7; i++) { scl[2 * i] = std::sin(a[i]); scl[2 * i + 1] = std::cos(a[i]); } }
#define RZ_(i) rotz_sc(scl[2 * (i)], scl[2 * (i) + 1])
  const T sg = side ? T(-1) : T(1), kn = ang[3], sh = ang[4], ta = ang[5];
  // ---- planar part in the hip-pitch frame (z = common axis of knee, shin, tarsus): the four-bar closure
  const V A{0, 0, T(0.045) * sg}, k0{T(0.12), 0, T(0.0045) * sg}, o4{T(0.06068), T(0.04741), 0}, o5{T(0.43476), T(0.02), 0}, hsp{T(-0.01269), T(-0.03059), T(0.00092) * sg}, Bl{T(0.11877), T(-0.01), 0}, ez{0, 0, 1};
  V hx{T(-0.91211), T(0.40829), T(0.036948) * sg}, hy{T(-0.40992), T(-0.90952), T(-0.068841) * sg};
  hx = (T(1) / std::sqrt(dot(hx, hx))) * hx; hy = hy - dot(hx, hy) * hx; hy = (T(1) / std::sqrt(dot(hy, hy))) * hy;
  const M HF{hx, hy, crs(hx, hy)};
  const V s0 = k0 + RZ_(3) * o4, t0 = s0 + RZ_(4) * o5;
  const M R3 = RZ_(5), RH = R3 * HF;
  const V hs0 = t0 + R3 * hsp, axh = RH.c2;
  T H = 0, gd = 1; V B{}, dB{};
  for (int it = 0; it < 9; it++) {   // Newton on |B - A|^2 = L^2 from 0, 8 updates as the oracle: 4 reach the last bit only for |H| < 0.3, and a leg
                                     // driven beyond its joint limits (tarsus ~2.4 rad) got forces off by up to 80 % from them
    B = hs0 + RH * (rotz(H) * Bl); dB = B - A;
    gd = 2 * dot(dB, crs(axh, B - hs0));
    if (it < 8) H -= (dot(dB, dB) - T(0.5012) * T(0.5012)) / gd;
  }
  const T a = -2 * dot(dB, crs(ez, B - t0)) / gd, b = -2 * dot(dB, crs(ez, B - s0)) / gd;   // dH/dtarsus, dH/dshin
  // ---- serial chain pelvis -> hip roll -> hip yaw -> hip pitch: frame A2 of the hip-pitch link (exact quarter turns)
  const M F0{{0, 0, -1}, {0, 1, 0}, {1, 0, 0}}, F1{{0, 0, 1}, {0, 1, 0}, {-1, 0, 0}}, F2{{0, 0, -1}, {1, 0, 0}, {0, -1, 0}};
  const M A0 = F0 * RZ_(0);
  const M A1 = A0 * F1 * RZ_(1);
  const M A2 = A1 * F2 * RZ_(2);
  // foot point in the hip-pitch frame and its partials w.r.t. shin / tarsus (rotations about z through s0 / t0)
  const V f0 = t0 + R3 * V{T(0.408), T(-0.04), 0}, u = f0 + RZ_(6) * V{T(0.01762), T(0.05219), 0};
  const V ps = A2 * crs(ez, u - s0), pt = A2 * crs(ez, u - t0);
  const T j00 = ps.x - pt.x * b / a, j10 = ps.z - pt.z * b / a, j01 = pt.x / a, j11 = pt.z / a, det = j00 * j11 - j10 * j01;
  const T t0_ = T(1500.0) * sh, t1_ = T(1250.0) * (H - T(2.586e-6));
  const T fx = T(-0.5) * (t0_ * j11 - t1_ * j10) / det, fz = T(-0.5) * (-t0_ * j01 + t1_ * j00) / det;
  // ---- heading-free world frame
  const T w = quat[0], x = quat[1], y = quat[2], z = quat[3];
  const T wx = (1 - 2 * (y * y + z * z)) * fx + 2 * (x * z + w * y) * fz, wy = 2 * (x * y + w * z) * fx + 2 * (y * z - w * x) * fz, wz = 2 * (x * z - w * y) * fx + (1 - 2 * (x * x + y * y)) * fz;
  // heading: cos / sin of yaw = atan2(a, b) are b / |(a, b)| and a / |(a, b)|
  const T ya = 2 * (w * z + x * y), yb = 1 - 2 * (y * y + z * z), yn = std::sqrt(ya * ya + yb * yb), cy = yn > 0 ? yb / yn : T(1), sy = yn > 0 ? ya / yn : T(0);
  force[0] = cy * wx + sy * wy; force[1] = -sy * wx + cy * wy; force[2] = wz;
#undef RZ_
}
CASSIE_HD inline void estimator_leg_force(int side, const double ang[7], const double quat[4], double force[3]) { estimator_leg_force_t<double>(side, ang, quat, force); }

// ---- the estimator's filters (pelvis.position / translationalVelocity / externalForce, terrain.height of state_out_t).  Recovered from the
// closed block's own memory (it keeps states, covariances and noise matrices as plain doubles; DESIGN.md section 5): three per-axis Kalman filters
// in the world frame at 2 kHz with the block's nominal mass (31 kg) and gravity (9.806).
//   y_i = -R(q) foot_i (pelvis relative to foot i),  a = R(q) translationalAcceleration,  f_i = min(F_i.z, 0) with F_i = toeForce + heelForce
//   contact = -(f_L + f_R) > 1 N;   w_meas = contact ? f_L / (f_L + f_R) : 1/2;   q_i = F_i.z < -50 N ? 1e-10 : 1e-6   (foot process noise)
//   x, y:  state [p, v, footL, footR, w, F_ext]; in contact v follows a linear inverted pendulum (height 1 m) over w footL + (1 - w) footR plus
//          F_ext / m, else it is held; measurements [p - footL, p - footR, w, v] = [y_L, y_R, w_meas, v_prev + dt a], R = diag(1e-6, 1e-6, 1e-6, 1)
//   z:     state [p, v, footL, footR, F_ext]; v' = -g - (f_L + f_R) / m + F_ext / m; measurements [p - footL, p - footR] = [y_L.z, y_R.z]
//   terrain.height: 1 s first-order lag of p_z - (w_meas y_L.z + (1 - w_meas) y_R.z), advanced in contact only.
// The covariance update keeps the block's own form P <- P - K (H P) (not symmetrised): the block's trajectories are reproduced to 1e-13 with
// it, and a mathematically equal symmetric form drifts away from them within a second of simulated time.
// Measurement rows are differences of two states or single states: row l = e_plus[l] - e_minus[l] (minus < 0: none), R diagonal.  The sums keep the
// term order of the dense products, so dropping the structural zeros changes no bit.
template <int N, int K>
CASSIE_HD inline void kalman_update(double *x, double *P, const int *plus, const int *minus, const double *Rd, const double *zm) {
  double HP[K * N], S[K][2 * K], G[N * K];
  for (int l = 0; l < K; l++) for (int j = 0; j < N; j++) HP[l * N + j] = minus[l] < 0 ? P[plus[l] * N + j] : P[plus[l] * N + j] - P[minus[l] * N + j];
  for (int i = 0; i < N; i++) for (int j = 0; j < K; j++) G[i * K + j] = minus[j] < 0 ? P[i * N + plus[j]] : P[i * N + plus[j]] - P[i * N + minus[j]];   // P H'
  for (int i = 0; i < K; i++) for (int j = 0; j < K; j++) { double a = (i == j ? Rd[i] : 0) + G[plus[i] * K + j]; if (minus[i] >= 0) a -= G[minus[i] * K + j]; S[i][j] = a; S[i][K + j] = i == j; }
  for (int c = 0; c < K; c++) {   // S is symmetric positive definite (R > 0): elimination without row exchanges
    const double inv = 1.0 / S[c][c];
    for (int j = 0; j < 2 * K; j++) S[c][j] *= inv;
    for (int r = 0; r < K; r++) if (r != c) { const double f = S[r][c]; for (int j = 0; j < 2 * K; j++) S[r][j] -= f * S[c][j]; }
  }
  double Kg[N * K], inn[K];
  for (int i = 0; i < N; i++) for (int j = 0; j < K; j++) { double a = 0; for (int l = 0; l < K; l++) a += G[i * K + l] * S[l][K + j]; Kg[i * K + j] = a; }
  for (int j = 0; j < K; j++) { double a = zm[j] - x[plus[j]]; if (minus[j] >= 0) a += x[minus[j]]; inn[j] = a; }
  for (int i = 0; i < N; i++) for (int j = 0; j < K; j++) x[i] += Kg[i * K + j] * inn[j];
  for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) { double a = 0; for (int l = 0; l < K; l++) a += Kg[i * K + l] * HP[l * N + j]; P[i * N + j] -= a; }
}
// P <- A P A' + diag(Qd) for A = identity except A[0][1] = dt and row 1 = a1 (a1[1] = 1)
template <int N>
CASSIE_HD inline void kalman_predict_cov(double *P, double dt, const double *a1, const double *Qd) {
  double T0[N], T1[N];   // rows 0 and 1 of A P; the other rows are P's
  for (int j = 0; j < N; j++) { T0[j] = P[j] + dt * P[N + j]; double a = 0; for (int q = 0; q < N; q++) a += a1[q] * P[q * N + j]; T1[j] = a; }
  for (int j = 0; j < N; j++) { P[j] = T0[j]; P[N + j] = T1[j]; }
  for (int i = 0; i < N; i++) {   // (A P) A': columns 0 and 1 mix, the others only receive Q on the diagonal
    const double *T = P + i * N;
    double c1 = i == 1 ? Qd[1] : 0; for (int q = 0; q < N; q++) c1 += T[q] * a1[q];
    const double c0 = ((i == 0 ? Qd[0] : 0) + T[0]) + T[1] * dt;
    P[i * N] = c0; P[i * N + 1] = c1;
    if (i >= 2) P[i * N + i] = Qd[i] + T[i];
  }
}

// One call of the three filters is written axis by axis: an axis only touches its own state, so on the device three lanes run them side by side.
// The contact terms derived from the two leg forces are shared.
struct EstimatorContact { bool contact; double fl, fr, wm, qL, qR; };
CASSIE_HD inline EstimatorContact estimator_contact(double FLz, double FRz) {
  EstimatorContact k; k.fl = FLz < 0 ? FLz : 0; k.fr = FRz < 0 ? FRz : 0; k.contact = -(k.fl + k.fr) > 1.0;
  k.wm = k.contact ? k.fl / (k.fl + k.fr) : 0.5; k.qL = FLz < -50 ? 1e-10 : 1e-6; k.qR = FRz < -50 ? 1e-10 : 1e-6; return k;
}
constexpr double EST_DT = 0.0005, EST_MASS = 31.0, EST_GRAV = 9.806;
CASSIE_HD inline void estimator_axis_start_xy(double *x, double *P, double yL, double yR) {   // the block's own start: pelvis at 0, the foot states at +y (sic), weight 1/2
  const double x0[6] = {0, 0, yL, yR, 0.5, 0}; for (int i = 0; i < 6; i++) x[i] = x0[i];
  for (int i = 0; i < 36; i++) P[i] = (i % 7 == 0) ? 1e-6 : 0;
}
CASSIE_HD inline void estimator_axis_start_z(double *z, double *P, double yL, double yR) {    // ... and the whole weight on the external force
  const double z0[5] = {0, 0, yL, yR, EST_MASS * EST_GRAV}; for (int i = 0; i < 5; i++) z[i] = z0[i];
  for (int i = 0; i < 25; i++) P[i] = (i % 6 == 0) ? 1e-6 : 0;
}
CASSIE_HD inline void estimator_axis_xy(double *x, double *P, double yL, double yR, double a, const EstimatorContact &k) {
  const double dt = EST_DT, c = EST_DT * EST_GRAV;
  const int plus6[4] = {0, 0, 4, 1}, minus6[4] = {2, 3, -1, -1};   // measurements p - footL, p - footR, w, v
  const double R4[4] = {1e-6, 1e-6, 1e-6, 1};
  const double zm[4] = {yL, yR, k.wm, x[1] + dt * a}, Qd[6] = {1e-8, 1e-8, k.qL, k.qR, 1e-5, 1e-2}, p0 = x[0], v0 = x[1], wt = x[4];
  double a1[6] = {0, 1, 0, 0, 0, 0};   // row 1 of the Jacobian
  if (k.contact) { a1[0] = c; a1[2] = -c * wt; a1[3] = -c * (1 - wt); a1[4] = -c * (x[2] - x[3]); a1[5] = dt / EST_MASS;
                   x[1] = v0 + c * (p0 - wt * x[2] - (1 - wt) * x[3]) + dt / EST_MASS * x[5]; }
  x[0] = p0 + dt * v0;
  kalman_predict_cov<6>(P, dt, a1, Qd);
  kalman_update<6, 4>(x, P, plus6, minus6, R4, zm);
}
CASSIE_HD inline void estimator_axis_z(double *z, double *P, double yL, double yR, const EstimatorContact &k) {
  const double dt = EST_DT;
  const int plus5[2] = {0, 0}, minus5[2] = {2, 3};
  const double R2[2] = {1e-6, 1e-6}, a1[5] = {0, 1, 0, 0, dt / EST_MASS};
  const double zm[2] = {yL, yR}, Qd[5] = {1e-8, 1e-8, k.qL, k.qR, 1e-2}, p0 = z[0], v0 = z[1];
  z[0] = p0 + dt * v0; z[1] = v0 + dt / EST_MASS * z[4] + dt * (-EST_GRAV - (k.fl + k.fr) / EST_MASS);
  kalman_predict_cov<5>(P, dt, a1, Qd);
  kalman_update<5, 2>(z, P, plus5, minus5, R2, zm);
}
CASSIE_HD inline double estimator_terrain(double terrain, double pz, double yLz, double yRz, const EstimatorContact &k) {
  return k.contact ? (terrain + EST_DT * (pz - (k.wm * yLz + (1 - k.wm) * yRz))) / (1 + EST_DT) : terrain;
}

struct EstimatorFilter {
  bool started = false;
  double xy[2][6] = {}, Pxy[2][36] = {}, z[5] = {}, Pz[25] = {}, terrain = 0;
  void reset() { *this = EstimatorFilter(); }
  // quat: pelvis.orientation; footL / footR: foot points in the pelvis frame; FLz / FRz: z of toeForce + heelForce; acc: translationalAcceleration
  void step(const double quat[4], const double footL[3], const double footR[3], double FLz, double FRz, const double acc[3],
            double pos[3], double vel[3], double ext_force[3], double *terrain_height) {
    const double w = quat[0], qx = quat[1], qy = quat[2], qz = quat[3];
    const M3 R{{w * w + qx * qx - qy * qy - qz * qz, 2 * (qx * qy + w * qz), 2 * (qx * qz - w * qy)},
               {2 * (qx * qy - w * qz), w * w - qx * qx + qy * qy - qz * qz, 2 * (qy * qz + w * qx)},
               {2 * (qx * qz + w * qy), 2 * (qy * qz - w * qx), w * w - qx * qx - qy * qy + qz * qz}};
    const V3 yl = -1.0 * (R * V3{footL[0], footL[1], footL[2]}), yr = -1.0 * (R * V3{footR[0], footR[1], footR[2]}), a = R * V3{acc[0], acc[1], acc[2]};
    const double yL[3] = {yl.x, yl.y, yl.z}, yR[3] = {yr.x, yr.y, yr.z}, aw[3] = {a.x, a.y, a.z};
    const EstimatorContact k = estimator_contact(FLz, FRz);
    if (!started) { for (int ax = 0; ax < 2; ax++) estimator_axis_start_xy(xy[ax], Pxy[ax], yL[ax], yR[ax]);
                    estimator_axis_start_z(z, Pz, yL[2], yR[2]); terrain = 0; started = true; }
    for (int ax = 0; ax < 2; ax++) estimator_axis_xy(xy[ax], Pxy[ax], yL[ax], yR[ax], aw[ax], k);
    estimator_axis_z(z, Pz, yL[2], yR[2], k);
    terrain = estimator_terrain(terrain, z[0], yL[2], yR[2], k);
    for (int ax = 0; ax < 2; ax++) { pos[ax] = xy[ax][0]; vel[ax] = xy[ax][1]; ext_force[ax] = xy[ax][5]; }
    pos[2] = z[0]; vel[2] = z[1]; ext_force[2] = z[4];
    *terrain_height = terrain;
  }
};

}  // namespace cassie
