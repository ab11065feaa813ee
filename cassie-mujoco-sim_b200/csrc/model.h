// model.h -- host-side compiled model ("what mj_loadXML + mj_setConst would have produced") for the Cassie model family.
//
// The reference obtains these tables from MuJoCo's XML compiler (mj_loadXML, src/cassiemujoco.c:851,997)
// and mj_setConst (:952).  Here they come from our own MJCF-subset compiler (mjcf.cpp) or from a ".cmodel" text table
// written by it (so a machine without the original project's checkout can load the same constants).
#pragma once
#include <string>
#include <vector>

namespace cassie {

enum JntType { JNT_FREE = 0, JNT_BALL = 1, JNT_SLIDE = 2, JNT_HINGE = 3 };
enum GeomType { GEOM_PLANE = 0, GEOM_HFIELD = 1, GEOM_SPHERE = 2, GEOM_CAPSULE = 3, GEOM_BOX = 6, GEOM_MESH = 7 };
// sensor kinds private to this table (the 29-number Cassie layout, model/cassie.xml:272-292)
enum CameraMode { CAM_FIXED = 0, CAM_TRACK = 1, CAM_TRACKCOM = 2, CAM_TARGETBODY = 3, CAM_TARGETBODYCOM = 4 };
enum SensorKind { SENS_ACTUATORPOS = 0, SENS_JOINTPOS = 1, SENS_FRAMEQUAT = 2, SENS_GYRO = 3, SENS_ACCEL = 4, SENS_MAG = 5 };

struct HostModel {
  // sizes
  int nq = 0, nv = 0, nu = 0, nbody = 0, njnt = 0, ngeom = 0, nsite = 0, neq = 0, nM = 0, nsensor = 0, nhfield = 0;
  // options
  double timestep = 0.002, gravity[3] = {0, 0, -9.81}, magnetic[3] = {0, -0.5, 0}, tolerance = 1e-8, impratio = 1, meaninertia = 1;
  int iterations = 100;
  // bodies
  std::vector<int> body_parentid, body_rootid, body_weldid, body_jntnum, body_jntadr, body_dofnum, body_dofadr;
  std::vector<double> body_pos, body_quat, body_ipos, body_iquat, body_mass, body_inertia, body_invweight0, body_subtreemass;
  // joints
  std::vector<int> jnt_type, jnt_qposadr, jnt_dofadr, jnt_bodyid, jnt_limited;
  std::vector<double> jnt_pos, jnt_axis, jnt_stiffness, jnt_range, jnt_margin, jnt_solref, jnt_solimp;
  // dofs
  std::vector<int> dof_bodyid, dof_jntid, dof_parentid, dof_Madr;
  std::vector<double> dof_armature, dof_damping, dof_invweight0;
  std::vector<double> qpos0, qpos_spring;
  // geoms (mesh geoms are dropped: in every Cassie model they have contype = conaffinity = 0)
  std::vector<int> geom_type, geom_bodyid, geom_contype, geom_conaffinity, geom_condim, geom_priority, geom_hfid, geom_user, geom_group;
  std::vector<double> geom_pos, geom_quat, geom_size, geom_friction, geom_solref, geom_solimp, geom_rbound, geom_solmix,
      geom_margin, geom_gap;
  // sites
  std::vector<int> site_bodyid;
  std::vector<double> site_pos, site_quat;
  // equality (connect only)
  std::vector<int> eq_obj1id, eq_obj2id;
  std::vector<double> eq_data, eq_solref, eq_solimp;
  // actuators (joint motors)
  std::vector<int> actuator_jntid, actuator_ctrllimited;
  std::vector<double> actuator_gear, actuator_ctrlrange, actuator_user;
  // sensors
  std::vector<int> sensor_type, sensor_objid;
  std::vector<double> sensor_user, sensor_cutoff;
  // rangefinders (<rangefinder site= cutoff=>): kept apart from the sensor table, whose 29 numbers the step kernel reads; optional table entries
  std::vector<int> rangefinder_site;
  std::vector<double> rangefinder_cutoff;
  // cameras (<camera>): pose in the body frame, vertical field of view (degrees) and mode (CAM_FIXED ..); optional table entries (cassie_batch_set_camera)
  std::vector<int> camera_body, camera_mode;
  std::vector<double> camera_pos, camera_quat, camera_fovy;
  // height field (at most one)
  std::vector<int> hfield_nrow, hfield_ncol;
  std::vector<double> hfield_size;
  // names
  std::vector<std::string> names_body, names_site, names_geom, names_joint, names_camera;

  int body_id(const std::string &n) const { for (int i = 0; i < (int)names_body.size(); i++) if (names_body[i] == n) return i; return -1; }
  int site_id(const std::string &n) const { for (int i = 0; i < (int)names_site.size(); i++) if (names_site[i] == n) return i; return -1; }
  int joint_id(const std::string &n) const { for (int i = 0; i < (int)names_joint.size(); i++) if (names_joint[i] == n) return i; return -1; }
  int camera_id(const std::string &n) const { for (int i = 0; i < (int)names_camera.size(); i++) if (names_camera[i] == n) return i; return -1; }
  int geom_id(const std::string &n) const { for (int i = 0; i < (int)names_geom.size(); i++) if (names_geom[i] == n) return i; return -1; }
};

// mjcf.cpp
bool compile_mjcf(const std::string &xml_path, HostModel &out, std::string &err);
bool save_cmodel(const HostModel &m, const std::string &path);
bool load_cmodel(const std::string &path, HostModel &out, std::string &err);
// picks by extension: .xml -> compile_mjcf, otherwise load_cmodel
bool load_model_any(const std::string &path, HostModel &out, std::string &err);
// recompute the mj_setConst-type constants (invweights, meaninertia, subtree masses) after masses/inertias changed
void set_const(HostModel &m);

}  // namespace cassie
