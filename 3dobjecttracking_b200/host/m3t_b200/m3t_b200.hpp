// m3t_b200.hpp — header-only C++17 mirror of M3T's object model for the pose-optimisation path, on top of the
// C ABI of libm3t_b200 (include/m3t_b200.h). It keeps the reference's class and method names, argument meaning and
// bool-return / std::cerr error convention (DLR-RM/3DObjectTracking M3T/include/m3t/{body,camera,color_histograms,
// region_model,depth_model,modality,region_modality,depth_modality,link,optimizer,tracker}.h) so that code written
// against m3t:: reads the same against m3t_b200::, and so that the parity tests read like the reference's tests.
//
//   m3t::Modality::{StartModality,CalculateCorrespondences,CalculateGradientAndHessian,CalculateResults}
//       -> the fine-grained entry points (one batched launch per phase for ALL bodies of the Batch; the adapters
//          de-duplicate the per-object calls a Tracker fans out, see Batch::Phase)
//   m3t::Optimizer::CalculateOptimization              -> m3tb_calculate_optimization
//   m3t::Tracker::ExecuteTrackingStep                  -> m3tb_tracking_step + m3tb_calculate_results (fast path)
//
// Focused depth / silhouette renderers exist as device renderers (k_render), full depth / silhouette / normal
// renderers, the focused normal renderer and the normal viewers as k_view_*, the image viewers on the camera frames and
// NormalizedDepthImage (k_normalized_depth), model generation as DepthModel::GenerateModel (k_model_raster /
// k_model_points) and RegionModel::GenerateModel (k_model_raster / k_region_contours / k_region_points), the texture
// modality as TextureModality (ORB; the caller detects the features). Everything else the reference has outside this
// path (detectors, feature detection, YAML metafiles) is out of scope here (DESIGN.md). Poses use a minimal Transform3fA (row-major 3x4).
#ifndef M3T_B200_HPP_
#define M3T_B200_HPP_

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "m3t_b200.h"

namespace m3t_b200 {

// ---- common.h ------------------------------------------------------------------------------------------------
struct Transform3fA {  // the top three rows of m3t::Transform3fA (Eigen::Transform<float,3,Affine>), row-major
  float m[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
  static Transform3fA Identity() { return Transform3fA(); }
  float& operator()(int r, int c) { return m[4 * r + c]; }
  float operator()(int r, int c) const { return m[4 * r + c]; }
  const float* data() const { return m; }
  float* data() { return m; }
};
using Intrinsics = m3tb_intrinsics;

inline bool Check(m3tb_ctx* ctx, int status, const char* what) {
  if (status == M3TB_OK) return true;
  std::cerr << what << ": " << (ctx ? m3tb_last_error(ctx) : "no context") << " (status " << status << ")" << std::endl;
  return false;
}

// ---- the batch = one m3tb context shared by all objects of a tracker ---------------------------------------------
// A reference Tracker fans every phase out over its modalities / optimizers one object at a time
// (tracker.cpp:447-489). Here a phase is ONE launch for all bodies; the first object that asks for a phase triggers
// it, the others find it done (same iteration / corr_iteration / opt_iteration and unchanged poses).
class Batch {
 public:
  Batch(int device, int max_bodies, int max_cameras, int max_models) {
    if (m3tb_create(device, max_bodies, max_cameras, max_models, &ctx_) != M3TB_OK) {
      ctx_ = nullptr;
      std::cerr << "m3t_b200::Batch: no usable sm_90 CUDA device / context creation failed" << std::endl;
    }
    max_bodies_ = max_bodies;
  }
  ~Batch() {
    if (ctx_) m3tb_destroy(ctx_);
  }
  Batch(const Batch&) = delete;
  Batch& operator=(const Batch&) = delete;
  m3tb_ctx* ctx() const { return ctx_; }
  bool ok() const { return ctx_ != nullptr; }

  enum PhaseKind { kRegionCorr, kDepthCorr, kRegionGH, kDepthGH, kOptimize, kStart, kResults, kRender, kTextureCorr,
                   kTextureGH, kNPhases };
  struct Key {
    int iteration = -1, corr = -1, opt = -1;
    long pose_version = -1;
    bool operator==(const Key& o) const {
      return iteration == o.iteration && corr == o.corr && opt == o.opt && pose_version == o.pose_version;
    }
  };
  // Returns true if the phase still has to run for this key (and records it as done).
  bool Claim(PhaseKind k, int iteration, int corr, int opt) {
    Key key{iteration, corr, opt, pose_version_};
    if (done_[k] == key) return false;
    done_[k] = key;
    return true;
  }
  void MarkDone(PhaseKind k, int iteration, int corr, int opt) { done_[k] = Key{iteration, corr, opt, pose_version_}; }
  void PosesChanged() { ++pose_version_; }
  int NextRenderer() { return n_renderers_++; }
  int NextBody() { return n_bodies_++; }
  int NextColorCamera() { return n_color_++; }
  int NextDepthCamera() { return n_depth_++; }
  int NextRegionModel() { return n_rmodels_++; }
  int NextDepthModel() { return n_dmodels_++; }
  int NextStructure() { return n_structures_++; }
  int NextViewer() { return n_viewers_++; }
  int NextFullRenderer() { return n_full_renderers_++; }
  int NextFocusedNormalRenderer() { return n_focused_normal_renderers_++; }
  int NextEvaluationModel() { return n_evaluation_models_++; }
  // every m3tb_update_viewers renders all viewers of the batch: read-backs older than the last update are stale
  void ViewersUpdated() { ++viewer_version_; }
  long viewer_version() const { return viewer_version_; }
  int n_bodies() const { return n_bodies_; }

  std::vector<float> region_g, region_h, depth_g, depth_h, texture_g, texture_h;  // last batched gradients / Hessians (all bodies)

  // Texture features uploaded from device memory (TextureModality::SetFeatures(const m3tb_device_features&)): their
  // float descriptors are checked on the device, so whether a body's were dropped as non-finite is known once the
  // stream has passed the upload. Every synchronising read of the mirror (Body::body2world_pose, the texture
  // gradient / Hessian) reports it here: a message on std::cerr, and features_dropped(body) until the next upload.
  void NoteDeviceFeatures(int body) {
    pending_features_.push_back(body);
    if (int(dropped_.size()) <= body) dropped_.resize(size_t(body) + 1, 0);
    dropped_[body] = 0;
  }
  bool ReportDroppedFeatures() {
    for (int b : pending_features_) {
      int32_t nonfinite = 0;
      if (m3tb_get_texture_feature_flags(ctx_, b, 1, &nonfinite) != M3TB_OK) {
        std::cerr << "m3tb_get_texture_feature_flags: " << m3tb_last_error(ctx_) << std::endl;
        return false;
      }
      dropped_[b] = nonfinite != 0;
      if (nonfinite)
        std::cerr << "Body " << b << ": non-finite texture descriptor, the frame's features were dropped" << std::endl;
    }
    pending_features_.clear();
    return true;
  }
  bool features_dropped(int body) const { return body < int(dropped_.size()) && dropped_[body]; }

 private:
  m3tb_ctx* ctx_ = nullptr;
  int max_bodies_ = 0, n_bodies_ = 0, n_renderers_ = 0, n_color_ = 0, n_depth_ = 0, n_rmodels_ = 0, n_dmodels_ = 0, n_structures_ = 0;
  int n_viewers_ = 0, n_full_renderers_ = 0, n_focused_normal_renderers_ = 0, n_evaluation_models_ = 0;
  long viewer_version_ = 0;
  long pose_version_ = 0;
  Key done_[kNPhases];
  std::vector<int> pending_features_;
  std::vector<char> dropped_;
};

// ---- body.h --------------------------------------------------------------------------------------------------------
class Body {
 public:
  Body(const std::string& name, const std::shared_ptr<Batch>& batch) : name_(name), batch_(batch) {
    index_ = batch->NextBody();
  }
  const std::string& name() const { return name_; }
  int index() const { return index_; }
  const std::shared_ptr<Batch>& batch() const { return batch_; }
  // Body::set_body2world_pose (body.cpp:85-90)
  bool set_body2world_pose(const Transform3fA& pose) {
    body2world_pose_ = pose;
    batch_->PosesChanged();
    return Check(batch_->ctx(), m3tb_set_poses(batch_->ctx(), index_, 1, pose.data()), "Body::set_body2world_pose");
  }
  // Body::body2world_pose(): reads the pose back from the device (it is updated there by the optimizer)
  const Transform3fA& body2world_pose() {
    Check(batch_->ctx(), m3tb_get_poses(batch_->ctx(), index_, 1, body2world_pose_.data()), "Body::body2world_pose");
    batch_->ReportDroppedFeatures();
    return body2world_pose_;
  }
  // geometry setters (body.h:57-66). The mesh is handed over as the triangle soup Body::SetUp would load from
  // geometry_path: [n][3][3] floats in metres, geometry frame, counter-clockwise seen from outside.
  void set_geometry_triangles(const std::vector<float>& triangles) { triangles_ = triangles; }
  void set_geometry2body_pose(const Transform3fA& p) { geometry2body_pose_ = p; }
  void set_geometry_enable_culling(bool v) { geometry_enable_culling_ = v; }
  void set_maximum_body_diameter(float v) { maximum_body_diameter_ = v; }
  void set_body_id(uint8_t v) { body_id_ = v; }
  void set_region_id(uint8_t v) { region_id_ = v; }
  // what a saved model records about the mesh (Model::SaveBodyData, model.cpp:301-323); the soup above is already
  // scaled and wound, these only describe where it came from
  void set_geometry_path(const std::string& v) { geometry_path_ = v; }
  void set_geometry_unit_in_meter(float v) { geometry_unit_in_meter_ = v; }
  void set_geometry_counterclockwise(bool v) { geometry_counterclockwise_ = v; }
  const std::string& geometry_path() const { return geometry_path_; }
  float geometry_unit_in_meter() const { return geometry_unit_in_meter_; }
  bool geometry_counterclockwise() const { return geometry_counterclockwise_; }
  bool geometry_enable_culling() const { return geometry_enable_culling_; }
  const Transform3fA& geometry2body_pose() const { return geometry2body_pose_; }
  float maximum_body_diameter() const { return maximum_body_diameter_; }
  uint8_t body_id() const { return body_id_; }
  uint8_t region_id() const { return region_id_; }
  // the geometry part of Body::SetUp (body.cpp:201-249): uploads the soup (RendererGeometry::AddBody calls it)
  bool SetUpGeometry() {
    if (triangles_.empty() || triangles_.size() % 9 != 0) {
      std::cerr << "Body " << name_ << " has no geometry" << std::endl;
      return false;
    }
    return Check(batch_->ctx(),
                 m3tb_set_body_geometry(batch_->ctx(), index_, triangles_.data(), int(triangles_.size() / 9),
                                        geometry2body_pose_.data(), maximum_body_diameter_, geometry_enable_culling_ ? 1 : 0,
                                        body_id_, region_id_),
                 "Body::SetUp");
  }

 private:
  std::string name_;
  std::shared_ptr<Batch> batch_;
  int index_ = 0;
  Transform3fA body2world_pose_;
  std::vector<float> triangles_;
  Transform3fA geometry2body_pose_;
  bool geometry_enable_culling_ = true;
  float maximum_body_diameter_ = 0.0f;
  uint8_t body_id_ = 0, region_id_ = 0;
  std::string geometry_path_;
  float geometry_unit_in_meter_ = 1.0f;
  bool geometry_counterclockwise_ = true;
};

// ---- camera.h --------------------------------------------------------------------------------------------------------
class Camera {
 public:
  virtual ~Camera() = default;
  const std::string& name() const { return name_; }
  const Intrinsics& intrinsics() const { return intrinsics_; }
  const Transform3fA& world2camera_pose() const { return world2camera_pose_; }
  int index() const { return index_; }
  bool set_up() const { return set_up_; }
  const std::shared_ptr<Batch>& batch() const { return batch_; }

 protected:
  Camera(const std::string& name, const std::shared_ptr<Batch>& batch) : name_(name), batch_(batch) {}
  std::string name_;
  std::shared_ptr<Batch> batch_;
  Intrinsics intrinsics_{};
  Transform3fA world2camera_pose_;
  int index_ = 0;
  bool set_up_ = false;
};

class ColorCamera : public Camera {
 public:
  ColorCamera(const std::string& name, const std::shared_ptr<Batch>& batch, const Intrinsics& intrinsics,
              const Transform3fA& world2camera_pose)
      : Camera(name, batch) {
    intrinsics_ = intrinsics;
    world2camera_pose_ = world2camera_pose;
    index_ = batch->NextColorCamera();
  }
  bool SetUp() {
    set_up_ = Check(batch_->ctx(), m3tb_set_color_camera(batch_->ctx(), index_, &intrinsics_, world2camera_pose_.data()),
                    "ColorCamera::SetUp");
    return set_up_;
  }
  // Camera::UpdateImage with a caller-owned BGR8 frame (cv::Mat::data / step)
  bool UpdateImage(const uint8_t* bgr, size_t pitch) {
    if (!set_up_) {
      std::cerr << "Set up color camera " << name_ << " first" << std::endl;
      return false;
    }
    return Check(batch_->ctx(), m3tb_upload_color(batch_->ctx(), index_, bgr, pitch), "ColorCamera::UpdateImage");
  }
};

class DepthCamera : public Camera {
 public:
  DepthCamera(const std::string& name, const std::shared_ptr<Batch>& batch, const Intrinsics& intrinsics,
              const Transform3fA& world2camera_pose, float depth_scale)
      : Camera(name, batch), depth_scale_(depth_scale) {
    intrinsics_ = intrinsics;
    world2camera_pose_ = world2camera_pose;
    index_ = batch->NextDepthCamera();
  }
  float depth_scale() const { return depth_scale_; }
  bool SetUp() {
    set_up_ = Check(batch_->ctx(),
                    m3tb_set_depth_camera(batch_->ctx(), index_, &intrinsics_, world2camera_pose_.data(), depth_scale_),
                    "DepthCamera::SetUp");
    return set_up_;
  }
  bool UpdateImage(const uint16_t* depth, size_t pitch) {
    if (!set_up_) {
      std::cerr << "Set up depth camera " << name_ << " first" << std::endl;
      return false;
    }
    return Check(batch_->ctx(), m3tb_upload_depth(batch_->ctx(), index_, depth, pitch), "DepthCamera::UpdateImage");
  }
  // DepthCamera::NormalizedDepthImage (camera.cpp:108-115) of the frame the camera holds: width x height u8 (empty on
  // failure)
  std::vector<uint8_t> NormalizedDepthImage(float min_depth, float max_depth) const {
    std::vector<uint8_t> image(size_t(intrinsics_.width) * size_t(intrinsics_.height));
    if (!Check(batch_->ctx(),
               m3tb_get_normalized_depth_image(batch_->ctx(), M3TB_NORMALIZED_DEPTH_CAMERA, index_, min_depth, max_depth,
                                               image.data(), size_t(intrinsics_.width)),
               "DepthCamera::NormalizedDepthImage"))
      image.clear();
    return image;
  }

 private:
  float depth_scale_;
};

// ---- azure_kinect_camera.h, without the SDK -------------------------------------------------------------------------
// The calibration k4a::device::get_calibration reports for one camera (k4a_calibration_intrinsic_parameters_t::_param
// and the resolution). The caller reads it from the SDK (or a file) and hands it over.
struct AzureKinectCalibration {
  float fx = 0, fy = 0, cx = 0, cy = 0;
  float k1 = 0, k2 = 0, k3 = 0, k4 = 0, k5 = 0, k6 = 0, p1 = 0, p2 = 0;
  int width = 0, height = 0;
};

// GetIntrinsicsAndDistortionMap (azure_kinect_camera.cpp:234-265, 387-419): fu / fv scaled by image_scale, ppu / ppv
// kept; the map of cv::initUndistortRectifyMap + convertMaps(CV_16SC2) from camera matrix (fx, fy, cx, cy) to that
// camera, coefficients in OpenCV order.
inline bool AzureKinectIntrinsicsAndDistortionMap(const AzureKinectCalibration& c, float image_scale, Intrinsics* intrinsics,
                                                  std::vector<int16_t>* map) {
  Intrinsics raw{c.fx, c.fy, c.cx, c.cy, c.width, c.height};
  *intrinsics = raw;
  intrinsics->fu *= image_scale;
  intrinsics->fv *= image_scale;
  const float coefficients[8] = {c.k1, c.k2, c.p1, c.p2, c.k3, c.k4, c.k5, c.k6};
  if (c.width <= 0 || c.height <= 0) return false;
  map->assign(size_t(c.width) * size_t(c.height) * 2, 0);
  return m3tb_undistortion_map(&raw, coefficients, intrinsics, map->data(), size_t(c.width) * 4) == M3TB_OK;
}

// AzureKinectColorCamera: UpdateImage takes the SDK's BGRA32 colour buffer (get_color_image().get_buffer()) and leaves
// the rectified BGR frame on the device (cvtColor(RGBA2RGB) + remap, azure_kinect_camera.cpp:175-195).
class AzureKinectColorCamera : public ColorCamera {
 public:
  AzureKinectColorCamera(const std::string& name, const std::shared_ptr<Batch>& batch,
                         const AzureKinectCalibration& calibration, float image_scale = 1.05f,
                         const Transform3fA& world2camera_pose = Transform3fA())
      : ColorCamera(name, batch, Intrinsics{}, world2camera_pose), calibration_(calibration), image_scale_(image_scale) {}
  float image_scale() const { return image_scale_; }
  bool SetUp() {
    set_up_ = false;
    if (!AzureKinectIntrinsicsAndDistortionMap(calibration_, image_scale_, &intrinsics_, &distortion_map_)) {
      std::cerr << "Azure Kinect color camera " << name_ << ": invalid calibration" << std::endl;
      return false;
    }
    if (!ColorCamera::SetUp()) return false;
    set_up_ = Check(batch_->ctx(),
                    m3tb_set_camera_undistortion(batch_->ctx(), 0, index_, distortion_map_.data(),
                                                 size_t(intrinsics_.width) * 4, 4, 0),
                    "AzureKinectColorCamera::SetUp");
    return set_up_;
  }
  // `buffer`: the BGRA32 image, `pitch` bytes per row (k4a::image::get_stride_bytes)
  bool UpdateImage(const uint8_t* buffer, size_t pitch) {
    if (!set_up_) {
      std::cerr << "Set up azure kinect color camera " << name_ << " first" << std::endl;
      return false;
    }
    return Check(batch_->ctx(), m3tb_upload_color(batch_->ctx(), index_, buffer, pitch),
                 "AzureKinectColorCamera::UpdateImage");
  }
  const std::vector<int16_t>& distortion_map() const { return distortion_map_; }

 private:
  AzureKinectCalibration calibration_;
  float image_scale_;
  std::vector<int16_t> distortion_map_;
};

// AzureKinectDepthCamera: UpdateImage takes the SDK's u16 depth buffer and leaves the rectified frame, plus
// short(depth_offset / depth_scale) with saturation, on the device (azure_kinect_camera.cpp:321-345).
class AzureKinectDepthCamera : public DepthCamera {
 public:
  AzureKinectDepthCamera(const std::string& name, const std::shared_ptr<Batch>& batch,
                         const AzureKinectCalibration& calibration, float image_scale = 1.0f, float depth_offset = 0.0f,
                         float depth_scale = 0.001f, const Transform3fA& world2camera_pose = Transform3fA())
      : DepthCamera(name, batch, Intrinsics{}, world2camera_pose, depth_scale),
        calibration_(calibration),
        image_scale_(image_scale),
        depth_offset_(depth_offset) {}
  float image_scale() const { return image_scale_; }
  float depth_offset() const { return depth_offset_; }
  // short depth_value_offset = depth_offset_ / depth_scale_ (C++ truncation); false outside the range of short
  bool depth_value_offset(int* out) const {
    const float q = depth_offset_ / depth_scale();
    if (!(q > -32769.0f && q < 32768.0f)) return false;
    *out = int(short(q));
    return true;
  }
  bool SetUp() {
    set_up_ = false;
    int offset = 0;
    if (!depth_value_offset(&offset)) {
      std::cerr << "Azure Kinect depth camera " << name_ << ": depth offset outside the range of short" << std::endl;
      return false;
    }
    if (!AzureKinectIntrinsicsAndDistortionMap(calibration_, image_scale_, &intrinsics_, &distortion_map_)) {
      std::cerr << "Azure Kinect depth camera " << name_ << ": invalid calibration" << std::endl;
      return false;
    }
    if (!DepthCamera::SetUp()) return false;
    set_up_ = Check(batch_->ctx(),
                    m3tb_set_camera_undistortion(batch_->ctx(), 1, index_, distortion_map_.data(),
                                                 size_t(intrinsics_.width) * 4, 1, depth_offset_ ? offset : 0),
                    "AzureKinectDepthCamera::SetUp");
    return set_up_;
  }
  // `buffer`: the u16 depth image as bytes, `pitch` bytes per row
  bool UpdateImage(const uint8_t* buffer, size_t pitch) {
    if (!set_up_) {
      std::cerr << "Set up azure kinect depth camera " << name_ << " first" << std::endl;
      return false;
    }
    return Check(batch_->ctx(),
                 m3tb_upload_depth(batch_->ctx(), index_, reinterpret_cast<const uint16_t*>(buffer), pitch),
                 "AzureKinectDepthCamera::UpdateImage");
  }
  const std::vector<int16_t>& distortion_map() const { return distortion_map_; }

 private:
  AzureKinectCalibration calibration_;
  float image_scale_, depth_offset_;
  std::vector<int16_t> distortion_map_;
};

// ---- region_model.h / depth_model.h: views in the reference's DataPoint layout ---------------------------------------
class Model {
 public:
  const std::string& name() const { return name_; }
  int index() const { return index_; }
  bool set_up() const { return set_up_; }
  int n_views() const { return n_views_; }
  int n_points() const { return n_points_; }
  // Views as stored by RegionModel/DepthModel::SaveModel: n_views x (n_points x DataPoint), orientations, scalars
  void SetViews(int n_views, int n_points, const float* orientations, const float* view_scalars, const void* points) {
    n_views_ = n_views;
    n_points_ = n_points;
    orientations_.assign(orientations, orientations + size_t(3) * n_views);
    scalars_.assign(view_scalars, view_scalars + n_views);
    const size_t bytes = size_t(n_views) * n_points * point_bytes_;
    points_.assign(static_cast<const uint8_t*>(points), static_cast<const uint8_t*>(points) + bytes);
  }
  // Model::LoadModel for the view block of a .bin (header / body blocks skipped, see 3dobjecttracking_b200/model_io.py)
  bool LoadViews(const std::string& path, size_t view_block_offset, int n_views, int n_points) {
    std::ifstream ifs(path, std::ios::in | std::ios::binary);
    if (!ifs.is_open()) {
      std::cerr << "Could not open model file " << path << std::endl;
      return false;
    }
    ifs.seekg(std::streamoff(view_block_offset));
    n_views_ = n_views;
    n_points_ = n_points;
    orientations_.resize(size_t(3) * n_views);
    scalars_.resize(n_views);
    points_.resize(size_t(n_views) * n_points * point_bytes_);
    for (int v = 0; v < n_views; ++v) {
      ifs.read(reinterpret_cast<char*>(points_.data() + size_t(v) * n_points * point_bytes_), std::streamsize(n_points) * point_bytes_);
      ifs.read(reinterpret_cast<char*>(&orientations_[3 * v]), 12);
      ifs.read(reinterpret_cast<char*>(&scalars_[v]), 4);
    }
    return bool(ifs);
  }

  // model.h setters (model.h:161-167); stride / max radius are also what SetUp hands to the device
  void set_sphere_radius(float v) { params_.sphere_radius = v; }
  void set_n_divides(int v) { params_.n_divides = v; }
  void set_n_points(int v) { params_.n_points = v; }
  void set_max_radius_depth_offset(float v) { params_.max_radius_depth_offset = v; }
  void set_stride_depth_offset(float v) { params_.stride_depth_offset = v; }
  void set_use_random_seed(bool v) { params_.use_random_seed = v ? 1 : 0; }
  void set_image_size(int v) { params_.image_size = v; }
  const m3tb_model_params& params() const { return params_; }

 protected:
  Model(const std::string& name, const std::shared_ptr<Batch>& batch, int point_bytes)
      : name_(name), batch_(batch), point_bytes_(point_bytes) {
    m3tb_model_params_default(&params_);
  }

  // Uploads the meshes of the model's body and `others` (m3tb_set_body_geometry); false if there is no body
  bool SetUpGeometries(const char* kind, const std::vector<std::shared_ptr<Body>>& others) {
    if (!body_ptr_) {
      std::cerr << kind << " model " << name_ << " has no body" << std::endl;
      return false;
    }
    if (!body_ptr_->SetUpGeometry()) return false;
    for (auto& b : others)
      if (!b->SetUpGeometry()) return false;
    return true;
  }

  // Model::SaveModel (model.cpp:286-323): header and body block; the caller writes its associated bodies, then
  // WriteViews
  bool OpenAndWriteHeader(std::ofstream& ofs, const std::string& path, char type, int32_t version) const {
    if (!body_ptr_ || n_views_ == 0) {
      std::cerr << "Model " << name_ << " has no body or no views" << std::endl;
      return false;
    }
    ofs.open(path, std::ios::out | std::ios::binary);
    if (!ofs.is_open()) {
      std::cerr << "Could not open model file " << path << std::endl;
      return false;
    }
    const bool use_random_seed = params_.use_random_seed != 0;
    Write(ofs, type);
    Write(ofs, version);
    Write(ofs, params_.sphere_radius);
    Write(ofs, int32_t(params_.n_divides));
    Write(ofs, int32_t(n_points_));
    Write(ofs, params_.max_radius_depth_offset);
    Write(ofs, params_.stride_depth_offset);
    Write(ofs, use_random_seed);
    Write(ofs, int32_t(params_.image_size));
    WriteBody(ofs, *body_ptr_);
    return true;
  }
  bool WriteViews(std::ofstream& ofs) const {
    Write(ofs, uint64_t(n_views_));
    for (int v = 0; v < n_views_; ++v) {
      ofs.write(reinterpret_cast<const char*>(points_.data() + size_t(v) * n_points_ * point_bytes_),
                std::streamsize(n_points_) * point_bytes_);
      ofs.write(reinterpret_cast<const char*>(&orientations_[3 * size_t(v)]), 12);
      Write(ofs, scalars_[v]);
    }
    ofs.flush();
    return bool(ofs);
  }
  template <typename T>
  static void Write(std::ofstream& ofs, const T& v) {
    ofs.write(reinterpret_cast<const char*>(&v), sizeof(T));
  }
  // Model::SaveBodyData: path, unit, winding, culling, diameter, geometry2body as Eigen's column-major 4x4
  static void WriteBody(std::ofstream& ofs, const Body& b) {
    Write(ofs, uint64_t(b.geometry_path().size()));
    ofs.write(b.geometry_path().data(), std::streamsize(b.geometry_path().size()));
    Write(ofs, b.geometry_unit_in_meter());
    Write(ofs, b.geometry_counterclockwise());
    Write(ofs, b.geometry_enable_culling());
    Write(ofs, b.maximum_body_diameter());
    const Transform3fA& g = b.geometry2body_pose();
    for (int c = 0; c < 4; ++c)
      for (int r = 0; r < 4; ++r) Write(ofs, r < 3 ? g(r, c) : (c == 3 ? 1.0f : 0.0f));
  }
  static void WriteBodies(std::ofstream& ofs, const std::vector<std::shared_ptr<Body>>& bodies) {
    Write(ofs, uint64_t(bodies.size()));
    for (auto& b : bodies) WriteBody(ofs, *b);
  }

  std::string name_;
  std::shared_ptr<Batch> batch_;
  int point_bytes_;
  int index_ = 0, n_views_ = 0, n_points_ = 0;
  std::vector<float> orientations_, scalars_;
  std::vector<uint8_t> points_;
  bool set_up_ = false;
  m3tb_model_params params_{};
  std::shared_ptr<Body> body_ptr_;
};

class RegionModel : public Model {
 public:
  RegionModel(const std::string& name, const std::shared_ptr<Batch>& batch) : Model(name, batch, M3TB_REGION_POINT_BYTES) {
    index_ = batch->NextRegionModel();
  }
  // RegionModel(name, body_ptr, model_path, ...) with the body whose model is generated (region_model.h:108-114)
  RegionModel(const std::string& name, const std::shared_ptr<Batch>& batch, const std::shared_ptr<Body>& body_ptr)
      : RegionModel(name, batch) {
    body_ptr_ = body_ptr;
  }
  bool SetUp() {
    if (n_views_ == 0) {
      std::cerr << "Region model " << name_ << " has no views" << std::endl;
      return false;
    }
    set_up_ = Check(batch_->ctx(),
                    m3tb_set_region_model(batch_->ctx(), index_, n_views_, n_points_, orientations_.data(), scalars_.data(),
                                          points_.data(), params_.stride_depth_offset, params_.max_radius_depth_offset),
                    "RegionModel::SetUp");
    return set_up_;
  }

  // RegionModel::AddAssociatedBody (region_model.cpp:61-82): refused for a name already added; the four groups keep
  // insertion order
  bool AddAssociatedBody(const std::shared_ptr<Body>& body_ptr, bool movable, bool same_region) {
    for (auto& a : associated_)
      if (a.body->name() == body_ptr->name()) {
        std::cerr << "Body " << body_ptr->name() << " already exists" << std::endl;
        return false;
      }
    associated_.push_back({body_ptr, movable, same_region});
    return true;
  }

  // RegionModel::GenerateModel (region_model.cpp:187-257) on the device: uploads the meshes, generates, installs the
  // model for tracking and keeps its views so that SaveModel can write them
  bool GenerateModel() {
    std::vector<std::shared_ptr<Body>> others;
    std::vector<m3tb_associated_body> assoc;
    for (auto& a : associated_) {
      others.push_back(a.body);
      assoc.push_back({int32_t(a.body->index()), int32_t(a.movable), int32_t(a.same_region)});
    }
    if (!SetUpGeometries("Region", others)) return false;
    m3tb_ctx* ctx = batch_->ctx();
    if (!Check(ctx, m3tb_generate_region_model(ctx, index_, body_ptr_->index(), assoc.data(), int(assoc.size()), &params_),
               "RegionModel::GenerateModel"))
      return false;
    int nv = 0, np = 0;
    if (!Check(ctx, m3tb_get_region_model(ctx, index_, &nv, &np, nullptr, nullptr, nullptr, nullptr, nullptr),
               "RegionModel::GenerateModel"))
      return false;
    std::vector<float> ori(size_t(3) * nv), length(nv), points(size_t(nv) * np * (M3TB_REGION_POINT_BYTES / 4));
    if (!Check(ctx, m3tb_get_region_model(ctx, index_, nullptr, nullptr, ori.data(), length.data(), points.data(),
                                          nullptr, nullptr),
               "RegionModel::GenerateModel"))
      return false;
    SetViews(nv, np, ori.data(), length.data(), points.data());
    set_up_ = true;
    return true;
  }

  // RegionModel::SaveModel (model.cpp:286-323, region_model.cpp:309-345): the reference's .bin layout, version 10, with
  // the associated bodies as fixed, fixed same-region, movable, movable same-region
  bool SaveModel(const std::string& path) const {
    std::ofstream ofs;
    if (!OpenAndWriteHeader(ofs, path, 'r', 10)) return false;
    Write(ofs, uint64_t(associated_.size()));
    for (int group = 0; group < 4; ++group) {
      std::vector<std::shared_ptr<Body>> bodies;
      for (auto& a : associated_)
        if (int(a.movable) * 2 + int(a.same_region) == group) bodies.push_back(a.body);
      WriteBodies(ofs, bodies);
    }
    return WriteViews(ofs);
  }

 private:
  struct Associated {
    std::shared_ptr<Body> body;
    bool movable, same_region;
  };
  std::vector<Associated> associated_;
};

class DepthModel : public Model {
 public:
  DepthModel(const std::string& name, const std::shared_ptr<Batch>& batch) : Model(name, batch, M3TB_DEPTH_POINT_BYTES) {
    index_ = batch->NextDepthModel();
  }
  // DepthModel(name, body_ptr, model_path, ...) with the body whose model is generated (depth_model.h:108-114)
  DepthModel(const std::string& name, const std::shared_ptr<Batch>& batch, const std::shared_ptr<Body>& body_ptr)
      : DepthModel(name, batch) {
    body_ptr_ = body_ptr;
  }
  bool SetUp() {
    if (n_views_ == 0) {
      std::cerr << "Depth model " << name_ << " has no views" << std::endl;
      return false;
    }
    set_up_ = Check(batch_->ctx(),
                    m3tb_set_depth_model(batch_->ctx(), index_, n_views_, n_points_, orientations_.data(), scalars_.data(),
                                         points_.data(), params_.stride_depth_offset, params_.max_radius_depth_offset),
                    "DepthModel::SetUp");
    return set_up_;
  }

  // DepthModel::AddOcclusionBody (depth_model.cpp:61-69)
  bool AddOcclusionBody(const std::shared_ptr<Body>& body_ptr) {
    for (auto& b : occlusion_body_ptrs_)
      if (b->name() == body_ptr->name()) {
        std::cerr << "Occlusion body " << body_ptr->name() << " already exists" << std::endl;
        return false;
      }
    occlusion_body_ptrs_.push_back(body_ptr);
    return true;
  }

  // DepthModel::GenerateModel (depth_model.cpp:144-213) on the device: uploads the meshes, generates, installs the
  // model for tracking and keeps its views so that SaveModel can write them
  bool GenerateModel() {
    if (!SetUpGeometries("Depth", occlusion_body_ptrs_)) return false;
    std::vector<int> occ;
    for (auto& b : occlusion_body_ptrs_) occ.push_back(b->index());
    m3tb_ctx* ctx = batch_->ctx();
    if (!Check(ctx, m3tb_generate_depth_model(ctx, index_, body_ptr_->index(), occ.data(), int(occ.size()), &params_),
               "DepthModel::GenerateModel"))
      return false;
    int nv = 0, np = 0;
    if (!Check(ctx, m3tb_get_depth_model(ctx, index_, &nv, &np, nullptr, nullptr, nullptr, nullptr, nullptr),
               "DepthModel::GenerateModel"))
      return false;
    std::vector<float> ori(size_t(3) * nv), area(nv), points(size_t(nv) * np * (M3TB_DEPTH_POINT_BYTES / 4));
    if (!Check(ctx, m3tb_get_depth_model(ctx, index_, nullptr, nullptr, ori.data(), area.data(), points.data(), nullptr,
                                         nullptr),
               "DepthModel::GenerateModel"))
      return false;
    SetViews(nv, np, ori.data(), area.data(), points.data());
    set_up_ = true;
    return true;
  }

  // DepthModel::SaveModel (model.cpp:286-323, depth_model.cpp:265-291): the reference's .bin layout, version 9
  bool SaveModel(const std::string& path) const {
    std::ofstream ofs;
    if (!OpenAndWriteHeader(ofs, path, 'd', 9)) return false;
    WriteBodies(ofs, occlusion_body_ptrs_);
    return WriteViews(ofs);
  }

 private:
  std::vector<std::shared_ptr<Body>> occlusion_body_ptrs_;
};

// ---- renderer_geometry.h / renderer.h / basic_depth_renderer.h / silhouette_renderer.h: device renderers (k_render) ----
class RendererGeometry {
 public:
  RendererGeometry(const std::string& name, const std::shared_ptr<Batch>& batch) : name_(name), batch_(batch) {}
  // RendererGeometry::AddBody: uploads the body's triangle soup; bodies are drawn in the order they were added
  bool AddBody(const std::shared_ptr<Body>& body_ptr) {
    for (auto& b : body_ptrs_)
      if (b->name() == body_ptr->name()) {
        std::cerr << "Body " << body_ptr->name() << " already exists" << std::endl;
        return false;
      }
    if (!body_ptr->SetUpGeometry()) return false;
    body_ptrs_.push_back(body_ptr);
    return true;
  }
  bool SetUp() { set_up_ = true; return true; }
  bool set_up() const { return set_up_; }
  const std::string& name() const { return name_; }
  const std::vector<std::shared_ptr<Body>>& body_ptrs() const { return body_ptrs_; }

 private:
  std::string name_;
  std::shared_ptr<Batch> batch_;
  std::vector<std::shared_ptr<Body>> body_ptrs_;
  bool set_up_ = false;
};

enum class IDType { BODY = 0, REGION = 1 };  // body.h

// FocusedDepthRenderer (renderer.h:199-230). Every device renderer also produces the silhouette image, so the two
// focused renderer classes below only differ in their defaults.
class FocusedDepthRenderer {
 public:
  virtual ~FocusedDepthRenderer() = default;
  bool AddReferencedBody(const std::shared_ptr<Body>& body_ptr) {
    for (auto& b : referenced_body_ptrs_)
      if (b->name() == body_ptr->name()) {
        std::cerr << "Body " << body_ptr->name() << " already exists" << std::endl;
        return false;
      }
    referenced_body_ptrs_.push_back(body_ptr);
    set_up_ = false;
    return true;
  }
  bool SetUp() {
    set_up_ = false;
    std::vector<int> geo, ref;
    for (auto& b : renderer_geometry_ptr_->body_ptrs()) geo.push_back(b->index());
    for (auto& b : referenced_body_ptrs_) ref.push_back(b->index());
    const int kind = std::dynamic_pointer_cast<ColorCamera>(camera_ptr_) ? 0 : 1;
    if (!Check(batch_->ctx(),
               m3tb_set_focused_renderer(batch_->ctx(), index_, kind, camera_ptr_->index(), image_size_, z_min_, z_max_,
                                         int(id_type_), geo.data(), int(geo.size()), ref.data(), int(ref.size())),
               "FocusedRenderer::SetUp"))
      return false;
    set_up_ = true;
    return true;
  }
  // FocusedRenderer::StartRendering: one k_render launch for every device renderer of the batch (the renderers a
  // Tracker starts one after another at the same poses share it)
  bool StartRendering() {
    if (!set_up_) {
      std::cerr << "Set up renderer " << name_ << " first" << std::endl;
      return false;
    }
    fetched_ = false;
    if (!batch_->Claim(Batch::kRender, 0, 0, 0)) return true;
    return Check(batch_->ctx(), m3tb_render(batch_->ctx()), "FocusedRenderer::StartRendering");
  }
  bool FetchDepthImage() { return Fetch(); }
  bool IsBodyVisible(const std::string& body_name) {
    if (!Fetch()) return false;
    for (size_t k = 0; k < referenced_body_ptrs_.size(); ++k)
      if (referenced_body_ptrs_[k]->name() == body_name) return visible_[k] != 0;
    return false;
  }
  bool IsBodyReferenced(const std::string& body_name) const {
    for (auto& b : referenced_body_ptrs_)
      if (b->name() == body_name) return true;
    return false;
  }
  const std::vector<uint16_t>& focused_depth_image() { Fetch(); return depth_; }
  float corner_u() { Fetch(); return corner_u_; }
  float corner_v() { Fetch(); return corner_v_; }
  float scale() { Fetch(); return scale_; }
  float projection_term_a() { Fetch(); return projection_term_a_; }
  float projection_term_b() { Fetch(); return projection_term_b_; }
  int image_size() const { return image_size_; }
  float z_min() const { return z_min_; }
  float z_max() const { return z_max_; }
  IDType id_type() const { return id_type_; }
  void set_image_size(int v) { image_size_ = v; set_up_ = false; }
  void set_z_min(float v) { z_min_ = v; set_up_ = false; }
  void set_z_max(float v) { z_max_ = v; set_up_ = false; }
  bool set_up() const { return set_up_; }
  int index() const { return index_; }
  const std::string& name() const { return name_; }
  const std::shared_ptr<Camera>& camera_ptr() const { return camera_ptr_; }
  const std::vector<std::shared_ptr<Body>>& referenced_body_ptrs() const { return referenced_body_ptrs_; }

 protected:
  FocusedDepthRenderer(const std::string& name, const std::shared_ptr<Batch>& batch,
                       const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr, const std::shared_ptr<Camera>& camera_ptr,
                       IDType id_type, int image_size, float z_min, float z_max)
      : name_(name), batch_(batch), renderer_geometry_ptr_(renderer_geometry_ptr), camera_ptr_(camera_ptr), id_type_(id_type),
        image_size_(image_size), z_min_(z_min), z_max_(z_max) {
    index_ = batch->NextRenderer();
  }
  // FetchDepthImage / FetchSilhouetteImage: one read-back of the last rendering (debug / display)
  bool Fetch() {
    if (fetched_) return true;
    const size_t n = size_t(image_size_) * image_size_;
    depth_.resize(n);
    silhouette_.resize(n);
    visible_.assign(referenced_body_ptrs_.size(), 0);
    fetched_ = Check(batch_->ctx(),
                     m3tb_get_rendering(batch_->ctx(), index_, depth_.data(), silhouette_.data(), &corner_u_, &corner_v_,
                                        &scale_, &projection_term_a_, &projection_term_b_, visible_.data()),
                     "FocusedRenderer::FetchImage");
    return fetched_;
  }
  std::string name_;
  std::shared_ptr<Batch> batch_;
  std::shared_ptr<RendererGeometry> renderer_geometry_ptr_;
  std::shared_ptr<Camera> camera_ptr_;
  std::vector<std::shared_ptr<Body>> referenced_body_ptrs_;
  IDType id_type_;
  int image_size_;
  float z_min_, z_max_;
  int index_ = 0;
  bool set_up_ = false, fetched_ = false;
  std::vector<uint16_t> depth_;
  std::vector<uint8_t> silhouette_;
  std::vector<int> visible_;
  float corner_u_ = 0, corner_v_ = 0, scale_ = 0, projection_term_a_ = 0, projection_term_b_ = 0;
};

class FocusedBasicDepthRenderer : public FocusedDepthRenderer {
 public:
  FocusedBasicDepthRenderer(const std::string& name, const std::shared_ptr<Batch>& batch,
                            const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr,
                            const std::shared_ptr<Camera>& camera_ptr, int image_size = 200, float z_min = 0.02f,
                            float z_max = 10.0f)
      : FocusedDepthRenderer(name, batch, renderer_geometry_ptr, camera_ptr, IDType::BODY, image_size, z_min, z_max) {}
};

class FocusedSilhouetteRenderer : public FocusedDepthRenderer {
 public:
  FocusedSilhouetteRenderer(const std::string& name, const std::shared_ptr<Batch>& batch,
                            const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr,
                            const std::shared_ptr<Camera>& camera_ptr, IDType id_type = IDType::BODY, int image_size = 200,
                            float z_min = 0.02f, float z_max = 10.0f)
      : FocusedDepthRenderer(name, batch, renderer_geometry_ptr, camera_ptr, id_type, image_size, z_min, z_max) {}
  bool FetchSilhouetteImage() { return Fetch(); }
  const std::vector<uint8_t>& focused_silhouette_image() { Fetch(); return silhouette_; }
};

// ---- renderer.h / basic_depth_renderer.h / silhouette_renderer.h / normal_renderer.h: full renderers ----------------
struct Point2i {  // cv::Point2i: x = column, y = row
  int x = 0, y = 0;
};

// FullDepthRenderer (renderer.h:234-251) over the whole image of its camera, with its own z range. On the device every
// full renderer produces the depth, silhouette and normal images (m3tb_set_full_renderer); StartRendering renders every
// full renderer of the batch in one m3tb_render_full call. The images are those of the last Fetch...Image.
class FullDepthRenderer {
 public:
  virtual ~FullDepthRenderer() = default;
  bool SetUp() {
    set_up_ = false;
    rendered_ = false;
    if (!renderer_geometry_ptr_ || !renderer_geometry_ptr_->set_up()) {
      std::cerr << "Set up renderer geometry of renderer " << name_ << " first" << std::endl;
      return false;
    }
    if (!camera_ptr_ || !camera_ptr_->set_up()) {
      std::cerr << "Set up camera of renderer " << name_ << " first" << std::endl;
      return false;
    }
    std::vector<int> geo;
    for (auto& b : renderer_geometry_ptr_->body_ptrs()) geo.push_back(b->index());
    const int kind = std::dynamic_pointer_cast<ColorCamera>(camera_ptr_) ? 0 : 1;
    if (!Check(batch_->ctx(),
               m3tb_set_full_renderer(batch_->ctx(), index_, kind, camera_ptr_->index(), z_min_, z_max_, int(id_type_),
                                      geo.data(), int(geo.size())),
               "FullRenderer::SetUp"))
      return false;
    intrinsics_ = camera_ptr_->intrinsics();
    // FullDepthRenderer::CalculateProjectionTerms (renderer.cpp:476-477)
    projection_term_a_ = z_max_ * z_min_ * USHRT_MAX_F / (z_max_ - z_min_);
    projection_term_b_ = z_max_ * USHRT_MAX_F / (z_max_ - z_min_);
    set_up_ = true;
    return true;
  }
  // FullRenderer::StartRendering: one m3tb_render_full for every full renderer of the batch
  bool StartRendering() {
    if (!set_up_) {
      std::cerr << "Set up renderer " << name_ << " first" << std::endl;
      return false;
    }
    if (!Check(batch_->ctx(), m3tb_render_full(batch_->ctx()), "FullRenderer::StartRendering")) return false;
    rendered_ = true;
    return true;
  }
  bool FetchDepthImage() { return Fetch(&depth_image_, nullptr, nullptr, "FullDepthRenderer::FetchDepthImage"); }
  const std::vector<uint16_t>& depth_image() const { return depth_image_; }  // height x width, row-major
  // renderer.cpp:431-452
  float Depth(uint16_t depth_image_value) const {
    return projection_term_a_ / (projection_term_b_ - float(depth_image_value));
  }
  float Depth(const Point2i& image_coordinate) const {
    const float depth_image_value = float(DepthImageValue(image_coordinate));
    return projection_term_a_ / (projection_term_b_ - depth_image_value);
  }
  uint16_t DepthImageValue(const Point2i& image_coordinate) const {
    return depth_image_[size_t(image_coordinate.y) * size_t(intrinsics_.width) + size_t(image_coordinate.x)];
  }
  std::array<float, 3> PointVector(const Point2i& image_coordinate) const {
    const float depth_image_value = float(DepthImageValue(image_coordinate));
    const float depth = projection_term_a_ / (projection_term_b_ - depth_image_value);
    return {depth * (image_coordinate.x - intrinsics_.ppu) / intrinsics_.fu,
            depth * (image_coordinate.y - intrinsics_.ppv) / intrinsics_.fv, depth};
  }
  const std::string& name() const { return name_; }
  const std::shared_ptr<Camera>& camera_ptr() const { return camera_ptr_; }
  const Intrinsics& intrinsics() const { return intrinsics_; }
  float z_min() const { return z_min_; }
  float z_max() const { return z_max_; }
  float projection_term_a() const { return projection_term_a_; }
  float projection_term_b() const { return projection_term_b_; }
  void set_z_min(float v) { z_min_ = v; set_up_ = false; }
  void set_z_max(float v) { z_max_ = v; set_up_ = false; }
  bool set_up() const { return set_up_; }
  int index() const { return index_; }
  // FullDepthRenderer::NormalizedDepthImage (renderer.cpp:407-427) of the last render: height x width u8 (empty on
  // failure or before the first render)
  std::vector<uint8_t> NormalizedDepthImage(float min_depth, float max_depth) const {
    std::vector<uint8_t> image(size_t(intrinsics_.width) * size_t(intrinsics_.height));
    if (!set_up_ || !rendered_ ||
        !Check(batch_->ctx(),
               m3tb_get_normalized_depth_image(batch_->ctx(), M3TB_NORMALIZED_DEPTH_FULL_RENDERER, index_, min_depth,
                                               max_depth, image.data(), size_t(intrinsics_.width)),
               "FullDepthRenderer::NormalizedDepthImage"))
      image.clear();
    return image;
  }

 protected:
  static constexpr float USHRT_MAX_F = 65535.0f;
  FullDepthRenderer(const std::string& name, const std::shared_ptr<Batch>& batch,
                    const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr,
                    const std::shared_ptr<Camera>& camera_ptr, IDType id_type, float z_min, float z_max)
      : name_(name), batch_(batch), renderer_geometry_ptr_(renderer_geometry_ptr), camera_ptr_(camera_ptr),
        id_type_(id_type), z_min_(z_min), z_max_(z_max) {
    index_ = batch->NextFullRenderer();
  }
  // one read-back of the last render into the images asked for; fails before SetUp and before the first render
  bool Fetch(std::vector<uint16_t>* depth, std::vector<uint8_t>* silhouette, std::vector<uint8_t>* normal,
             const char* what) {
    if (!set_up_) {
      std::cerr << "Set up renderer " << name_ << " first" << std::endl;
      return false;
    }
    if (!rendered_) {
      std::cerr << "Renderer " << name_ << " has not rendered" << std::endl;
      return false;
    }
    const size_t W = size_t(intrinsics_.width), H = size_t(intrinsics_.height);
    if (depth) depth->resize(W * H);
    if (silhouette) silhouette->resize(W * H);
    if (normal) normal->resize(4 * W * H);
    return Check(batch_->ctx(),
                 m3tb_get_full_rendering(batch_->ctx(), index_, depth ? depth->data() : nullptr, 2 * W,
                                         silhouette ? silhouette->data() : nullptr, W,
                                         normal ? normal->data() : nullptr, 4 * W, nullptr, nullptr),
                 what);
  }
  std::string name_;
  std::shared_ptr<Batch> batch_;
  std::shared_ptr<RendererGeometry> renderer_geometry_ptr_;
  std::shared_ptr<Camera> camera_ptr_;
  IDType id_type_;
  float z_min_, z_max_;
  Intrinsics intrinsics_{};
  float projection_term_a_ = 0.0f, projection_term_b_ = 0.0f;
  int index_ = 0;
  bool set_up_ = false, rendered_ = false;
  std::vector<uint16_t> depth_image_;
  std::vector<uint8_t> silhouette_image_, normal_image_;
};

class FullBasicDepthRenderer : public FullDepthRenderer {
 public:
  FullBasicDepthRenderer(const std::string& name, const std::shared_ptr<Batch>& batch,
                         const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr,
                         const std::shared_ptr<Camera>& camera_ptr, float z_min = 0.02f, float z_max = 10.0f)
      : FullDepthRenderer(name, batch, renderer_geometry_ptr, camera_ptr, IDType::BODY, z_min, z_max) {}
};

class FullSilhouetteRenderer : public FullDepthRenderer {
 public:
  FullSilhouetteRenderer(const std::string& name, const std::shared_ptr<Batch>& batch,
                         const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr,
                         const std::shared_ptr<Camera>& camera_ptr, IDType id_type = IDType::BODY, float z_min = 0.02f,
                         float z_max = 10.0f)
      : FullDepthRenderer(name, batch, renderer_geometry_ptr, camera_ptr, id_type, z_min, z_max) {}
  bool FetchSilhouetteImage() {
    return Fetch(nullptr, &silhouette_image_, nullptr, "FullSilhouetteRenderer::FetchSilhouetteImage");
  }
  const std::vector<uint8_t>& silhouette_image() const { return silhouette_image_; }  // height x width
  uint8_t SilhouetteValue(const Point2i& image_coordinate) const {
    return silhouette_image_[size_t(image_coordinate.y) * size_t(intrinsics_.width) + size_t(image_coordinate.x)];
  }
  IDType id_type() const { return id_type_; }
};

// FullNormalRenderer (normal_renderer.h:81-93) on a full-renderer slot of its own, any z range
class FullNormalRenderer : public FullDepthRenderer {
 public:
  FullNormalRenderer(const std::string& name, const std::shared_ptr<Batch>& batch,
                     const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr,
                     const std::shared_ptr<Camera>& camera_ptr, float z_min = 0.02f, float z_max = 10.0f)
      : FullDepthRenderer(name, batch, renderer_geometry_ptr, camera_ptr, IDType::BODY, z_min, z_max) {}
  bool FetchNormalImage() { return Fetch(nullptr, nullptr, &normal_image_, "FullNormalRenderer::FetchNormalImage"); }
  // BGRA8, height x width, GL_BGRA order (byte 0 encodes x)
  const std::vector<uint8_t>& normal_image() const { return normal_image_; }
};

using Vec4b = std::array<uint8_t, 4>;  // cv::Vec4b

// FocusedNormalRenderer (normal_renderer.h:135-176) on a focused-normal-renderer slot of its own
// (m3tb_set_focused_normal_renderer), with FocusedDepthRenderer's getters. StartRendering renders every focused normal
// renderer of the batch in one m3tb_render_focused_normals call; the images, focus and visible flags are those of the
// last Fetch...Image.
class FocusedNormalRenderer {
 public:
  FocusedNormalRenderer(const std::string& name, const std::shared_ptr<Batch>& batch,
                        const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr,
                        const std::shared_ptr<Camera>& camera_ptr, int image_size = 200, float z_min = 0.02f,
                        float z_max = 10.0f)
      : name_(name), batch_(batch), renderer_geometry_ptr_(renderer_geometry_ptr), camera_ptr_(camera_ptr),
        image_size_(image_size), z_min_(z_min), z_max_(z_max) {
    index_ = batch->NextFocusedNormalRenderer();
  }
  bool AddReferencedBody(const std::shared_ptr<Body>& body_ptr) {
    for (auto& b : referenced_body_ptrs_)
      if (b->name() == body_ptr->name()) {
        std::cerr << "Body " << body_ptr->name() << " already exists" << std::endl;
        return false;
      }
    referenced_body_ptrs_.push_back(body_ptr);
    set_up_ = false;
    return true;
  }
  bool SetUp() {
    set_up_ = false;
    rendered_ = false;
    if (!renderer_geometry_ptr_ || !renderer_geometry_ptr_->set_up()) {
      std::cerr << "Set up renderer geometry of renderer " << name_ << " first" << std::endl;
      return false;
    }
    if (!camera_ptr_ || !camera_ptr_->set_up()) {
      std::cerr << "Set up camera of renderer " << name_ << " first" << std::endl;
      return false;
    }
    if (referenced_body_ptrs_.empty()) {
      std::cerr << "No referenced bodys were assigned to renderer " << name_ << std::endl;
      return false;
    }
    std::vector<int> geo, ref;
    for (auto& b : renderer_geometry_ptr_->body_ptrs()) geo.push_back(b->index());
    for (auto& b : referenced_body_ptrs_) ref.push_back(b->index());
    const int kind = std::dynamic_pointer_cast<ColorCamera>(camera_ptr_) ? 0 : 1;
    if (!Check(batch_->ctx(),
               m3tb_set_focused_normal_renderer(batch_->ctx(), index_, kind, camera_ptr_->index(), image_size_, z_min_,
                                                z_max_, geo.data(), int(geo.size()), ref.data(), int(ref.size())),
               "FocusedNormalRenderer::SetUp"))
      return false;
    // FocusedDepthRenderer::CalculateProjectionTerms (renderer.cpp:567-570)
    projection_term_a_ = z_max_ * z_min_ * 65535.0f / (z_max_ - z_min_);
    projection_term_b_ = z_max_ * 65535.0f / (z_max_ - z_min_);
    set_up_ = true;
    return true;
  }
  bool StartRendering() {
    if (!set_up_) {
      std::cerr << "Set up renderer " << name_ << " first" << std::endl;
      return false;
    }
    if (!Check(batch_->ctx(), m3tb_render_focused_normals(batch_->ctx()), "FocusedNormalRenderer::StartRendering"))
      return false;
    rendered_ = true;
    return true;
  }
  bool FetchNormalImage() { return Fetch("FocusedNormalRenderer::FetchNormalImage"); }
  bool FetchDepthImage() { return Fetch("FocusedNormalRenderer::FetchDepthImage"); }
  // BGRA8, image_size x image_size, GL_BGRA order (byte 0 encodes x)
  const std::vector<uint8_t>& focused_normal_image() const { return normal_; }
  const std::vector<uint16_t>& focused_depth_image() const { return depth_; }
  // normal_renderer.cpp:393-415
  std::array<float, 3> NormalVector(Vec4b normal_image_value) const {
    return {1.0f - float(normal_image_value[0]) / 127.5f, 1.0f - float(normal_image_value[1]) / 127.5f,
            1.0f - float(normal_image_value[2]) / 127.5f};
  }
  std::array<float, 3> NormalVector(const Point2i& image_coordinate) const {
    return NormalVector(NormalImageValue(image_coordinate));
  }
  Vec4b NormalImageValue(const Point2i& image_coordinate) const {
    const int u = int((image_coordinate.x - corner_u_) * scale_ + 0.5f);
    const int v = int((image_coordinate.y - corner_v_) * scale_ + 0.5f);
    const uint8_t* p = normal_.data() + 4 * (size_t(v) * size_t(image_size_) + size_t(u));
    return {p[0], p[1], p[2], p[3]};
  }
  bool IsBodyVisible(const std::string& body_name) const {
    for (size_t k = 0; k < referenced_body_ptrs_.size() && k < visible_.size(); ++k)
      if (referenced_body_ptrs_[k]->name() == body_name) return visible_[k] != 0;
    return false;
  }
  bool IsBodyReferenced(const std::string& body_name) const {
    for (auto& b : referenced_body_ptrs_)
      if (b->name() == body_name) return true;
    return false;
  }
  float corner_u() const { return corner_u_; }
  float corner_v() const { return corner_v_; }
  float scale() const { return scale_; }
  float projection_term_a() const { return projection_term_a_; }
  float projection_term_b() const { return projection_term_b_; }
  int image_size() const { return image_size_; }
  float z_min() const { return z_min_; }
  float z_max() const { return z_max_; }
  void set_image_size(int v) { image_size_ = v; set_up_ = false; }
  void set_z_min(float v) { z_min_ = v; set_up_ = false; }
  void set_z_max(float v) { z_max_ = v; set_up_ = false; }
  bool set_up() const { return set_up_; }
  int index() const { return index_; }
  const std::string& name() const { return name_; }
  const std::shared_ptr<Camera>& camera_ptr() const { return camera_ptr_; }
  const std::vector<std::shared_ptr<Body>>& referenced_body_ptrs() const { return referenced_body_ptrs_; }

 private:
  // one read-back of the last render: both images, the focus and the visible flags; fails before SetUp and before the
  // first render
  bool Fetch(const char* what) {
    if (!set_up_) {
      std::cerr << "Set up renderer " << name_ << " first" << std::endl;
      return false;
    }
    if (!rendered_) {
      std::cerr << "Renderer " << name_ << " has not rendered" << std::endl;
      return false;
    }
    const size_t n = size_t(image_size_) * size_t(image_size_);
    depth_.resize(n);
    normal_.resize(4 * n);
    visible_.assign(referenced_body_ptrs_.size(), 0);
    return Check(batch_->ctx(),
                 m3tb_get_focused_normal_rendering(batch_->ctx(), index_, depth_.data(), normal_.data(), &corner_u_,
                                                   &corner_v_, &scale_, &projection_term_a_, &projection_term_b_,
                                                   visible_.data()),
                 what);
  }
  std::string name_;
  std::shared_ptr<Batch> batch_;
  std::shared_ptr<RendererGeometry> renderer_geometry_ptr_;
  std::shared_ptr<Camera> camera_ptr_;
  std::vector<std::shared_ptr<Body>> referenced_body_ptrs_;
  int image_size_;
  float z_min_, z_max_;
  int index_ = 0;
  bool set_up_ = false, rendered_ = false;
  std::vector<uint16_t> depth_;
  std::vector<uint8_t> normal_;
  std::vector<int> visible_;
  float corner_u_ = 0, corner_v_ = 0, scale_ = 0, projection_term_a_ = 0, projection_term_b_ = 0;
};

// ---- normal_viewer.h -----------------------------------------------------------------------------------------------
// The FullNormalRenderer of a viewer (normal_viewer.h:59,104) over the whole image of its camera. On the device it is
// the renderer of one viewer slot (m3tb_set_viewer); StartRendering renders every viewer of the batch in one
// m3tb_update_viewers call. Only the viewers' z range 0.02 .. 10 is built.
class ViewerNormalRenderer {
 public:
  ViewerNormalRenderer(const std::string& name, const std::shared_ptr<Batch>& batch,
                       const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr,
                       const std::shared_ptr<Camera>& camera_ptr, float z_min = 0.02f, float z_max = 10.0f)
      : name_(name), batch_(batch), renderer_geometry_ptr_(renderer_geometry_ptr), camera_ptr_(camera_ptr), z_min_(z_min),
        z_max_(z_max) {
    index_ = batch->NextViewer();
  }
  bool SetUp() { return SetUpViewer(0.0f, 0.0f, 1.0f); }
  bool StartRendering() {
    if (!set_up_) {
      std::cerr << "Set up renderer " << name_ << " first" << std::endl;
      return false;
    }
    batch_->ViewersUpdated();
    return Check(batch_->ctx(), m3tb_update_viewers(batch_->ctx()), "FullNormalRenderer::StartRendering");
  }
  bool FetchNormalImage() { return Fetch(); }
  // BGRA8, width x height, GL_BGRA order (byte 0 encodes x)
  const std::vector<uint8_t>& normal_image() { Fetch(); return normal_; }
  const std::vector<uint8_t>& blended_image() { Fetch(); return image_; }
  int index() const { return index_; }
  bool set_up() const { return set_up_; }
  const std::shared_ptr<Camera>& camera_ptr() const { return camera_ptr_; }

  // the viewer slot behind the renderer: kind 0 colour / 1 depth camera, the viewer's blend parameters
  bool SetUpViewer(float opacity, float min_depth, float max_depth) {
    set_up_ = false;
    if (z_min_ != 0.02f || z_max_ != 10.0f) {
      std::cerr << "FullNormalRenderer " << name_ << ": only the z range 0.02 .. 10 is built" << std::endl;
      return false;
    }
    std::vector<int> geo;
    for (auto& b : renderer_geometry_ptr_->body_ptrs()) geo.push_back(b->index());
    const int kind = std::dynamic_pointer_cast<ColorCamera>(camera_ptr_) ? 0 : 1;
    if (!Check(batch_->ctx(),
               m3tb_set_viewer(batch_->ctx(), index_, kind, camera_ptr_->index(), geo.data(), int(geo.size()), opacity,
                               min_depth, max_depth),
               "FullNormalRenderer::SetUp"))
      return false;
    set_up_ = true;
    fetched_ = -1;
    return true;
  }

 private:
  bool Fetch() {
    if (fetched_ == batch_->viewer_version()) return true;
    const Intrinsics& in = camera_ptr_->intrinsics();
    normal_.resize(size_t(in.width) * in.height * 4);
    image_.resize(size_t(in.width) * in.height * 3);
    if (!Check(batch_->ctx(),
               m3tb_get_viewer_image(batch_->ctx(), index_, image_.data(), size_t(in.width) * 3, normal_.data(),
                                     size_t(in.width) * 4),
               "FullNormalRenderer::FetchNormalImage"))
      return false;
    fetched_ = batch_->viewer_version();
    return true;
  }
  std::string name_;
  std::shared_ptr<Batch> batch_;
  std::shared_ptr<RendererGeometry> renderer_geometry_ptr_;
  std::shared_ptr<Camera> camera_ptr_;
  float z_min_, z_max_;
  int index_ = 0;
  bool set_up_ = false;
  long fetched_ = -1;  // the batch's viewer version the images below were read at
  std::vector<uint8_t> normal_, image_;
};

// Viewer (viewer.h): SetUp, UpdateViewer, and the image of the last update, read back by image() instead of being
// displayed or saved
class Viewer {
 public:
  virtual ~Viewer() = default;
  virtual bool SetUp() = 0;
  virtual bool UpdateViewer(int save_index) = 0;
  virtual const std::vector<uint8_t>& image() = 0;
  // true for the normal viewers, which m3tb_update_viewers draws all together (Tracker::UpdateViewers)
  virtual bool drawn_by_update_viewers() const { return false; }
  const std::string& name() const { return name_; }
  bool set_up() const { return set_up_; }
  bool dirty() const { return dirty_; }

 protected:
  explicit Viewer(const std::string& name) : name_(name) {}
  std::string name_;
  bool set_up_ = false, dirty_ = false;
};

// The normal viewers (normal_viewer.h): UpdateViewer renders and blends; image() is the blended BGR8 image
class NormalViewer : public Viewer {
 public:
  // UpdateViewer(save_index): one m3tb_update_viewers for every normal viewer of the batch
  bool UpdateViewer(int /*save_index*/) override {
    if (!set_up_) {
      std::cerr << "Set up viewer " << name_ << " first" << std::endl;
      return false;
    }
    if (dirty_ && !SetUp()) return false;
    return renderer_.StartRendering();
  }
  // the image CalculateAlphaBlend returned at the last update: width x height BGR8
  const std::vector<uint8_t>& image() override { return renderer_.blended_image(); }
  bool drawn_by_update_viewers() const override { return true; }
  ViewerNormalRenderer& renderer() { return renderer_; }
  void set_opacity(float opacity) { opacity_ = opacity; dirty_ = true; }
  float opacity() const { return opacity_; }

 protected:
  NormalViewer(const std::string& name, const std::shared_ptr<Batch>& batch,
               const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr, const std::shared_ptr<Camera>& camera_ptr,
               float opacity)
      : Viewer(name), renderer_("renderer", batch, renderer_geometry_ptr, camera_ptr), opacity_(opacity) {}
  bool SetUpWith(float min_depth, float max_depth) {
    set_up_ = false;
    if (!renderer_.camera_ptr()->set_up()) {
      std::cerr << "Camera " << renderer_.camera_ptr()->name() << " was not set up" << std::endl;
      return false;
    }
    if (!renderer_.SetUpViewer(opacity_, min_depth, max_depth)) return false;
    set_up_ = true;
    dirty_ = false;
    return true;
  }
  ViewerNormalRenderer renderer_;
  float opacity_;
};

class NormalColorViewer : public NormalViewer {
 public:
  NormalColorViewer(const std::string& name, const std::shared_ptr<Batch>& batch,
                    const std::shared_ptr<ColorCamera>& color_camera_ptr,
                    const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr, float opacity = 0.5f)
      : NormalViewer(name, batch, renderer_geometry_ptr, color_camera_ptr, opacity) {}
  bool SetUp() override { return SetUpWith(0.0f, 1.0f); }
};

class NormalDepthViewer : public NormalViewer {
 public:
  NormalDepthViewer(const std::string& name, const std::shared_ptr<Batch>& batch,
                    const std::shared_ptr<DepthCamera>& depth_camera_ptr,
                    const std::shared_ptr<RendererGeometry>& renderer_geometry_ptr, float min_depth = 0.0f,
                    float max_depth = 1.0f, float opacity = 0.5f)
      : NormalViewer(name, batch, renderer_geometry_ptr, depth_camera_ptr, opacity), min_depth_(min_depth),
        max_depth_(max_depth) {}
  bool SetUp() override { return SetUpWith(min_depth_, max_depth_); }
  void set_min_depth(float v) { min_depth_ = v; dirty_ = true; }
  void set_max_depth(float v) { max_depth_ = v; dirty_ = true; }

 private:
  float min_depth_, max_depth_;
};

// ImageColorViewer (image_viewer.cpp:9-35): image() is the frame the colour camera holds (Camera::image()), width x
// height BGR8, read at each UpdateViewer
class ImageColorViewer : public Viewer {
 public:
  ImageColorViewer(const std::string& name, const std::shared_ptr<ColorCamera>& color_camera_ptr)
      : Viewer(name), color_camera_ptr_(color_camera_ptr) {}
  bool SetUp() override {
    set_up_ = false;
    if (!color_camera_ptr_->set_up()) {
      std::cerr << "Color camera " << color_camera_ptr_->name() << " was not set up" << std::endl;
      return false;
    }
    set_up_ = true;
    return true;
  }
  bool UpdateViewer(int /*save_index*/) override {
    if (!set_up_) {
      std::cerr << "Set up image color viewer " << name_ << " first" << std::endl;
      return false;
    }
    const Intrinsics& in = color_camera_ptr_->intrinsics();
    image_.resize(size_t(in.width) * size_t(in.height) * 3);
    const auto& batch = color_camera_ptr_->batch();
    return Check(batch->ctx(),
                 m3tb_get_camera_image(batch->ctx(), 0, color_camera_ptr_->index(), image_.data(), size_t(in.width) * 3),
                 "ImageColorViewer::UpdateViewer");
  }
  const std::vector<uint8_t>& image() override { return image_; }

 private:
  std::shared_ptr<ColorCamera> color_camera_ptr_;
  std::vector<uint8_t> image_;
};

// ImageDepthViewer (image_viewer.cpp:50-78): image() is DepthCamera::NormalizedDepthImage(min_depth, max_depth) of the
// frame the depth camera holds, width x height u8, computed at each UpdateViewer
class ImageDepthViewer : public Viewer {
 public:
  ImageDepthViewer(const std::string& name, const std::shared_ptr<DepthCamera>& depth_camera_ptr, float min_depth = 0.0f,
                   float max_depth = 1.0f)
      : Viewer(name), depth_camera_ptr_(depth_camera_ptr), min_depth_(min_depth), max_depth_(max_depth) {}
  bool SetUp() override {
    set_up_ = false;
    if (!depth_camera_ptr_->set_up()) {
      std::cerr << "Depth camera " << depth_camera_ptr_->name() << " was not set up" << std::endl;
      return false;
    }
    set_up_ = true;
    return true;
  }
  bool UpdateViewer(int /*save_index*/) override {
    if (!set_up_) {
      std::cerr << "Set up image depth viewer " << name_ << " first" << std::endl;
      return false;
    }
    image_ = depth_camera_ptr_->NormalizedDepthImage(min_depth_, max_depth_);
    return !image_.empty();
  }
  const std::vector<uint8_t>& image() override { return image_; }
  void set_min_depth(float v) { min_depth_ = v; }
  void set_max_depth(float v) { max_depth_ = v; }
  float min_depth() const { return min_depth_; }
  float max_depth() const { return max_depth_; }

 private:
  std::shared_ptr<DepthCamera> depth_camera_ptr_;
  float min_depth_, max_depth_;
  std::vector<uint8_t> image_;
};

// ---- modality.h ----------------------------------------------------------------------------------------------------
class Modality {
 public:
  virtual ~Modality() = default;
  virtual bool SetUp() = 0;
  virtual bool StartModality(int iteration, int corr_iteration) = 0;
  virtual bool CalculateCorrespondences(int iteration, int corr_iteration) = 0;
  virtual bool CalculateGradientAndHessian(int iteration, int corr_iteration, int opt_iteration) = 0;
  virtual bool CalculateResults(int iteration) = 0;
  const std::array<float, 6>& gradient() const { return gradient_; }
  const std::array<float, 36>& hessian() const { return hessian_; }
  const std::string& name() const { return name_; }
  const std::shared_ptr<Body>& body_ptr() const { return body_ptr_; }
  bool set_up() const { return set_up_; }
  // Modality::correspondence_renderer_ptrs (modality.h): what Tracker renders before CalculateCorrespondences
  virtual std::vector<std::shared_ptr<FocusedDepthRenderer>> correspondence_renderer_ptrs() const {
    std::vector<std::shared_ptr<FocusedDepthRenderer>> out;
    if (depth_renderer_ptr_) out.push_back(depth_renderer_ptr_);
    if (silhouette_renderer_ptr_) out.push_back(silhouette_renderer_ptr_);
    return out;
  }
  const std::shared_ptr<FocusedDepthRenderer>& depth_renderer_ptr() const { return depth_renderer_ptr_; }
  const std::shared_ptr<FocusedSilhouetteRenderer>& silhouette_renderer_ptr() const { return silhouette_renderer_ptr_; }

 protected:
  // RegionModality / DepthModality::SetUp checks on the renderers (region_modality.cpp:50-86, depth_modality.cpp:45-76)
  bool CheckRenderers(IDType silhouette_id_type) const {
    for (auto& r : correspondence_renderer_ptrs()) {
      if (!r->set_up()) {
        std::cerr << "Focused renderer " << r->name() << " was not set up" << std::endl;
        return false;
      }
      if (!r->IsBodyReferenced(body_ptr_->name())) {
        std::cerr << "Focused renderer " << r->name() << " does not reference body " << body_ptr_->name() << std::endl;
        return false;
      }
    }
    if (silhouette_renderer_ptr_ && silhouette_renderer_ptr_->id_type() != silhouette_id_type) {
      std::cerr << "Focused silhouette renderer " << silhouette_renderer_ptr_->name() << " does not use id_type "
                << (silhouette_id_type == IDType::REGION ? "REGION" : "BODY") << std::endl;
      return false;
    }
    return true;
  }
  std::shared_ptr<FocusedDepthRenderer> depth_renderer_ptr_;
  std::shared_ptr<FocusedSilhouetteRenderer> silhouette_renderer_ptr_;
  Modality(const std::string& name, const std::shared_ptr<Batch>& batch, const std::shared_ptr<Body>& body_ptr)
      : name_(name), batch_(batch), body_ptr_(body_ptr) {}
  bool IsSetup() const {
    if (!set_up_) std::cerr << "Set up modality " << name_ << " first" << std::endl;
    return set_up_;
  }
  void FetchGH(const std::vector<float>& g, const std::vector<float>& h) {
    const int b = body_ptr_->index();
    std::memcpy(gradient_.data(), g.data() + 6 * b, sizeof(float) * 6);
    std::memcpy(hessian_.data(), h.data() + 36 * b, sizeof(float) * 36);
  }
  std::string name_;
  std::shared_ptr<Batch> batch_;
  std::shared_ptr<Body> body_ptr_;
  std::array<float, 6> gradient_{};
  std::array<float, 36> hessian_{};
  bool set_up_ = false;
  friend class Optimizer;
};

// ---- region_modality.h --------------------------------------------------------------------------------------------
// ---- color_histograms.h: only what a SHARED object needs (a modality's own histograms live with its body) ---------------
// The object's n_bins and learning rates (color_histograms.h:38-45) stand for those of every modality that uses it; on
// the device they are the parameters of the owner, the body of the first modality the object was given to.
class ColorHistograms {
 public:
  explicit ColorHistograms(const std::string& name, int n_bins = 16, float learning_rate_f = 0.2f, float learning_rate_b = 0.2f)
      : name_(name), n_bins_(n_bins), learning_rate_f_(learning_rate_f), learning_rate_b_(learning_rate_b) {}
  const std::string& name() const { return name_; }
  void set_n_bins(int v) { n_bins_ = v; }
  void set_learning_rate_f(float v) { learning_rate_f_ = v; }
  void set_learning_rate_b(float v) { learning_rate_b_ = v; }
  int n_bins() const { return n_bins_; }
  float learning_rate_f() const { return learning_rate_f_; }
  float learning_rate_b() const { return learning_rate_b_; }
  bool SetUp() { set_up_ = true; return true; }
  bool set_up() const { return set_up_; }
  int owner_body() const { return owner_body_; }
  void claim_owner(int body) { if (owner_body_ < 0) owner_body_ = body; }

 private:
  std::string name_;
  int n_bins_;
  float learning_rate_f_, learning_rate_b_;
  bool set_up_ = false;
  int owner_body_ = -1;
};

class RegionModality : public Modality {
 public:
  RegionModality(const std::string& name, const std::shared_ptr<Batch>& batch, const std::shared_ptr<Body>& body_ptr,
                 const std::shared_ptr<ColorCamera>& color_camera_ptr, const std::shared_ptr<RegionModel>& region_model_ptr)
      : Modality(name, batch, body_ptr), color_camera_ptr_(color_camera_ptr), region_model_ptr_(region_model_ptr) {
    m3tb_region_params_default(&params_);
  }
  // setters of the reference (region_modality.h:196-260), same names
  void set_n_lines_max(int v) { params_.n_lines_max = v; set_up_ = false; }
  void set_min_continuous_distance(float v) { params_.min_continuous_distance = v; set_up_ = false; }
  void set_function_amplitude(float v) { params_.function_amplitude = v; set_up_ = false; }
  void set_function_slope(float v) { params_.function_slope = v; set_up_ = false; }
  void set_learning_rate(float v) { params_.learning_rate = v; set_up_ = false; }
  void set_n_global_iterations(int v) { params_.n_global_iterations = v; set_up_ = false; }
  void set_scales(const std::vector<int>& v) {
    params_.n_scales = int(v.size());
    for (size_t i = 0; i < v.size() && i < M3TB_MAX_SCHEDULE; ++i) params_.scales[i] = v[i];
    set_up_ = false;
  }
  void set_standard_deviations(const std::vector<float>& v) {
    params_.n_standard_deviations = int(v.size());
    for (size_t i = 0; i < v.size() && i < M3TB_MAX_SCHEDULE; ++i) params_.standard_deviations[i] = v[i];
    set_up_ = false;
  }
  // region_modality.cpp:168-203: with a shared ColorHistograms object the three histogram parameters are the object's
  void UseSharedColorHistograms(const std::shared_ptr<ColorHistograms>& color_histograms_ptr) {
    color_histograms_ptr_ = color_histograms_ptr;
    set_up_ = false;
  }
  void DoNotUseSharedColorHistograms() { color_histograms_ptr_ = nullptr; set_up_ = false; }
  // region_modality.cpp:230-267 with a device renderer (DESIGN.md "k_render")
  void ModelOcclusions(const std::shared_ptr<FocusedDepthRenderer>& depth_renderer_ptr) {
    depth_renderer_ptr_ = depth_renderer_ptr; params_.model_occlusions = 1; set_up_ = false;
  }
  void DoNotModelOcclusions() { depth_renderer_ptr_ = nullptr; params_.model_occlusions = 0; set_up_ = false; }
  void UseRegionChecking(const std::shared_ptr<FocusedSilhouetteRenderer>& silhouette_renderer_ptr) {
    silhouette_renderer_ptr_ = silhouette_renderer_ptr; params_.use_region_checking = 1; set_up_ = false;
  }
  void DoNotUseRegionChecking() { silhouette_renderer_ptr_ = nullptr; params_.use_region_checking = 0; set_up_ = false; }
  void set_n_unoccluded_iterations(int v) { params_.n_unoccluded_iterations = v; set_up_ = false; }
  const std::shared_ptr<ColorHistograms>& color_histograms_ptr() const { return color_histograms_ptr_; }
  bool set_n_histogram_bins(int v) {
    if (color_histograms_ptr_) { std::cerr << "Modality " << name_ << " uses shared color histograms" << std::endl; return false; }
    params_.n_histogram_bins = v; set_up_ = false; return true;
  }
  bool set_learning_rate_f(float v) {
    if (color_histograms_ptr_) { std::cerr << "Modality " << name_ << " uses shared color histograms" << std::endl; return false; }
    params_.learning_rate_f = v; set_up_ = false; return true;
  }
  bool set_learning_rate_b(float v) {
    if (color_histograms_ptr_) { std::cerr << "Modality " << name_ << " uses shared color histograms" << std::endl; return false; }
    params_.learning_rate_b = v; set_up_ = false; return true;
  }
  void set_unconsidered_line_length(float v) { params_.unconsidered_line_length = v; set_up_ = false; }
  void set_max_considered_line_length(float v) { params_.max_considered_line_length = v; set_up_ = false; }
  const m3tb_region_params& params() const { return params_; }
  const std::shared_ptr<ColorCamera>& color_camera_ptr() const { return color_camera_ptr_; }
  const std::shared_ptr<RegionModel>& region_model_ptr() const { return region_model_ptr_; }

  bool SetUp() override {  // the body's device record is written by Optimizer::SetUp
    if (!CheckRenderers(IDType::REGION)) return false;
    if (color_histograms_ptr_) {
      if (!color_histograms_ptr_->set_up()) {
        std::cerr << "Color histograms " << color_histograms_ptr_->name() << " was not set up" << std::endl;
        return false;
      }
      params_.n_histogram_bins = color_histograms_ptr_->n_bins();
      params_.learning_rate_f = color_histograms_ptr_->learning_rate_f();
      params_.learning_rate_b = color_histograms_ptr_->learning_rate_b();
    }
    set_up_ = true;
    return true;
  }
  bool StartModality(int iteration, int corr_iteration) override {
    if (!IsSetup()) return false;
    (void)corr_iteration;
    if (!batch_->Claim(Batch::kStart, iteration, 0, 0)) return true;
    return Check(batch_->ctx(), m3tb_start_modalities(batch_->ctx(), iteration), "RegionModality::StartModality");
  }
  bool CalculateCorrespondences(int iteration, int corr_iteration) override {
    if (!IsSetup()) return false;
    if (!batch_->Claim(Batch::kRegionCorr, iteration, corr_iteration, 0)) return true;
    return Check(batch_->ctx(), m3tb_region_correspondences(batch_->ctx(), iteration, corr_iteration),
                 "RegionModality::CalculateCorrespondences");
  }
  bool CalculateGradientAndHessian(int iteration, int corr_iteration, int opt_iteration) override {
    if (!IsSetup()) return false;
    if (batch_->Claim(Batch::kRegionGH, iteration, corr_iteration, opt_iteration)) {
      batch_->region_g.resize(size_t(6) * batch_->n_bodies());
      batch_->region_h.resize(size_t(36) * batch_->n_bodies());
      if (!Check(batch_->ctx(),
                 m3tb_region_gradient_hessian(batch_->ctx(), iteration, corr_iteration, opt_iteration,
                                              batch_->region_g.data(), batch_->region_h.data()),
                 "RegionModality::CalculateGradientAndHessian"))
        return false;
    }
    FetchGH(batch_->region_g, batch_->region_h);
    return true;
  }
  bool CalculateResults(int iteration) override {
    if (!IsSetup()) return false;
    if (!batch_->Claim(Batch::kResults, iteration, 0, 0)) return true;
    return Check(batch_->ctx(), m3tb_calculate_results(batch_->ctx(), iteration), "RegionModality::CalculateResults");
  }

 private:
  m3tb_region_params params_;
  std::shared_ptr<ColorCamera> color_camera_ptr_;
  std::shared_ptr<RegionModel> region_model_ptr_;
  std::shared_ptr<ColorHistograms> color_histograms_ptr_;  // null: the modality's own histograms
};

// ---- depth_modality.h ----------------------------------------------------------------------------------------------
class DepthModality : public Modality {
 public:
  DepthModality(const std::string& name, const std::shared_ptr<Batch>& batch, const std::shared_ptr<Body>& body_ptr,
                const std::shared_ptr<DepthCamera>& depth_camera_ptr, const std::shared_ptr<DepthModel>& depth_model_ptr)
      : Modality(name, batch, body_ptr), depth_camera_ptr_(depth_camera_ptr), depth_model_ptr_(depth_model_ptr) {
    m3tb_depth_params_default(&params_);
  }
  void set_n_points_max(int v) { params_.n_points_max = v; set_up_ = false; }
  // Each value must be finite and positive (refused here, whatever the order of the calls); SetUp refuses a schedule
  // whose considered distances are not at least half the stride length, as m3tb_set_body does.
  bool set_stride_length(float v) {
    if (!(v > 0.0f) || !std::isfinite(v)) return Refuse("stride_length must be finite and positive");
    params_.stride_length = v; set_up_ = false; return true;
  }
  bool set_considered_distances(const std::vector<float>& v) {
    for (float d : v)
      if (!(d > 0.0f) || !std::isfinite(d)) return Refuse("considered distances must be finite and positive");
    params_.n_considered_distances = int(v.size());
    for (size_t i = 0; i < v.size() && i < M3TB_MAX_SCHEDULE; ++i) params_.considered_distances[i] = v[i];
    set_up_ = false;
    return true;
  }
  void set_standard_deviations(const std::vector<float>& v) {
    params_.n_standard_deviations = int(v.size());
    for (size_t i = 0; i < v.size() && i < M3TB_MAX_SCHEDULE; ++i) params_.standard_deviations[i] = v[i];
    set_up_ = false;
  }
  // depth_modality.cpp:128-161 with a device renderer (DESIGN.md "k_render")
  void ModelOcclusions(const std::shared_ptr<FocusedDepthRenderer>& depth_renderer_ptr) {
    depth_renderer_ptr_ = depth_renderer_ptr; params_.model_occlusions = 1; set_up_ = false;
  }
  void DoNotModelOcclusions() { depth_renderer_ptr_ = nullptr; params_.model_occlusions = 0; set_up_ = false; }
  void UseSilhouetteChecking(const std::shared_ptr<FocusedSilhouetteRenderer>& silhouette_renderer_ptr) {
    silhouette_renderer_ptr_ = silhouette_renderer_ptr; params_.use_silhouette_checking = 1; set_up_ = false;
  }
  void DoNotUseSilhouetteChecking() { silhouette_renderer_ptr_ = nullptr; params_.use_silhouette_checking = 0; set_up_ = false; }
  void set_n_unoccluded_iterations(int v) { params_.n_unoccluded_iterations = v; set_up_ = false; }
  const m3tb_depth_params& params() const { return params_; }
  const std::shared_ptr<DepthCamera>& depth_camera_ptr() const { return depth_camera_ptr_; }
  const std::shared_ptr<DepthModel>& depth_model_ptr() const { return depth_model_ptr_; }

  bool SetUp() override {
    const int n = std::min(params_.n_considered_distances, int(M3TB_MAX_SCHEDULE));
    for (int k = 0; k < n; ++k) {  // max_n_strides_ = int(d / stride_length + 0.5f) must lie in [1, 2^31)
      const float strides = params_.considered_distances[k] / params_.stride_length + 0.5f;
      if (!(strides >= 1.0f) || !(strides < 2147483648.0f))
        return Refuse("considered distances must be at least half the stride length and under 2^31 strides");
    }
    if (!CheckRenderers(IDType::BODY)) return false;
    set_up_ = true;
    return true;
  }
  bool StartModality(int, int) override { return IsSetup(); }  // depth_modality.cpp:248-250
  bool CalculateCorrespondences(int iteration, int corr_iteration) override {
    if (!IsSetup()) return false;
    if (!batch_->Claim(Batch::kDepthCorr, iteration, corr_iteration, 0)) return true;
    return Check(batch_->ctx(), m3tb_depth_correspondences(batch_->ctx(), iteration, corr_iteration),
                 "DepthModality::CalculateCorrespondences");
  }
  bool CalculateGradientAndHessian(int iteration, int corr_iteration, int opt_iteration) override {
    if (!IsSetup()) return false;
    if (batch_->Claim(Batch::kDepthGH, iteration, corr_iteration, opt_iteration)) {
      batch_->depth_g.resize(size_t(6) * batch_->n_bodies());
      batch_->depth_h.resize(size_t(36) * batch_->n_bodies());
      if (!Check(batch_->ctx(),
                 m3tb_depth_gradient_hessian(batch_->ctx(), iteration, corr_iteration, opt_iteration,
                                             batch_->depth_g.data(), batch_->depth_h.data()),
                 "DepthModality::CalculateGradientAndHessian"))
        return false;
    }
    FetchGH(batch_->depth_g, batch_->depth_h);
    return true;
  }
  bool CalculateResults(int) override { return IsSetup(); }  // depth_modality.cpp:393

 private:
  bool Refuse(const char* what) const {
    std::cerr << "Modality " << name_ << ": " << what << std::endl;
    return false;
  }
  m3tb_depth_params params_;
  std::shared_ptr<DepthCamera> depth_camera_ptr_;
  std::shared_ptr<DepthModel> depth_model_ptr_;
};

// ---- texture_modality.h ------------------------------------------------------------------------------------------------
// No OpenCV here. For ORB bodies DetectFeatures runs DetectAndComputeCorrKeypoints on the device (cv::ORB at the
// orb_* settings, m3tb_texture_detect_orb). Otherwise the caller asks for the body's focus region with CalculateFocus,
// detects features in the cropped and scaled grey image and hands them over with SetFeatures, once per frame.
// DescriptorType ORB (32-byte descriptors), BRISK and FREAK (64-byte descriptors), SIFT and DAISY (float descriptors)
// are implemented; ORB_CUDA is not.
class TextureModality : public Modality {
 public:
  enum class DescriptorType { BRISK = 0, DAISY = 1, FREAK = 2, SIFT = 3, ORB = 4, ORB_CUDA = 5 };  // texture_modality.h

  TextureModality(const std::string& name, const std::shared_ptr<Batch>& batch, const std::shared_ptr<Body>& body_ptr,
                  const std::shared_ptr<ColorCamera>& color_camera_ptr,
                  const std::shared_ptr<FocusedSilhouetteRenderer>& silhouette_renderer_ptr)
      : Modality(name, batch, body_ptr), color_camera_ptr_(color_camera_ptr) {
    silhouette_renderer_ptr_ = silhouette_renderer_ptr;
    m3tb_texture_params_default(&params_);
    m3tb_orb_params_default(&orb_params_);
  }
  // setters of the reference (texture_modality.h:186-194, 218-226), same names
  void set_descriptor_type(DescriptorType v) { descriptor_type_ = v; set_up_ = false; }
  void set_focused_image_size(int v) { params_.focused_image_size = v; set_up_ = false; }
  void set_descriptor_distance_threshold(float v) { params_.descriptor_distance_threshold = v; set_up_ = false; }
  void set_tukey_norm_constant(float v) { params_.tukey_norm_constant = v; set_up_ = false; }
  void set_standard_deviations(const std::vector<float>& v) {
    params_.n_standard_deviations = int(v.size());
    for (size_t i = 0; i < v.size() && i < M3TB_MAX_SCHEDULE; ++i) params_.standard_deviations[i] = v[i];
    set_up_ = false;
  }
  void set_max_keyframe_rotation_difference(float v) { params_.max_keyframe_rotation_difference = v; set_up_ = false; }
  void set_max_keyframe_age(int v) { params_.max_keyframe_age = v; set_up_ = false; }
  void set_n_keyframes(int v) { params_.n_keyframes = v; set_up_ = false; }
  void MeasureOcclusions(const std::shared_ptr<DepthCamera>& depth_camera_ptr) {
    depth_camera_ptr_ = depth_camera_ptr; params_.measure_occlusions = 1; set_up_ = false;
  }
  void DoNotMeasureOcclusions() { depth_camera_ptr_ = nullptr; params_.measure_occlusions = 0; set_up_ = false; }
  void ModelOcclusions(const std::shared_ptr<FocusedDepthRenderer>& depth_renderer_ptr) {
    depth_renderer_ptr_ = depth_renderer_ptr; params_.model_occlusions = 1; set_up_ = false;
  }
  void DoNotModelOcclusions() { depth_renderer_ptr_ = nullptr; params_.model_occlusions = 0; set_up_ = false; }
  void set_measured_occlusion_radius(float v) { params_.measured_occlusion_radius = v; set_up_ = false; }
  void set_measured_occlusion_threshold(float v) { params_.measured_occlusion_threshold = v; set_up_ = false; }
  void set_modeled_occlusion_radius(float v) { params_.modeled_occlusion_radius = v; set_up_ = false; }
  void set_modeled_occlusion_threshold(float v) { params_.modeled_occlusion_threshold = v; set_up_ = false; }
  // the detector settings of the reference (texture_modality.h:410-412: 300, 1.2, 3), used by DetectFeatures
  void set_orb_n_features(int v) { orb_params_.n_features = v; set_up_ = false; }
  void set_orb_scale_factor(float v) { orb_params_.scale_factor = v; set_up_ = false; }
  void set_orb_n_levels(int v) { orb_params_.n_levels = v; set_up_ = false; }
  int orb_n_features() const { return orb_params_.n_features; }
  float orb_scale_factor() const { return orb_params_.scale_factor; }
  int orb_n_levels() const { return orb_params_.n_levels; }
  const m3tb_orb_params& orb_params() const { return orb_params_; }
  // A device capacity the reference does not have: the most features SetFeatures may hand over per frame, 512 (the
  // default) .. 4096. It sizes the context's texture tables (m3tb_texture_params::n_features_max).
  void set_n_features_max(int v) { params_.n_features_max = v; set_up_ = false; }
  int n_features_max() const { return params_.n_features_max; }
  DescriptorType descriptor_type() const { return descriptor_type_; }
  static const char* DescriptorName(DescriptorType type) {
    static const char* const names[] = {"BRISK", "DAISY", "FREAK", "SIFT", "ORB", "ORB_CUDA"};
    return int(type) >= 0 && int(type) < 6 ? names[int(type)] : "unknown";
  }
  const m3tb_texture_params& params() const { return params_; }
  const std::shared_ptr<ColorCamera>& color_camera_ptr() const { return color_camera_ptr_; }
  const std::shared_ptr<DepthCamera>& depth_camera_ptr() const { return depth_camera_ptr_; }
  // the texture modality renders only for StartModality / CalculateResults (texture_modality.h)
  std::vector<std::shared_ptr<FocusedDepthRenderer>> correspondence_renderer_ptrs() const override { return {}; }

  // TextureModality::SetUp (texture_modality.cpp:39-88); the body's device record is written by Optimizer::SetUp
  bool SetUp() override {
    set_up_ = false;
    if (descriptor_type_ == DescriptorType::ORB_CUDA) {
      std::cerr << "Modality " << name_ << ": DescriptorType::ORB_CUDA is not implemented" << std::endl;
      return false;
    }
    if (!silhouette_renderer_ptr_) {
      std::cerr << "Modality " << name_ << " has no focused silhouette renderer" << std::endl;
      return false;
    }
    if (!color_camera_ptr_) {
      std::cerr << "Modality " << name_ << " has no color camera" << std::endl;
      return false;
    }
    if (params_.measure_occlusions && !depth_camera_ptr_) {
      std::cerr << "Modality " << name_ << " measures occlusions without a depth camera" << std::endl;
      return false;
    }
    for (auto* r : {static_cast<FocusedDepthRenderer*>(silhouette_renderer_ptr_.get()), depth_renderer_ptr_.get()}) {
      if (!r) continue;
      if (!r->set_up()) {
        std::cerr << "Focused renderer " << r->name() << " was not set up" << std::endl;
        return false;
      }
      if (!r->IsBodyReferenced(body_ptr_->name())) {
        std::cerr << "Focused renderer " << r->name() << " does not reference body " << body_ptr_->name() << std::endl;
        return false;
      }
    }
    if (silhouette_renderer_ptr_->id_type() != IDType::BODY) {
      std::cerr << "Focused silhouette renderer " << silhouette_renderer_ptr_->name() << " does not use id_type BODY"
                << std::endl;
      return false;
    }
    params_.descriptor_type = int32_t(descriptor_type_);
    set_up_ = true;
    return true;
  }

  // The caller's detection hook. CalculateFocus: CalculateScaleAndRegionOfInterest from the current device pose,
  // roi = (x, y, width, height) of the crop and the factor it is resized by; false when the reference skips detection.
  bool CalculateFocus(std::array<int32_t, 4>* roi, float* scale) {
    int32_t valid = 0;
    if (!Check(batch_->ctx(), m3tb_get_texture_focus(batch_->ctx(), body_ptr_->index(), 1, roi->data(), scale, &valid),
               "TextureModality::CalculateFocus"))
      return false;
    return valid != 0;
  }
  // SetFeatures: the keypoints (x, y in crop coordinates, keypoints_xy[2 n]) and binary descriptors detected in the
  // crop of CalculateFocus: 32 bytes each for ORB (descriptors[32 n]), 64 for BRISK and FREAK (descriptors[64 n])
  bool SetFeatures(const std::vector<float>& keypoints_xy, const std::vector<uint8_t>& descriptors,
                   const std::array<int32_t, 4>& roi, float scale) {
    const int n = int(keypoints_xy.size() / 2);
    const size_t width = descriptor_type_ == DescriptorType::BRISK || descriptor_type_ == DescriptorType::FREAK ? 64 : 32;
    if (descriptors.size() != width * n) {
      std::cerr << "Modality " << name_ << ": one " << width << "-byte " << DescriptorName(descriptor_type_)
                << " descriptor per keypoint" << std::endl;
      return false;
    }
    return Check(batch_->ctx(),
                 m3tb_upload_texture_features(batch_->ctx(), body_ptr_->index(), keypoints_xy.data(), descriptors.data(), n,
                                              roi[0], roi[1], scale),
                 "TextureModality::SetFeatures");
  }
  // SetFeatures for SIFT and DAISY: `length` floats per keypoint (descriptors[length n]); 128 for SIFT, 1 .. 256 for
  // DAISY, the same length for every frame until SetUp runs again
  bool SetFeatures(const std::vector<float>& keypoints_xy, const std::vector<float>& descriptors, int length,
                   const std::array<int32_t, 4>& roi, float scale) {
    const int n = int(keypoints_xy.size() / 2);
    if (length < 1 || descriptors.size() != size_t(length) * n) {
      std::cerr << "Modality " << name_ << ": one descriptor of `length` floats per keypoint" << std::endl;
      return false;
    }
    return Check(batch_->ctx(),
                 m3tb_upload_texture_float_features(batch_->ctx(), body_ptr_->index(), keypoints_xy.data(),
                                                    descriptors.data(), n, length, roi[0], roi[1], scale),
                 "TextureModality::SetFeatures");
  }
  // The device crops of several texture modalities of one Batch in ONE m3tb_texture_crop call (one pose download, one
  // stream synchronisation, one launch per 128 bodies): modality k's focused grey image of CalculateFocus's region
  // (cvtColor BGR2GRAY, roi, resize by scale, bit-exact against OpenCV) at d_out + k * body_stride in device memory,
  // rows `pitch` bytes apart; per modality its roi, scale, size (width, height) and whether it has a focus. Each crop
  // also records the focus that SetFeatures(const m3tb_device_features&) uses. False on an error, e.g. a crop larger
  // than capacity_width x capacity_height (sizes are still filled then).
  static bool CropFocusedImages(const std::vector<std::shared_ptr<TextureModality>>& modalities, uint8_t* d_out,
                                size_t pitch, size_t body_stride, int capacity_width, int capacity_height,
                                std::vector<std::array<int32_t, 4>>* rois, std::vector<float>* scales,
                                std::vector<std::array<int32_t, 2>>* sizes, std::vector<char>* valid) {
    const size_t n = modalities.size();
    rois->assign(n, {});
    scales->assign(n, 0.0f);
    sizes->assign(n, {});
    valid->assign(n, 0);
    if (n == 0) return true;
    m3tb_ctx* ctx = modalities[0]->batch_->ctx();
    std::vector<int> bodies;
    for (auto& m : modalities) {
      if (m->batch_->ctx() != ctx) {
        std::cerr << "TextureModality::CropFocusedImages: the modalities belong to different batches" << std::endl;
        return false;
      }
      bodies.push_back(m->body_ptr_->index());
    }
    std::vector<int32_t> roi(4 * n), size(2 * n), ok(n);
    const bool done = Check(ctx, m3tb_texture_crop(ctx, bodies.data(), int(n), d_out, pitch, body_stride, capacity_width,
                                                   capacity_height, roi.data(), scales->data(), size.data(), ok.data()),
                            "TextureModality::CropFocusedImages");
    for (size_t k = 0; k < n; ++k) {
      for (int c = 0; c < 4; ++c) (*rois)[k][c] = roi[4 * k + c];
      (*sizes)[k] = {size[2 * k], size[2 * k + 1]};
      (*valid)[k] = ok[k] != 0;
    }
    return done;
  }
  // One modality's device crop; each call synchronises the stream, so several bodies go through CropFocusedImages
  bool CropFocusedImage(uint8_t* d_out, size_t pitch, int capacity_width, int capacity_height,
                        std::array<int32_t, 2>* size) {
    std::vector<std::array<int32_t, 4>> rois;
    std::vector<float> scales;
    std::vector<std::array<int32_t, 2>> sizes;
    std::vector<char> valid;
    std::vector<std::shared_ptr<TextureModality>> self{std::shared_ptr<TextureModality>(this, [](TextureModality*) {})};
    if (!CropFocusedImages(self, d_out, pitch, pitch * size_t(capacity_height), capacity_width, capacity_height, &rois,
                           &scales, &sizes, &valid))
      return false;
    *size = sizes[0];
    return valid[0] != 0;
  }
  // SetFeatures from device memory (e.g. cv::cuda::ORB's GpuMat keypoints and descriptors) in the crop of the last
  // CropFocusedImage(s); does not synchronise. A non-finite float descriptor drops the frame's features on the device;
  // the Batch reports it at the next synchronising read.
  bool SetFeatures(const m3tb_device_features& features) {
    const int body = body_ptr_->index();
    if (!Check(batch_->ctx(), m3tb_upload_texture_features_device(batch_->ctx(), &body, &features, 1),
               "TextureModality::SetFeatures"))
      return false;
    if (features.length != 0) batch_->NoteDeviceFeatures(body);
    return true;
  }
  // DetectAndComputeCorrKeypoints for several ORB modalities of one Batch in ONE m3tb_texture_detect_orb call (one pose
  // download, one stream synchronisation, two launches per 128 bodies): each body's focused crop of its camera's current
  // frame and cv::ORB detect + compute on it at the modality's orb_* settings, the features stored for the next
  // StartModality / CalculateCorrespondences / CalculateResults. A body without a focus gets no features, as the
  // reference returns early. cv::ORB keeps every tie at its cuts, so it can keep more than orb_n_features; a body that
  // keeps more than n_features_max gets none that frame (detections() reports the count). False, with nothing
  // launched, for a modality that is not set up or not ORB, modalities of different batches or bad orb_* settings.
  static bool DetectFeatures(const std::vector<std::shared_ptr<TextureModality>>& modalities) {
    if (modalities.empty()) return true;
    m3tb_ctx* ctx = modalities[0]->batch_->ctx();
    std::vector<int> bodies;
    std::vector<m3tb_orb_params> params;
    for (auto& m : modalities) {
      if (!m->IsSetup()) return false;
      if (m->descriptor_type_ != DescriptorType::ORB) {
        std::cerr << "Modality " << m->name_ << ": DetectFeatures runs cv::ORB; its descriptor type is "
                  << DescriptorName(m->descriptor_type_)
                  << std::endl;
        return false;
      }
      if (m->batch_->ctx() != ctx) {
        std::cerr << "TextureModality::DetectFeatures: the modalities belong to different batches" << std::endl;
        return false;
      }
      bodies.push_back(m->body_ptr_->index());
      params.push_back(m->orb_params_);
    }
    return Check(ctx, m3tb_texture_detect_orb(ctx, bodies.data(), int(bodies.size()), params.data()),
                 "TextureModality::DetectFeatures");
  }
  // One modality's detection; each call synchronises the stream, so several bodies go through DetectFeatures(modalities)
  bool DetectFeatures() {
    std::vector<std::shared_ptr<TextureModality>> self{std::shared_ptr<TextureModality>(this, [](TextureModality*) {})};
    return DetectFeatures(self);
  }
  // The keypoints cv::ORB kept at the body's last DetectFeatures (may exceed orb_n_features and n_features_max);
  // -1 on an error. Synchronises the stream.
  int detections() const {
    int32_t n = -1;
    if (!Check(batch_->ctx(), m3tb_get_texture_detections(batch_->ctx(), body_ptr_->index(), 1, &n),
               "TextureModality::detections"))
      return -1;
    return n;
  }

  bool StartModality(int iteration, int corr_iteration) override {
    if (!IsSetup()) return false;
    (void)corr_iteration;
    if (!batch_->Claim(Batch::kStart, iteration, 0, 0)) return true;
    return Check(batch_->ctx(), m3tb_start_modalities(batch_->ctx(), iteration), "TextureModality::StartModality");
  }
  bool CalculateCorrespondences(int iteration, int corr_iteration) override {
    if (!IsSetup()) return false;
    if (!batch_->Claim(Batch::kTextureCorr, iteration, corr_iteration, 0)) return true;
    return Check(batch_->ctx(), m3tb_texture_correspondences(batch_->ctx(), iteration, corr_iteration),
                 "TextureModality::CalculateCorrespondences");
  }
  bool CalculateGradientAndHessian(int iteration, int corr_iteration, int opt_iteration) override {
    if (!IsSetup()) return false;
    if (batch_->Claim(Batch::kTextureGH, iteration, corr_iteration, opt_iteration)) {
      batch_->texture_g.resize(size_t(6) * batch_->n_bodies());
      batch_->texture_h.resize(size_t(36) * batch_->n_bodies());
      if (!Check(batch_->ctx(),
                 m3tb_texture_gradient_hessian(batch_->ctx(), iteration, corr_iteration, opt_iteration,
                                               batch_->texture_g.data(), batch_->texture_h.data()),
                 "TextureModality::CalculateGradientAndHessian"))
        return false;
    }
    FetchGH(batch_->texture_g, batch_->texture_h);
    return batch_->ReportDroppedFeatures();  // the sums above synchronised the stream
  }
  bool CalculateResults(int iteration) override {
    if (!IsSetup()) return false;
    if (!batch_->Claim(Batch::kResults, iteration, 0, 0)) return true;
    return Check(batch_->ctx(), m3tb_calculate_results(batch_->ctx(), iteration), "TextureModality::CalculateResults");
  }

 private:
  m3tb_texture_params params_;
  m3tb_orb_params orb_params_;  // DetectFeatures
  DescriptorType descriptor_type_ = DescriptorType::ORB;
  std::shared_ptr<ColorCamera> color_camera_ptr_;
  std::shared_ptr<DepthCamera> depth_camera_ptr_;  // MeasureOcclusions
};

// ---- link.h: one node of a kinematic tree (M3T/include/m3t/link.h) ---------------------------------------------------------
class Link {
 public:
  // body_ptr may be null (a link that only carries a joint, e.g. a fixed base)
  Link(const std::string& name, const std::shared_ptr<Body>& body_ptr = nullptr,
       const Transform3fA& body2joint_pose = Transform3fA::Identity(),
       const Transform3fA& joint2parent_pose = Transform3fA::Identity(),
       const Transform3fA& link2world_pose = Transform3fA::Identity(),
       const std::array<bool, 6>& free_directions = {true, true, true, true, true, true},
       bool fixed_body2joint_pose = true)
      : name_(name), body_ptr_(body_ptr), body2joint_pose_(body2joint_pose), joint2parent_pose_(joint2parent_pose),
        link2world_pose_(link2world_pose), free_directions_(free_directions), fixed_body2joint_pose_(fixed_body2joint_pose) {}
  bool AddModality(const std::shared_ptr<Modality>& m) {
    modality_ptrs_.push_back(m);
    set_up_ = false;
    return true;
  }
  bool AddChildLink(const std::shared_ptr<Link>& l) {
    for (auto& c : child_link_ptrs_)
      if (c->name() == l->name()) {
        std::cerr << "Child link " << l->name() << " already exists" << std::endl;
        return false;
      }
    child_link_ptrs_.push_back(l);
    set_up_ = false;
    return true;
  }
  void set_body2joint_pose(const Transform3fA& p) { body2joint_pose_ = p; }
  void set_joint2parent_pose(const Transform3fA& p) { joint2parent_pose_ = p; }
  void set_link2world_pose(const Transform3fA& p) { link2world_pose_ = p; }
  void set_free_directions(const std::array<bool, 6>& f) { free_directions_ = f; set_up_ = false; }
  void set_fixed_body2joint_pose(bool v) { fixed_body2joint_pose_ = v; }
  // Link::SetUp (link.cpp:37-58): a link needs a body whenever it has modalities
  bool SetUp() {
    set_up_ = false;
    if (!modality_ptrs_.empty() && !body_ptr_) {
      std::cerr << "Link " << name_ << " has modalities but no body" << std::endl;
      return false;
    }
    for (auto& m : modality_ptrs_)
      if (m->body_ptr() != body_ptr_) {
        std::cerr << "Modality " << m->name() << " does not reference the body of link " << name_ << std::endl;
        return false;
      }
    set_up_ = true;
    return true;
  }
  int DegreesOfFreedom() const {
    int n = 0;
    for (bool f : free_directions_) n += f ? 1 : 0;
    return n;
  }
  const std::string& name() const { return name_; }
  const std::shared_ptr<Body>& body_ptr() const { return body_ptr_; }
  const std::vector<std::shared_ptr<Modality>>& modality_ptrs() const { return modality_ptrs_; }
  const std::vector<std::shared_ptr<Link>>& child_link_ptrs() const { return child_link_ptrs_; }
  // the three poses are refreshed from the device by Optimizer::FetchLinkPoses()
  const Transform3fA& body2joint_pose() const { return body2joint_pose_; }
  const Transform3fA& joint2parent_pose() const { return joint2parent_pose_; }
  const Transform3fA& link2world_pose() const { return link2world_pose_; }
  const std::array<bool, 6>& free_directions() const { return free_directions_; }
  bool fixed_body2joint_pose() const { return fixed_body2joint_pose_; }
  bool set_up() const { return set_up_; }

 private:
  friend class Optimizer;
  std::string name_;
  std::shared_ptr<Body> body_ptr_;
  std::vector<std::shared_ptr<Modality>> modality_ptrs_;
  std::vector<std::shared_ptr<Link>> child_link_ptrs_;
  Transform3fA body2joint_pose_, joint2parent_pose_, link2world_pose_;
  std::array<bool, 6> free_directions_;
  bool fixed_body2joint_pose_ = true;
  bool set_up_ = true;  // a link without children / modalities changes needs no explicit SetUp (rigid-body applications)
};

// ---- constraint.h / soft_constraint.h -----------------------------------------------------------------------------------
class Constraint {
 public:
  Constraint(const std::string& name, const std::shared_ptr<Link>& link1_ptr, const std::shared_ptr<Link>& link2_ptr,
             const Transform3fA& body12joint1_pose = Transform3fA::Identity(),
             const Transform3fA& body22joint2_pose = Transform3fA::Identity(),
             const std::array<bool, 6>& constraint_directions = {false, false, false, false, false, false})
      : name_(name), link1_ptr_(link1_ptr), link2_ptr_(link2_ptr), body12joint1_pose_(body12joint1_pose),
        body22joint2_pose_(body22joint2_pose), constraint_directions_(constraint_directions) {}
  virtual ~Constraint() = default;
  void set_body12joint1_pose(const Transform3fA& p) { body12joint1_pose_ = p; }
  void set_body22joint2_pose(const Transform3fA& p) { body22joint2_pose_ = p; }
  void set_constraint_directions(const std::array<bool, 6>& d) { constraint_directions_ = d; }
  bool SetUp() {  // constraint.cpp:24-41
    set_up_ = false;
    if (!link1_ptr_ || !link2_ptr_) {
      std::cerr << "Constraint " << name_ << " needs two links" << std::endl;
      return false;
    }
    set_up_ = true;
    return true;
  }
  int NumberOfConstraints() const {
    int n = 0;
    for (bool d : constraint_directions_) n += d ? 1 : 0;
    return n;
  }
  const std::string& name() const { return name_; }
  const std::shared_ptr<Link>& link1_ptr() const { return link1_ptr_; }
  const std::shared_ptr<Link>& link2_ptr() const { return link2_ptr_; }
  const Transform3fA& body12joint1_pose() const { return body12joint1_pose_; }
  const Transform3fA& body22joint2_pose() const { return body22joint2_pose_; }
  const std::array<bool, 6>& constraint_directions() const { return constraint_directions_; }
  bool set_up() const { return set_up_; }

 protected:
  std::string name_;
  std::shared_ptr<Link> link1_ptr_, link2_ptr_;
  Transform3fA body12joint1_pose_, body22joint2_pose_;
  std::array<bool, 6> constraint_directions_;
  bool set_up_ = false;
};

class SoftConstraint : public Constraint {
 public:
  SoftConstraint(const std::string& name, const std::shared_ptr<Link>& link1_ptr, const std::shared_ptr<Link>& link2_ptr,
                 const Transform3fA& body12joint1_pose = Transform3fA::Identity(),
                 const Transform3fA& body22joint2_pose = Transform3fA::Identity(),
                 const std::array<bool, 6>& constraint_directions = {false, false, false, false, false, false},
                 float max_distance_rotation = 0.0f, float max_distance_translation = 0.0f,
                 float standard_deviation_rotation = 0.01f, float standard_deviation_translation = 0.001f)
      : Constraint(name, link1_ptr, link2_ptr, body12joint1_pose, body22joint2_pose, constraint_directions),
        max_distance_rotation_(max_distance_rotation), max_distance_translation_(max_distance_translation),
        standard_deviation_rotation_(standard_deviation_rotation),
        standard_deviation_translation_(standard_deviation_translation) {}
  void set_max_distance_rotation(float v) { max_distance_rotation_ = v; }
  void set_max_distance_translation(float v) { max_distance_translation_ = v; }
  void set_standard_deviation_rotation(float v) { standard_deviation_rotation_ = v; }
  void set_standard_deviation_translation(float v) { standard_deviation_translation_ = v; }
  float max_distance_rotation() const { return max_distance_rotation_; }
  float max_distance_translation() const { return max_distance_translation_; }
  float standard_deviation_rotation() const { return standard_deviation_rotation_; }
  float standard_deviation_translation() const { return standard_deviation_translation_; }

 private:
  float max_distance_rotation_, max_distance_translation_, standard_deviation_rotation_, standard_deviation_translation_;
};

// ---- optimizer.h ----------------------------------------------------------------------------------------------------
class Optimizer {
 public:
  Optimizer(const std::string& name, const std::shared_ptr<Batch>& batch, const std::shared_ptr<Link>& root_link_ptr,
            float tikhonov_parameter_rotation = 1000.0f, float tikhonov_parameter_translation = 30000.0f)
      : name_(name), batch_(batch), root_link_ptr_(root_link_ptr) {
    params_.tikhonov_parameter_rotation = tikhonov_parameter_rotation;
    params_.tikhonov_parameter_translation = tikhonov_parameter_translation;
  }
  bool AddConstraint(const std::shared_ptr<Constraint>& c) { constraint_ptrs_.push_back(c); set_up_ = false; return true; }
  bool AddSoftConstraint(const std::shared_ptr<SoftConstraint>& c) { soft_constraint_ptrs_.push_back(c); set_up_ = false; return true; }
  void set_tikhonov_parameter_rotation(float v) { params_.tikhonov_parameter_rotation = v; set_up_ = false; }
  void set_tikhonov_parameter_translation(float v) { params_.tikhonov_parameter_translation = v; set_up_ = false; }
  const std::string& name() const { return name_; }
  const std::shared_ptr<Link>& root_link_ptr() const { return root_link_ptr_; }
  const std::vector<std::shared_ptr<Constraint>>& constraint_ptrs() const { return constraint_ptrs_; }
  const std::vector<std::shared_ptr<SoftConstraint>>& soft_constraint_ptrs() const { return soft_constraint_ptrs_; }
  bool set_up() const { return set_up_; }
  const std::shared_ptr<Batch>& batch() const { return batch_; }
  int structure_index() const { return structure_index_; }

  // Optimizer::ReferencedLinks (optimizer.cpp:254-260): pre-order
  std::vector<std::shared_ptr<Link>> ReferencedLinks() const {
    std::vector<std::shared_ptr<Link>> out;
    AddReferencedLinks(root_link_ptr_, &out);
    return out;
  }
  int DegreesOfFreedom() const {
    int n = 0;
    for (auto& l : ReferencedLinks()) n += l->DegreesOfFreedom();
    return n;
  }
  int NumberOfConstraints() const {
    int n = 0;
    for (auto& c : constraint_ptrs_) n += c->NumberOfConstraints();
    return n;
  }

  // Optimizer::SetUp (optimizer.cpp:22-64): here it also writes the device records - one body record per link with
  // a body (modalities + parameters) and, unless this is a plain rigid body, the structure (links + constraints) -
  // and makes the poses consistent (UpdatePoses with theta = 0)
  bool SetUp() {
    set_up_ = false;
    if (!root_link_ptr_) {
      std::cerr << "No root link assigned to optimizer " << name_ << std::endl;
      return false;
    }
    const auto links = ReferencedLinks();
    bool any_modality = false;
    for (auto& l : links) {
      if (!l->set_up()) {
        std::cerr << "Link " << l->name() << " was not set up" << std::endl;
        return false;
      }
      any_modality = any_modality || !l->modality_ptrs().empty();
    }
    if (!any_modality) {
      std::cerr << "No modalities were assigned to the links of optimizer " << name_ << std::endl;
      return false;
    }
    for (auto& c : constraint_ptrs_)
      if (!c->set_up()) {
        std::cerr << "Constraint " << c->name() << " was not set up" << std::endl;
        return false;
      }
    for (auto& c : soft_constraint_ptrs_)
      if (!c->set_up()) {
        std::cerr << "SoftConstraint " << c->name() << " was not set up" << std::endl;
        return false;
      }
    for (auto& l : links)
      if (l->body_ptr() && !SetUpBody(*l)) return false;
    const bool rigid = links.size() == 1 && constraint_ptrs_.empty() && soft_constraint_ptrs_.empty() &&
                       root_link_ptr_->DegreesOfFreedom() == 6 && IsIdentity(root_link_ptr_->body2joint_pose());
    if (!rigid || structure_index_ >= 0) {
      if (!SetUpStructure(links)) return false;
      if (!Check(batch_->ctx(), m3tb_calculate_consistent_poses(batch_->ctx()), "Optimizer::SetUp")) return false;
      batch_->PosesChanged();
    }
    set_up_ = true;
    return true;
  }
  // Optimizer::CalculateConsistentPoses (optimizer.cpp:133-142)
  bool CalculateConsistentPoses() {
    if (!set_up_) {
      std::cerr << "Set up optimizer " << name_ << " first" << std::endl;
      return false;
    }
    batch_->PosesChanged();
    return Check(batch_->ctx(), m3tb_calculate_consistent_poses(batch_->ctx()), "Optimizer::CalculateConsistentPoses");
  }
  // Optimizer::CalculateOptimization (optimizer.cpp:144-167): batched over all optimizers of the Batch
  bool CalculateOptimization(int iteration, int corr_iteration, int opt_iteration) {
    if (!set_up_) {
      std::cerr << "Set up optimizer " << name_ << " first" << std::endl;
      return false;
    }
    if (!batch_->Claim(Batch::kOptimize, iteration, corr_iteration, opt_iteration)) return true;
    bool ok = Check(batch_->ctx(), m3tb_calculate_optimization(batch_->ctx(), iteration, corr_iteration, opt_iteration),
                    "Optimizer::CalculateOptimization");
    batch_->PosesChanged();
    // the batched launch updated every body: the other optimizers of this phase must find it done
    batch_->MarkDone(Batch::kOptimize, iteration, corr_iteration, opt_iteration);
    return ok;
  }
  // Refreshes Link::body2joint_pose / joint2parent_pose / link2world_pose of every referenced link from the device
  bool FetchLinkPoses() {
    if (structure_index_ < 0) return true;
    const auto links = ReferencedLinks();
    std::vector<float> b2j(12 * links.size()), j2p(12 * links.size()), l2w(12 * links.size());
    if (!Check(batch_->ctx(), m3tb_get_link_poses(batch_->ctx(), structure_index_, b2j.data(), j2p.data(), l2w.data()),
               "Optimizer::FetchLinkPoses"))
      return false;
    for (size_t i = 0; i < links.size(); ++i) {
      std::copy(b2j.begin() + 12 * i, b2j.begin() + 12 * i + 12, links[i]->body2joint_pose_.m);
      std::copy(j2p.begin() + 12 * i, j2p.begin() + 12 * i + 12, links[i]->joint2parent_pose_.m);
      std::copy(l2w.begin() + 12 * i, l2w.begin() + 12 * i + 12, links[i]->link2world_pose_.m);
    }
    return true;
  }

 private:
  static bool IsIdentity(const Transform3fA& p) {
    const Transform3fA i;
    for (int k = 0; k < 12; ++k)
      if (p.m[k] != i.m[k]) return false;
    return true;
  }
  void AddReferencedLinks(const std::shared_ptr<Link>& l, std::vector<std::shared_ptr<Link>>* out) const {
    out->push_back(l);
    for (auto& c : l->child_link_ptrs()) AddReferencedLinks(c, out);
  }
  bool SetUpBody(const Link& link) {
    const m3tb_region_params* rp = nullptr;
    const m3tb_depth_params* dp = nullptr;
    int rmodel = 0, dmodel = 0, ccam = 0, dcam = 0;
    std::shared_ptr<ColorHistograms> shared;
    std::shared_ptr<TextureModality> texture;
    for (auto& m : link.modality_ptrs()) {
      if (!m->set_up()) {
        std::cerr << "Modality " << m->name() << " was not set up" << std::endl;
        return false;
      }
      if (auto r = std::dynamic_pointer_cast<RegionModality>(m)) {
        rp = &r->params();
        rmodel = r->region_model_ptr()->index();
        ccam = r->color_camera_ptr()->index();
        shared = r->color_histograms_ptr();
      } else if (auto d = std::dynamic_pointer_cast<DepthModality>(m)) {
        dp = &d->params();
        dmodel = d->depth_model_ptr()->index();
        dcam = d->depth_camera_ptr()->index();
      } else if (auto t = std::dynamic_pointer_cast<TextureModality>(m)) {
        texture = t;
      }
    }
    if (texture && texture->depth_camera_ptr() && !dp) dcam = texture->depth_camera_ptr()->index();  // MeasureOcclusions
    const int body = link.body_ptr()->index();
    if (!Check(batch_->ctx(), m3tb_set_body(batch_->ctx(), body, rp, dp, &params_, rmodel, dmodel, ccam, dcam), "Optimizer::SetUp"))
      return false;
    // the texture modality before its renderers are attached; removed from the device when it left the link
    auto was_textured = std::find(texture_bodies_.begin(), texture_bodies_.end(), body);
    if (texture) {
      if (!Check(batch_->ctx(),
                 m3tb_set_texture_modality(batch_->ctx(), body, &texture->params(), texture->color_camera_ptr()->index()),
                 "TextureModality::SetUp"))
        return false;
      if (was_textured == texture_bodies_.end()) texture_bodies_.push_back(body);
    } else if (was_textured != texture_bodies_.end()) {
      if (!Check(batch_->ctx(), m3tb_set_texture_modality(batch_->ctx(), body, nullptr, 0), "Link::DeleteModality"))
        return false;
      texture_bodies_.erase(was_textured);
    }
    // the modalities' renderers feed the body's renderer slots (-1: none, detaches an earlier one)
    for (auto& m : link.modality_ptrs()) {
      const int modality =
          std::dynamic_pointer_cast<RegionModality>(m) ? 0 : std::dynamic_pointer_cast<TextureModality>(m) ? 2 : 1;
      const int dr = m->depth_renderer_ptr() ? m->depth_renderer_ptr()->index() : -1;
      const int sr = m->silhouette_renderer_ptr() ? m->silhouette_renderer_ptr()->index() : -1;
      if (!Check(batch_->ctx(), m3tb_attach_renderer(batch_->ctx(), body, modality, 0, dr), "Modality::ModelOcclusions") ||
          !Check(batch_->ctx(), m3tb_attach_renderer(batch_->ctx(), body, modality, 1, sr), "Modality::UseSilhouetteChecking"))
        return false;
    }
    if (rp && shared) {  // UseSharedColorHistograms: the first body the object was given to owns it on the device
      shared->claim_owner(body);
      if (!Check(batch_->ctx(), m3tb_share_color_histograms(batch_->ctx(), body, shared->owner_body()),
                 "RegionModality::UseSharedColorHistograms"))
        return false;
      if (std::find(shared_bodies_.begin(), shared_bodies_.end(), body) == shared_bodies_.end()) shared_bodies_.push_back(body);
    } else {
      auto it = std::find(shared_bodies_.begin(), shared_bodies_.end(), body);
      if (it != shared_bodies_.end()) {  // DoNotUseSharedColorHistograms since the last SetUp
        if (!Check(batch_->ctx(), m3tb_share_color_histograms(batch_->ctx(), body, -1), "RegionModality::DoNotUseSharedColorHistograms"))
          return false;
        shared_bodies_.erase(it);
      }
    }
    return true;
  }
  bool SetUpStructure(const std::vector<std::shared_ptr<Link>>& links) {
    auto index_of = [&](const std::shared_ptr<Link>& l) {
      for (size_t i = 0; i < links.size(); ++i)
        if (links[i] == l) return int(i);
      return -1;
    };
    std::vector<m3tb_link> ml(links.size());
    for (size_t i = 0; i < links.size(); ++i) {
      const Link& l = *links[i];
      m3tb_link& o = ml[i];
      o.body = l.body_ptr() ? l.body_ptr()->index() : -1;
      o.parent = -1;
      for (size_t p = 0; p < i && o.parent < 0; ++p)
        for (auto& c : links[p]->child_link_ptrs())
          if (c == links[i]) o.parent = int(p);
      std::copy(l.body2joint_pose().m, l.body2joint_pose().m + 12, o.body2joint);
      std::copy(l.joint2parent_pose().m, l.joint2parent_pose().m + 12, o.joint2parent);
      std::copy(l.link2world_pose().m, l.link2world_pose().m + 12, o.link2world);
      for (int d = 0; d < 6; ++d) o.free_directions[d] = l.free_directions()[d] ? 1 : 0;
      o.fixed_body2joint_pose = l.fixed_body2joint_pose() ? 1 : 0;
    }
    std::vector<m3tb_constraint> mc;
    auto add = [&](const Constraint& c, const SoftConstraint* soft) -> bool {
      m3tb_constraint o{};
      o.link1 = index_of(c.link1_ptr());
      o.link2 = index_of(c.link2_ptr());
      if (o.link1 < 0 || o.link2 < 0) {
        std::cerr << "Constraint " << c.name() << " references a link outside optimizer " << name_ << std::endl;
        return false;
      }
      std::copy(c.body12joint1_pose().m, c.body12joint1_pose().m + 12, o.body12joint1);
      std::copy(c.body22joint2_pose().m, c.body22joint2_pose().m + 12, o.body22joint2);
      for (int d = 0; d < 6; ++d) o.directions[d] = c.constraint_directions()[d] ? 1 : 0;
      o.soft = soft ? 1 : 0;
      o.standard_deviation_rotation = soft ? soft->standard_deviation_rotation() : 0.01f;
      o.standard_deviation_translation = soft ? soft->standard_deviation_translation() : 0.001f;
      o.max_distance_rotation = soft ? soft->max_distance_rotation() : 0.0f;
      o.max_distance_translation = soft ? soft->max_distance_translation() : 0.0f;
      mc.push_back(o);
      return true;
    };
    for (auto& c : constraint_ptrs_)
      if (!add(*c, nullptr)) return false;
    for (auto& c : soft_constraint_ptrs_)
      if (!add(*c, c.get())) return false;
    if (structure_index_ < 0) structure_index_ = batch_->NextStructure();
    return Check(batch_->ctx(),
                 m3tb_set_structure(batch_->ctx(), structure_index_, ml.data(), int(ml.size()), mc.empty() ? nullptr : mc.data(),
                                    int(mc.size()), &params_),
                 "Optimizer::SetUp");
  }

  std::string name_;
  std::shared_ptr<Batch> batch_;
  std::shared_ptr<Link> root_link_ptr_;
  std::vector<std::shared_ptr<Constraint>> constraint_ptrs_;
  std::vector<std::shared_ptr<SoftConstraint>> soft_constraint_ptrs_;
  m3tb_optimizer_params params_{};
  std::vector<int> shared_bodies_;  // bodies whose region modality was set up with a shared ColorHistograms object
  std::vector<int> texture_bodies_;  // bodies whose texture modality this optimizer set on the device
  int structure_index_ = -1;
  bool set_up_ = false;
};

// ---- tracker.h ------------------------------------------------------------------------------------------------------
class Tracker {
 public:
  Tracker(const std::string& name, const std::shared_ptr<Batch>& batch, int n_corr_iterations = 5, int n_update_iterations = 2)
      : name_(name), batch_(batch), n_corr_iterations_(n_corr_iterations), n_update_iterations_(n_update_iterations) {}
  bool AddOptimizer(const std::shared_ptr<Optimizer>& o) {
    optimizer_ptrs_.push_back(o);
    for (auto& l : o->ReferencedLinks())
      for (auto& m : l->modality_ptrs()) modality_ptrs_.push_back(m);
    return true;
  }
  // Tracker::AddViewer (tracker.cpp): viewers are set up with the tracker and updated by UpdateViewers
  bool AddViewer(const std::shared_ptr<Viewer>& v) {
    for (auto& p : viewer_ptrs_)
      if (p->name() == v->name()) {
        std::cerr << "Viewer " << v->name() << " already exists" << std::endl;
        return false;
      }
    viewer_ptrs_.push_back(v);
    return true;
  }
  // Tracker::UpdateViewers (tracker.cpp:373): one m3tb_update_viewers for all normal viewers, from the current poses and
  // frames, and UpdateViewer of every image viewer
  bool UpdateViewers(int iteration) {
    bool any_normal = false;
    for (auto& v : viewer_ptrs_) {
      if (v->dirty() && !v->SetUp()) return false;
      if (v->drawn_by_update_viewers()) any_normal = true;
      else if (!v->UpdateViewer(iteration)) return false;
    }
    if (!any_normal) return true;
    batch_->ViewersUpdated();
    return Check(batch_->ctx(), m3tb_update_viewers(batch_->ctx()), "Tracker::UpdateViewers");
  }
  const std::vector<std::shared_ptr<Viewer>>& viewer_ptrs() const { return viewer_ptrs_; }
  void set_n_corr_iterations(int v) { n_corr_iterations_ = v; }
  void set_n_update_iterations(int v) { n_update_iterations_ = v; }
  int n_corr_iterations() const { return n_corr_iterations_; }
  int n_update_iterations() const { return n_update_iterations_; }

  bool SetUp() {  // Tracker::SetUp: set up all referenced objects (tracker.cpp:884-899 order: modalities, optimizers)
    for (auto& m : modality_ptrs_)
      if (!m->SetUp()) return false;
    for (auto& o : optimizer_ptrs_) {
      for (auto& l : o->ReferencedLinks())
        if (!l->SetUp()) return false;
      for (auto& c : o->constraint_ptrs())
        if (!c->SetUp()) return false;
      for (auto& c : o->soft_constraint_ptrs())
        if (!c->SetUp()) return false;
      if (!o->SetUp()) return false;
    }
    for (auto& v : viewer_ptrs_)
      if (!v->SetUp()) return false;
    set_up_ = true;
    return true;
  }
  // Tracker::StartModalities (tracker.cpp:430-445)
  bool StartModalities(int iteration) {
    for (auto& m : modality_ptrs_)
      if (!m->StartModality(iteration, 0)) return false;
    return true;
  }
  // Tracker::ExecuteTrackingStep (tracker.cpp:344-364), fast path: ONE fused launch for the whole
  // corr x update loop nest of every body + the histogram update
  bool ExecuteTrackingStep(int iteration) {
    if (!set_up_) {
      std::cerr << "Set up tracker " << name_ << " first" << std::endl;
      return false;
    }
    bool ok = Check(batch_->ctx(), m3tb_tracking_step(batch_->ctx(), iteration, n_corr_iterations_, n_update_iterations_),
                    "Tracker::ExecuteTrackingStep");
    batch_->PosesChanged();
    return ok && Check(batch_->ctx(), m3tb_calculate_results(batch_->ctx(), iteration), "Tracker::CalculateResults");
  }
  // The same step, phase by phase through the Modality / Optimizer objects exactly as the reference's Tracker fans
  // them out (tracker.cpp:447-517); used to show that the adapters compose and for step-wise debugging.
  bool ExecuteTrackingStepObjectWise(int iteration) {
    for (int corr = 0; corr < n_corr_iterations_; ++corr) {
      // Tracker::CalculateCorrespondences renders first (tracker.cpp:447-456)
      for (auto& m : modality_ptrs_)
        for (auto& r : m->correspondence_renderer_ptrs())
          if (!r->StartRendering()) return false;
      for (auto& m : modality_ptrs_)
        if (!m->CalculateCorrespondences(iteration, corr)) return false;
      for (int upd = 0; upd < n_update_iterations_; ++upd) {
        for (auto& m : modality_ptrs_)
          if (!m->CalculateGradientAndHessian(iteration, corr, upd)) return false;
        for (auto& o : optimizer_ptrs_)
          if (!o->CalculateOptimization(iteration, corr, upd)) return false;
      }
    }
    for (auto& m : modality_ptrs_)
      if (!m->CalculateResults(iteration)) return false;
    return true;
  }

 private:
  std::string name_;
  std::shared_ptr<Batch> batch_;
  int n_corr_iterations_, n_update_iterations_;
  std::vector<std::shared_ptr<Optimizer>> optimizer_ptrs_;
  std::vector<std::shared_ptr<Modality>> modality_ptrs_;
  std::vector<std::shared_ptr<Viewer>> viewer_ptrs_;
  bool set_up_ = false;
};

// ---- refiner.h ------------------------------------------------------------------------------------------------------
// Refiner (refiner.h): refines the poses of the named optimizers, e.g. after a detector, while every other body keeps
// tracking undisturbed. RefinePoses is one m3tb_refine_poses call: a rigid optimizer is refined through its body, a
// kinematic structure as a whole. When a named optimizer's links carry a TextureModality it is one
// m3tb_refine_poses_orb call instead, which detects the ORB features before every correspondence iteration at each
// modality's orb_* settings; SIFT / DAISY modalities have no device detector and cannot be refined.
class Refiner {
 public:
  Refiner(const std::string& name, int n_corr_iterations = 7, int n_update_iterations = 2)
      : name_(name), n_corr_iterations_(n_corr_iterations), n_update_iterations_(n_update_iterations) {}
  bool AddOptimizer(const std::shared_ptr<Optimizer>& o) {
    for (auto& p : optimizer_ptrs_)
      if (p->name() == o->name()) {
        std::cerr << "Optimizer " << o->name() << " already exists" << std::endl;
        return false;
      }
    if (!optimizer_ptrs_.empty() && optimizer_ptrs_.front()->batch() != o->batch()) {
      std::cerr << "Optimizer " << o->name() << " belongs to another batch than refiner " << name_ << std::endl;
      return false;
    }
    optimizer_ptrs_.push_back(o);
    set_up_ = false;
    return true;
  }
  // Refiner::SetUp (refiner.cpp:24-45) without set_up_all_objects: the optimizers are set up by the tracker (or
  // their own SetUp), so that the refiner and the tracker share the device records
  bool SetUp() {
    set_up_ = false;
    for (auto& o : optimizer_ptrs_)
      if (!o->set_up()) {
        std::cerr << "Optimizer " << o->name() << " was not set up" << std::endl;
        return false;
      }
    set_up_ = true;
    return true;
  }
  // Refiner::RefinePoses (refiner.cpp:76-117): names that match no optimizer are ignored
  bool RefinePoses(const std::set<std::string>& names) {
    if (!set_up_) {
      std::cerr << "Set up refiner " << name_ << " first" << std::endl;
      return false;
    }
    std::vector<int> bodies, structures;
    std::vector<std::pair<int, m3tb_orb_params>> texture;  // (body, orb_* settings) of the named texture modalities
    for (auto& o : optimizer_ptrs_) {
      if (names.find(o->name()) == names.end()) continue;
      if (o->structure_index() >= 0) structures.push_back(o->structure_index());
      else bodies.push_back(o->root_link_ptr()->body_ptr()->index());
      for (auto& l : o->ReferencedLinks())
        for (auto& m : l->modality_ptrs())
          if (auto t = std::dynamic_pointer_cast<TextureModality>(m)) {
            if (t->descriptor_type() != TextureModality::DescriptorType::ORB) {
              std::cerr << "Modality " << t->name() << ": only ORB features are detected on the device between the "
                        << "correspondence iterations, its descriptor type is "
                        << TextureModality::DescriptorName(t->descriptor_type()) << "; optimizer " << o->name()
                        << " cannot be refined" << std::endl;
              return false;
            }
            texture.emplace_back(t->body_ptr()->index(), t->orb_params());
          }
    }
    if (bodies.empty() && structures.empty()) return true;
    const auto& batch = optimizer_ptrs_.front()->batch();
    m3tb_ctx* ctx = batch->ctx();
    int rc;
    if (texture.empty()) {
      rc = m3tb_refine_poses(ctx, bodies.data(), int(bodies.size()), structures.data(), int(structures.size()),
                             n_corr_iterations_, n_update_iterations_);
    } else {
      std::vector<m3tb_orb_params> orb(std::max(m3tb_n_bodies(ctx), 1));
      for (auto& p : orb) m3tb_orb_params_default(&p);
      for (auto& t : texture) orb[t.first] = t.second;
      rc = m3tb_refine_poses_orb(ctx, bodies.data(), int(bodies.size()), structures.data(), int(structures.size()),
                                 n_corr_iterations_, n_update_iterations_, orb.data());
    }
    const bool ok = Check(ctx, rc, "Refiner::RefinePoses");
    batch->PosesChanged();
    return ok;
  }
  void set_name(const std::string& name) { name_ = name; }
  void set_n_corr_iterations(int v) { n_corr_iterations_ = v; }
  void set_n_update_iterations(int v) { n_update_iterations_ = v; }
  const std::string& name() const { return name_; }
  const std::vector<std::shared_ptr<Optimizer>>& optimizer_ptrs() const { return optimizer_ptrs_; }
  int n_corr_iterations() const { return n_corr_iterations_; }
  int n_update_iterations() const { return n_update_iterations_; }
  bool set_up() const { return set_up_; }

 private:
  std::string name_;
  int n_corr_iterations_, n_update_iterations_;
  std::vector<std::shared_ptr<Optimizer>> optimizer_ptrs_;
  bool set_up_ = false;
};

// ---- the evaluators' pose scoring (examples/{ycb,rtb,opt,rbot}_evaluator.cpp) -----------------------------------------
// The evaluators' model data: the vertices of a body (Body::vertices()), the reduced set GenderateReducedVertices
// draws from them, and the diameter CalculateDiameters computes. Bodies sharing a mesh share one EvaluationModel.
class EvaluationModel {
 public:
  EvaluationModel(const std::string& name, const std::shared_ptr<Batch>& batch) : name_(name), batch_(batch) {
    index_ = batch->NextEvaluationModel();
  }
  const std::string& name() const { return name_; }
  int index() const { return index_; }
  void set_n_vertices_evaluation(int n) { n_vertices_evaluation_ = n; }
  void set_vertices(const std::vector<float>& vertices) { vertices_ = vertices; }  // [n][3], Body::vertices() order
  bool SetUp() {
    return Check(batch_->ctx(),
                 m3tb_set_evaluation_model(batch_->ctx(), index_, vertices_.data(), int(vertices_.size() / 3),
                                           n_vertices_evaluation_),
                 "EvaluationModel::SetUp");
  }
  // scores `body` against this model; geometry2body: OPTEvaluator's kBody2Geometry2BodyPoseMap entry
  bool AddBody(const Body& body, const Transform3fA* geometry2body = nullptr) {
    return Check(batch_->ctx(),
                 m3tb_set_body_evaluation_model(batch_->ctx(), body.index(), index_,
                                                geometry2body ? geometry2body->data() : nullptr),
                 "EvaluationModel::AddBody");
  }
  // the reduced set, read back from the device ([n][3])
  std::vector<float> reduced_vertices() const {
    int n = 0;
    if (!Check(batch_->ctx(), m3tb_get_evaluation_vertices(batch_->ctx(), index_, nullptr, 0, &n), "reduced_vertices"))
      return {};
    std::vector<float> v(size_t(n) * 3);
    Check(batch_->ctx(), m3tb_get_evaluation_vertices(batch_->ctx(), index_, v.data(), n, &n), "reduced_vertices");
    return v;
  }
  // OPTEvaluator::CalculateDiameters for this model
  bool CalculateDiameter(float* diameter) const {
    return Check(batch_->ctx(), m3tb_calculate_diameters(batch_->ctx(), &index_, 1, diameter), "CalculateDiameters");
  }

 private:
  std::string name_;
  std::shared_ptr<Batch> batch_;
  int index_ = 0;
  int n_vertices_evaluation_ = -1;
  std::vector<float> vertices_;
};

namespace detail {
// One m3tb_score_poses call for bodies that share a batch, scored at their current device poses.
inline bool ScorePoses(const std::vector<std::shared_ptr<Body>>& bodies, const std::vector<Transform3fA>& gt_body2world_poses,
                       const m3tb_score_params& params, std::vector<m3tb_pose_score>* scores,
                       std::vector<float>* add_curves, std::vector<float>* adds_curves, const char* what) {
  if (bodies.empty() || bodies.size() != gt_body2world_poses.size()) {
    std::cerr << what << ": one ground-truth pose per body" << std::endl;
    return false;
  }
  m3tb_ctx* ctx = bodies[0]->batch()->ctx();
  for (const auto& b : bodies)
    if (b->batch() != bodies[0]->batch()) {
      std::cerr << what << ": body " << b->name() << " belongs to another Batch than body " << bodies[0]->name()
                << std::endl;
      return false;
    }
  std::vector<int> ids;
  std::vector<float> gt;
  for (size_t i = 0; i < bodies.size(); ++i) {
    ids.push_back(bodies[i]->index());
    gt.insert(gt.end(), gt_body2world_poses[i].m, gt_body2world_poses[i].m + 12);
  }
  scores->resize(bodies.size());
  if (add_curves) {
    add_curves->resize(bodies.size() * M3TB_N_CURVE_VALUES);
    adds_curves->resize(bodies.size() * M3TB_N_CURVE_VALUES);
  }
  return Check(ctx,
               m3tb_score_poses(ctx, ids.data(), int(ids.size()), gt.data(), 0, &params, scores->data(),
                                add_curves ? add_curves->data() : nullptr, add_curves ? adds_curves->data() : nullptr, 0),
               what);
}
}  // namespace detail

// YCBEvaluator::CalculatePoseResults (ycb_evaluator.cpp:803-848) for many bodies in one call: ADD / ADD-S AUC and curves
// of each body's current pose against its ground truth.
class YCBEvaluator {
 public:
  static constexpr size_t kNCurveValues = M3TB_N_CURVE_VALUES;
  static constexpr float kThresholdMax = 0.1f;
  struct Result {
    float add_auc = 0.0f, adds_auc = 0.0f;
    std::array<float, kNCurveValues> add_curve{}, adds_curve{};
  };
  static bool CalculatePoseResults(const std::vector<std::shared_ptr<Body>>& bodies,
                                   const std::vector<Transform3fA>& gt_body2world_poses, std::vector<Result>* results) {
    m3tb_score_params p;
    m3tb_score_params_default(&p);
    p.threshold_max = kThresholdMax;
    std::vector<m3tb_pose_score> s;
    std::vector<float> ca, cs;
    if (!detail::ScorePoses(bodies, gt_body2world_poses, p, &s, &ca, &cs, "YCBEvaluator::CalculatePoseResults"))
      return false;
    results->resize(bodies.size());
    for (size_t i = 0; i < bodies.size(); ++i) {
      auto& r = (*results)[i];
      r.add_auc = s[i].add_auc;
      r.adds_auc = s[i].adds_auc;
      std::copy(ca.begin() + i * kNCurveValues, ca.begin() + (i + 1) * kNCurveValues, r.add_curve.begin());
      std::copy(cs.begin() + i * kNCurveValues, cs.begin() + (i + 1) * kNCurveValues, r.adds_curve.begin());
    }
    return true;
  }
};

// RTBEvaluator::CalculatePoseResults (rtb_evaluator.cpp:930-989): per-body errors on the device, then the averages
// over each combined body and over the combined bodies on the host, in the reference's order. `bodies` holds every
// body the ids of ids_combined_bodies index, with its ground truth at the same position.
class RTBEvaluator {
 public:
  static constexpr size_t kNCurveValues = M3TB_N_CURVE_VALUES;
  struct Result {
    float add_auc = 0.0f, adds_auc = 0.0f;
    std::array<float, kNCurveValues> add_curve{}, adds_curve{};
  };
  static bool CalculatePoseResults(const std::vector<std::shared_ptr<Body>>& bodies,
                                   const std::vector<Transform3fA>& gt_body2world_poses,
                                   const std::vector<std::vector<int>>& ids_combined_bodies, float error_threshold,
                                   Result* result) {
    m3tb_score_params p;
    m3tb_score_params_default(&p);
    p.threshold_max = error_threshold;
    std::vector<m3tb_pose_score> s;
    if (!detail::ScorePoses(bodies, gt_body2world_poses, p, &s, nullptr, nullptr, "RTBEvaluator::CalculatePoseResults"))
      return false;
    float add_auc = 0.0f, adds_auc = 0.0f;
    for (const auto& ids_combined_body : ids_combined_bodies) {
      float add_error_combined_body = 0.0f, adds_error_combined_body = 0.0f;
      for (int id : ids_combined_body) {
        add_error_combined_body += s[size_t(id)].add_error;
        adds_error_combined_body += s[size_t(id)].adds_error;
      }
      add_error_combined_body /= ids_combined_body.size();
      adds_error_combined_body /= ids_combined_body.size();
      add_auc += 1.0f - std::min(add_error_combined_body / error_threshold, 1.0f);
      adds_auc += 1.0f - std::min(adds_error_combined_body / error_threshold, 1.0f);
    }
    add_auc /= ids_combined_bodies.size();
    adds_auc /= ids_combined_bodies.size();
    result->add_auc = add_auc;
    result->adds_auc = adds_auc;
    const float threshold_step = 1.0f / float(kNCurveValues);
    std::fill(begin(result->add_curve), end(result->add_curve), 1.0f);
    for (size_t i = 0; i < kNCurveValues; ++i) {
      if (add_auc < threshold_step * (0.5f + float(i))) break;
      result->add_curve[i] = 0.0f;
    }
    std::fill(begin(result->adds_curve), end(result->adds_curve), 1.0f);
    for (size_t i = 0; i < kNCurveValues; ++i) {
      if (adds_auc < threshold_step * (0.5f + float(i))) break;
      result->adds_curve[i] = 0.0f;
    }
    return true;
  }
};

// OPTEvaluator::CalculatePoseResults (opt_evaluator.cpp:462-488): the ADD curve and area under it, scaled by the
// diameter of the body's evaluation model (CalculateDiameter) and with the geometry2body term given to AddBody. One call
// scores bodies of one diameter.
class OPTEvaluator {
 public:
  static constexpr size_t kNCurveValues = M3TB_N_CURVE_VALUES;
  static constexpr float kThresholdMax = 0.2f;
  struct Result {
    float area_under_curve = 0.0f;
    std::array<float, kNCurveValues> curve_values{};
  };
  static bool CalculatePoseResults(const std::vector<std::shared_ptr<Body>>& bodies,
                                   const std::vector<Transform3fA>& gt_body2world_poses, float diameter,
                                   std::vector<Result>* results) {
    m3tb_score_params p;
    m3tb_score_params_default(&p);
    p.threshold_max = kThresholdMax;
    p.curve_scale = diameter;
    p.auc_scale = kThresholdMax;
    std::vector<m3tb_pose_score> s;
    std::vector<float> ca, cs;
    if (!detail::ScorePoses(bodies, gt_body2world_poses, p, &s, &ca, &cs, "OPTEvaluator::CalculatePoseResults"))
      return false;
    results->resize(bodies.size());
    for (size_t i = 0; i < bodies.size(); ++i) {
      (*results)[i].area_under_curve = s[i].add_auc;
      std::copy(ca.begin() + i * kNCurveValues, ca.begin() + (i + 1) * kNCurveValues, (*results)[i].curve_values.begin());
    }
    return true;
  }
};

// RBOTEvaluator::CalculatePoseResults (rbot_evaluator.cpp:416-433): translation and rotation error and tracking success
// (thresholds 0.05 m and 5 degrees).
class RBOTEvaluator {
 public:
  struct Result {
    float translation_error = 0.0f, rotation_error = 0.0f, tracking_success = 0.0f;
  };
  static bool CalculatePoseResults(const std::vector<std::shared_ptr<Body>>& bodies,
                                   const std::vector<Transform3fA>& gt_body2world_poses, std::vector<Result>* results) {
    m3tb_score_params p;
    m3tb_score_params_default(&p);
    std::vector<m3tb_pose_score> s;
    if (!detail::ScorePoses(bodies, gt_body2world_poses, p, &s, nullptr, nullptr, "RBOTEvaluator::CalculatePoseResults"))
      return false;
    results->resize(bodies.size());
    for (size_t i = 0; i < bodies.size(); ++i)
      (*results)[i] = {s[i].translation_error, s[i].rotation_error, s[i].tracking_success};
    return true;
  }
};

}  // namespace m3t_b200
#endif  // M3T_B200_HPP_
