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
// Everything the reference has outside this path (renderers, detectors, viewers, texture modality, YAML metafiles,
// kinematic constraints) is out of scope here (DESIGN.md). Poses use a minimal Transform3fA (row-major 3x4).
#ifndef M3T_B200_HPP_
#define M3T_B200_HPP_

#include <algorithm>
#include <array>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <memory>
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

  enum PhaseKind { kRegionCorr, kDepthCorr, kRegionGH, kDepthGH, kOptimize, kStart, kResults, kNPhases };
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
  int NextBody() { return n_bodies_++; }
  int NextColorCamera() { return n_color_++; }
  int NextDepthCamera() { return n_depth_++; }
  int NextRegionModel() { return n_rmodels_++; }
  int NextDepthModel() { return n_dmodels_++; }
  int NextStructure() { return n_structures_++; }
  int n_bodies() const { return n_bodies_; }

  std::vector<float> region_g, region_h, depth_g, depth_h;  // last batched gradients / Hessians (all bodies)

 private:
  m3tb_ctx* ctx_ = nullptr;
  int max_bodies_ = 0, n_bodies_ = 0, n_color_ = 0, n_depth_ = 0, n_rmodels_ = 0, n_dmodels_ = 0, n_structures_ = 0;
  long pose_version_ = 0;
  Key done_[kNPhases];
};

// ---- body.h --------------------------------------------------------------------------------------------------------
class Body {
 public:
  Body(const std::string& name, const std::shared_ptr<Batch>& batch) : name_(name), batch_(batch) {
    index_ = batch->NextBody();
  }
  const std::string& name() const { return name_; }
  int index() const { return index_; }
  // Body::set_body2world_pose (body.cpp:85-90)
  bool set_body2world_pose(const Transform3fA& pose) {
    body2world_pose_ = pose;
    batch_->PosesChanged();
    return Check(batch_->ctx(), m3tb_set_poses(batch_->ctx(), index_, 1, pose.data()), "Body::set_body2world_pose");
  }
  // Body::body2world_pose(): reads the pose back from the device (it is updated there by the optimizer)
  const Transform3fA& body2world_pose() {
    Check(batch_->ctx(), m3tb_get_poses(batch_->ctx(), index_, 1, body2world_pose_.data()), "Body::body2world_pose");
    return body2world_pose_;
  }

 private:
  std::string name_;
  std::shared_ptr<Batch> batch_;
  int index_ = 0;
  Transform3fA body2world_pose_;
};

// ---- camera.h --------------------------------------------------------------------------------------------------------
class Camera {
 public:
  const std::string& name() const { return name_; }
  const Intrinsics& intrinsics() const { return intrinsics_; }
  const Transform3fA& world2camera_pose() const { return world2camera_pose_; }
  int index() const { return index_; }
  bool set_up() const { return set_up_; }

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

 private:
  float depth_scale_;
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

 protected:
  Model(const std::string& name, const std::shared_ptr<Batch>& batch, int point_bytes)
      : name_(name), batch_(batch), point_bytes_(point_bytes) {}
  std::string name_;
  std::shared_ptr<Batch> batch_;
  int point_bytes_;
  int index_ = 0, n_views_ = 0, n_points_ = 0;
  std::vector<float> orientations_, scalars_;
  std::vector<uint8_t> points_;
  bool set_up_ = false;
};

class RegionModel : public Model {
 public:
  RegionModel(const std::string& name, const std::shared_ptr<Batch>& batch) : Model(name, batch, M3TB_REGION_POINT_BYTES) {
    index_ = batch->NextRegionModel();
  }
  bool SetUp() {
    if (n_views_ == 0) {
      std::cerr << "Region model " << name_ << " has no views" << std::endl;
      return false;
    }
    set_up_ = Check(batch_->ctx(),
                    m3tb_set_region_model(batch_->ctx(), index_, n_views_, n_points_, orientations_.data(), scalars_.data(),
                                          points_.data(), 0.002f, 0.05f),
                    "RegionModel::SetUp");
    return set_up_;
  }
};

class DepthModel : public Model {
 public:
  DepthModel(const std::string& name, const std::shared_ptr<Batch>& batch) : Model(name, batch, M3TB_DEPTH_POINT_BYTES) {
    index_ = batch->NextDepthModel();
  }
  bool SetUp() {
    if (n_views_ == 0) {
      std::cerr << "Depth model " << name_ << " has no views" << std::endl;
      return false;
    }
    set_up_ = Check(batch_->ctx(),
                    m3tb_set_depth_model(batch_->ctx(), index_, n_views_, n_points_, orientations_.data(), scalars_.data(),
                                         points_.data(), 0.002f, 0.05f),
                    "DepthModel::SetUp");
    return set_up_;
  }
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

 protected:
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
  void set_stride_length(float v) { params_.stride_length = v; set_up_ = false; }
  void set_considered_distances(const std::vector<float>& v) {
    params_.n_considered_distances = int(v.size());
    for (size_t i = 0; i < v.size() && i < M3TB_MAX_SCHEDULE; ++i) params_.considered_distances[i] = v[i];
    set_up_ = false;
  }
  void set_standard_deviations(const std::vector<float>& v) {
    params_.n_standard_deviations = int(v.size());
    for (size_t i = 0; i < v.size() && i < M3TB_MAX_SCHEDULE; ++i) params_.standard_deviations[i] = v[i];
    set_up_ = false;
  }
  const m3tb_depth_params& params() const { return params_; }
  const std::shared_ptr<DepthCamera>& depth_camera_ptr() const { return depth_camera_ptr_; }
  const std::shared_ptr<DepthModel>& depth_model_ptr() const { return depth_model_ptr_; }

  bool SetUp() override { set_up_ = true; return true; }
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
  m3tb_depth_params params_;
  std::shared_ptr<DepthCamera> depth_camera_ptr_;
  std::shared_ptr<DepthModel> depth_model_ptr_;
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
      }
    }
    const int body = link.body_ptr()->index();
    if (!Check(batch_->ctx(), m3tb_set_body(batch_->ctx(), body, rp, dp, &params_, rmodel, dmodel, ccam, dcam), "Optimizer::SetUp"))
      return false;
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
  bool set_up_ = false;
};

}  // namespace m3t_b200
#endif  // M3T_B200_HPP_
