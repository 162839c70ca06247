/* m3t_b200.h — C ABI of libm3t_b200: the H100-native (sm_90a) implementation of M3T's
 * per-frame pose-optimisation hot path (RegionModality correspondence lines + DepthModality
 * point-to-plane -> per-body 6x6 Hessian / 6-gradient -> Tikhonov Gauss-Newton solve -> SE(3) update).
 *
 * The reference (DLR-RM/3DObjectTracking, M3T/) has no FFI: its extension surface is C++ subclassing
 * of m3t::Modality (M3T/include/m3t/modality.h:56-155). This header is the boundary a maintainer binds
 * instead; every entry point names the reference method(s) it replaces. The header-only C++ adapters in
 * 3dobjecttracking_b200/host/ (m3t_b200::RegionModality, DepthModality, Optimizer, Tracker ...) keep the
 * reference's class / method names on top of these calls. See INTEGRATION.md.
 *
 * Conventions
 *  - plain C, opaque context handle, no torch / Eigen / OpenCV types in any signature;
 *  - every function returns an int status: 0 = ok, negative = m3tb_status error; never throws;
 *    m3tb_last_error() returns a human-readable message for the last failure on that context
 *    (the reference prints to std::cerr and returns false, e.g. region_modality.cpp:1813-1819);
 *  - poses are float[12], row-major 3x4 [R | t] (the top three rows of m3t::Transform3fA);
 *  - the 6-vector parameter order is [rot_x, rot_y, rot_z, trans_x, trans_y, trans_z], variation in
 *    the body frame, right-multiplied (link.cpp:222-238);
 *  - gradients are float[6]; Hessians float[36] (symmetric, so row/column-major is moot);
 *  - all work is enqueued on the context's CUDA stream (m3tb_set_stream); calls that return data
 *    to host memory synchronise that stream before returning;
 *  - one host thread per context (the reference's Calculate* methods are single-threaded as well,
 *    tracker.cpp:251-255). Contexts are independent.
 *  - there is NO CPU fallback: every compute entry point fails with M3TB_ERR_CUDA when no
 *    sm_90 (H100-class) device is usable.
 */
#ifndef M3T_B200_H_
#define M3T_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define M3TB_MAX_SCHEDULE 8      /* max entries in scales / standard_deviations / considered_distances */
#define M3TB_N_DEPTH_OFFSETS 30  /* kMaxNDepthOffsets, M3T/include/m3t/model.h:58 */
#define M3TB_FUNCTION_LENGTH 8   /* region_modality.h:415 (compiled-in; other values are rejected) */
#define M3TB_DISTRIBUTION_LENGTH 12 /* region_modality.h:416 (compiled-in) */
#define M3TB_REGION_POINT_BYTES 152 /* RegionModel::DataPoint as stored in .bin, region_model.h:89-95 */
#define M3TB_DEPTH_POINT_BYTES 144  /* DepthModel::DataPoint as stored in .bin, depth_model.h:67-71 */

typedef enum m3tb_status {
  M3TB_OK = 0,
  M3TB_ERR_INVALID = -1,   /* bad argument / id out of range / object not set up */
  M3TB_ERR_CUDA = -2,      /* CUDA runtime failure or no usable device */
  M3TB_ERR_UNSUPPORTED = -3, /* option of the reference that this build does not implement */
  M3TB_ERR_NOT_SET_UP = -4 /* mirrors "Set up ... first" (IsSetup() == false) */
} m3tb_status;

typedef struct m3tb_ctx m3tb_ctx;

/* m3t::Intrinsics, M3T/include/m3t/common.h:25-29 */
typedef struct m3tb_intrinsics {
  float fu, fv, ppu, ppv;
  int32_t width, height;
} m3tb_intrinsics;

/* Parameters of m3t::RegionModality, defaults region_modality.h:411-443 */
typedef struct m3tb_region_params {
  int32_t n_lines_max;             /* 200 */
  int32_t use_adaptive_coverage;   /* 0 */
  float reference_contour_length;  /* 0 */
  float min_continuous_distance;   /* 3 */
  int32_t function_length;         /* 8  (must equal M3TB_FUNCTION_LENGTH) */
  int32_t distribution_length;     /* 12 (must equal M3TB_DISTRIBUTION_LENGTH) */
  float function_amplitude;        /* 0.43 */
  float function_slope;            /* 0.5 */
  float learning_rate;             /* 1.3 */
  int32_t n_global_iterations;     /* 1 */
  int32_t n_scales;                /* 4 */
  int32_t scales[M3TB_MAX_SCHEDULE];           /* {6,4,2,1} */
  int32_t n_standard_deviations;   /* 4 */
  float standard_deviations[M3TB_MAX_SCHEDULE]; /* {15,5,3.5,1.5} */
  int32_t n_histogram_bins;        /* 16 */
  float learning_rate_f;           /* 0.2 */
  float learning_rate_b;           /* 0.2 */
  float unconsidered_line_length;  /* 0.5 */
  float max_considered_line_length; /* 20 */
  int32_t measure_occlusions;      /* 0 */
  float measured_depth_offset_radius; /* 0.01 */
  float measured_occlusion_radius;    /* 0.01 */
  float measured_occlusion_threshold; /* 0.03 */
  int32_t n_unoccluded_iterations; /* 10 */
  int32_t min_n_unoccluded_lines;  /* 0 */
  /* checks that read renderer images (handed over with m3tb_upload_*_rendering), region_modality.h:424-431 */
  int32_t model_occlusions;        /* 0  RegionModality::ModelOcclusions (focused depth rendering) */
  float modeled_depth_offset_radius;  /* 0.01 */
  float modeled_occlusion_radius;     /* 0.01 */
  float modeled_occlusion_threshold;  /* 0.03 */
  int32_t use_region_checking;     /* 0  RegionModality::UseRegionChecking (focused silhouette rendering) */
} m3tb_region_params;

/* Parameters of m3t::DepthModality, defaults depth_modality.h:302-321 */
typedef struct m3tb_depth_params {
  int32_t n_points_max;            /* 200 */
  int32_t use_adaptive_coverage;   /* 0 */
  int32_t use_depth_scaling;       /* 0 */
  float reference_surface_area;    /* 0 */
  float stride_length;             /* 0.005 */
  int32_t n_considered_distances;  /* 3 */
  float considered_distances[M3TB_MAX_SCHEDULE]; /* {0.05,0.02,0.01} */
  int32_t n_standard_deviations;   /* 3 */
  float standard_deviations[M3TB_MAX_SCHEDULE];  /* {0.05,0.03,0.02} */
  int32_t measure_occlusions;      /* 0 */
  float measured_depth_offset_radius; /* 0.01 */
  float measured_occlusion_radius;    /* 0.01 */
  float measured_occlusion_threshold; /* 0.03 */
  int32_t n_unoccluded_iterations; /* 10 */
  int32_t min_n_unoccluded_points; /* 0 */
  /* checks that read renderer images, depth_modality.h:305-312 */
  int32_t model_occlusions;        /* 0  DepthModality::ModelOcclusions (focused depth rendering) */
  float modeled_depth_offset_radius;  /* 0.01 */
  float modeled_occlusion_radius;     /* 0.01 */
  float modeled_occlusion_threshold;  /* 0.03 */
  int32_t use_silhouette_checking; /* 0  DepthModality::UseSilhouetteChecking (focused silhouette rendering) */
} m3tb_depth_params;

/* Parameters of m3t::Optimizer, defaults optimizer.h:52-53 */
typedef struct m3tb_optimizer_params {
  float tikhonov_parameter_rotation;    /* 1000 */
  float tikhonov_parameter_translation; /* 30000 */
} m3tb_optimizer_params;

/* One m3t::Link of a kinematic structure (M3T/include/m3t/link.h:150-156). */
typedef struct m3tb_link {
  int32_t body;                  /* body index of Link::body_ptr(), or -1 for a link without body */
  int32_t parent;                /* index of the parent link inside the structure's list, -1 for the root link */
  float body2joint[12];          /* Link::body2joint_pose(), row-major 3x4 */
  float joint2parent[12];        /* Link::joint2parent_pose() */
  float link2world[12];          /* Link::link2world_pose_ of a link without body (ignored when body >= 0) */
  int32_t free_directions[6];    /* Link::free_directions(): rot x,y,z, trans x,y,z */
  int32_t fixed_body2joint_pose; /* Link::fixed_body2joint_pose(), default 1 */
  /* Further modality sets of the SAME physical body (Link::modality_ptrs() holds an arbitrary list, link.h:151;
   * Link::CalculateGradientAndHessian sums it, link.cpp:184-193): e.g. a second colour + depth camera pair looking at the
   * body. Each set is an m3tb body of its own (own cameras, models, parameters, histograms); their gradients / Hessians
   * are added to the link's in list order and every pose update is written to all of them. */
  int32_t n_extra_bodies;        /* 0 .. M3TB_MAX_EXTRA_BODIES */
  int32_t extra_bodies[3];
} m3tb_link;
#define M3TB_MAX_EXTRA_BODIES 3

/* m3t::Constraint (M3T/include/m3t/constraint.h:109-112) or, with soft != 0, m3t::SoftConstraint
 * (M3T/include/m3t/soft_constraint.h:128-136). link1 / link2 index the structure's link list. */
typedef struct m3tb_constraint {
  int32_t link1, link2;
  float body12joint1[12], body22joint2[12];
  int32_t directions[6];         /* constraint_directions(): rot x,y,z, trans x,y,z */
  int32_t soft;
  float max_distance_rotation, max_distance_translation;             /* soft only, defaults 0 / 0 */
  float standard_deviation_rotation, standard_deviation_translation; /* soft only, defaults 0.01 / 0.001 */
} m3tb_constraint;

#define M3TB_MAX_LINKS 16         /* links per structure */
#define M3TB_MAX_SYSTEM 128       /* degrees of freedom + constraint rows of one structure */
#define M3TB_MAX_CONSTRAINTS 32   /* constraints + soft constraints per structure */

/* Per-line state kept between CalculateCorrespondences and CalculateGradientAndHessian
 * (RegionModality::DataLine, region_modality.h:150-165) - debug / parity read-back only. */
typedef struct m3tb_region_line {
  int32_t model_index;      /* index of the model point inside the closest view */
  int32_t valid;            /* 1 if the line survived IsLineValid + CalculateSegmentProbabilities */
  float center_f_body[3];
  float center_u, center_v;
  float normal_u, normal_v;
  float delta_r;
  float normal_component_to_scale;
  float distribution[M3TB_DISTRIBUTION_LENGTH];
  float mean;
  float measured_variance;
} m3tb_region_line;

/* DepthModality::DataPoint (depth_modality.h:139-150) - debug / parity read-back only. */
typedef struct m3tb_depth_point {
  int32_t model_index;
  int32_t valid;
  float center_f_body[3];
  float normal_f_body[3];
  float correspondence_center_f_camera[3];
} m3tb_depth_point;

/* ---- defaults (the reference's in-class member initialisers) ------------------------------- */
void m3tb_region_params_default(m3tb_region_params* p);       /* region_modality.h:411-443 */
void m3tb_depth_params_default(m3tb_depth_params* p);         /* depth_modality.h:302-321 */
void m3tb_optimizer_params_default(m3tb_optimizer_params* p); /* optimizer.h:52-53 */

/* ---- context -------------------------------------------------------------------------------- */
/* Creates a context on CUDA device `device`. Capacities are fixed at creation (the reference
 * allocates per object; here all bodies live in one batch). */
int m3tb_create(int device, int max_bodies, int max_cameras, int max_models, m3tb_ctx** out);
int m3tb_destroy(m3tb_ctx* ctx);
/* Use an existing cudaStream_t (e.g. torch's current stream) for all work; NULL = default stream. */
int m3tb_set_stream(m3tb_ctx* ctx, void* cuda_stream);
int m3tb_synchronize(m3tb_ctx* ctx);
const char* m3tb_last_error(const m3tb_ctx* ctx);
/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
int64_t m3tb_launch_count(const m3tb_ctx* ctx);

/* ---- sparse viewpoint models (inputs of RegionModel/DepthModel::GetClosestView) --------------- */
/* Replaces RegionModel::views_ (region_model.h:97-110) as filled by RegionModel::LoadModel
 * (region_model.cpp:259-307). `points` is n_views*n_points RegionModel::DataPoint records exactly
 * as stored in the .bin (152 B AoS); `orientations` n_views*3; `contour_lengths` n_views. */
int m3tb_set_region_model(m3tb_ctx* ctx, int model_id, int n_views, int n_points,
                          const float* orientations, const float* contour_lengths,
                          const void* points, float stride_depth_offset,
                          float max_radius_depth_offset);
/* Replaces DepthModel::views_ (depth_model.h:73-86); `points` are 144-B DepthModel::DataPoint. */
int m3tb_set_depth_model(m3tb_ctx* ctx, int model_id, int n_views, int n_points,
                         const float* orientations, const float* surface_areas,
                         const void* points, float stride_depth_offset,
                         float max_radius_depth_offset);

/* ---- cameras (Camera::intrinsics(), world2camera_pose(), image(); camera.h / camera.cpp:39) --- */
int m3tb_set_color_camera(m3tb_ctx* ctx, int cam, const m3tb_intrinsics* intrinsics,
                          const float world2camera[12]);
int m3tb_set_depth_camera(m3tb_ctx* ctx, int cam, const m3tb_intrinsics* intrinsics,
                          const float world2camera[12], float depth_scale);
/* Camera::UpdateImage: hand a host cv::Mat-style frame (CV_8UC3 BGR / CV_16UC1) to the device.
 * `pitch` is the host row pitch in bytes. Host memory stays caller-owned.
 *  - pageable memory: the whole frame is copied before the call returns control to the stream;
 *  - pinned (page-locked, mapped) memory: nothing is copied here. The next launch that consumes the frame first
 *    fetches, straight from the pinned frame over PCIe, only the rectangle each body can touch in this cycle
 *    (projected bounding sphere + longest correspondence line / widest depth window + motion margin); pixels
 *    outside it remain readable through the same zero-copy alias, so results never depend on the rectangle.
 *    LIFETIME (differs from Camera::UpdateImage, which copies): the camera keeps referring to the pinned frame.
 *    Every later launch on that camera - the tracking step, m3tb_calculate_results, a re-run on the same frame, any
 *    sample outside the fetched rectangle - may read it, so the frame must stay valid and unchanged until the NEXT
 *    upload to that camera has replaced it, or until m3tb_detach_frames() has returned. */
int m3tb_upload_color(m3tb_ctx* ctx, int cam, const uint8_t* bgr, size_t pitch);
int m3tb_upload_depth(m3tb_ctx* ctx, int cam, const uint16_t* depth, size_t pitch);
/* Gives the pinned frames back to the caller: every camera that still refers to a pinned host frame gets the whole
 * frame copied into its device copy (on the context's stream, synchronised before returning) and forgets the host
 * pointer. Afterwards the host buffers may be reused or freed; results of later calls are unchanged. */
int m3tb_detach_frames(m3tb_ctx* ctx);
/* Same, for frames that already live in device memory (device-resident pipelines, bench `value`). */
int m3tb_upload_color_device(m3tb_ctx* ctx, int cam, const void* dev_bgr, size_t pitch);
int m3tb_upload_depth_device(m3tb_ctx* ctx, int cam, const void* dev_depth, size_t pitch);

/* Renderer images for the checks that need them (the renderers themselves - OpenGL - stay with the caller):
 * FocusedDepthRenderer::focused_depth_image() for modeled occlusion handling (region_modality.cpp:1391-1431,
 * depth_modality.cpp:778-824) and FocusedSilhouetteRenderer::focused_silhouette_image() for region checking
 * (region_modality.cpp:1157-1223,1293-1341) / silhouette checking (depth_modality.cpp:728-734).
 * `modality`: 0 = the body's RegionModality (renderers of the colour camera), 1 = its DepthModality (depth camera).
 * image_size x image_size pixels, `pitch` bytes per row, host or device memory; corner_u / corner_v / scale as
 * FocusedRenderer reports them (renderer.h:195-197), projection terms as FocusedDepthRenderer::Depth uses them
 * (renderer.cpp:511-513: depth = a / (b - value)), `id` = Body::region_id() (region) / Body::body_id() (depth) the
 * silhouette is compared with, `visible` = FocusedRenderer::IsBodyVisible (0: the check is skipped, as in the
 * reference). The image is copied; call again whenever the renderer has produced a new one. */
typedef struct m3tb_rendering {
  const void* image;
  int32_t image_size;
  size_t pitch;
  float corner_u, corner_v, scale;
  float projection_term_a, projection_term_b; /* depth renderings only */
  int32_t id;                                 /* silhouette renderings only */
  int32_t visible;
} m3tb_rendering;
int m3tb_upload_depth_rendering(m3tb_ctx* ctx, int body, int modality, const m3tb_rendering* rendering);
int m3tb_upload_silhouette_rendering(m3tb_ctx* ctx, int body, int modality, const m3tb_rendering* rendering);

/* Loader-style batch ingest: `count` frames for cameras [first_cam, first_cam+count), frame k at
 * base + k*frame_stride bytes. Cameras of equal size share one device pool, so this is a single
 * host->device copy when the host frames are contiguous (frame_stride == height*pitch). */
int m3tb_upload_color_batch(m3tb_ctx* ctx, int first_cam, int count, const uint8_t* bgr,
                            size_t frame_stride, size_t pitch);
int m3tb_upload_depth_batch(m3tb_ctx* ctx, int first_cam, int count, const uint16_t* depth,
                            size_t frame_stride, size_t pitch);

/* ---- bodies: one rigid body = Body + RegionModality and/or DepthModality + root Link + Optimizer.
 * region == NULL / depth == NULL leaves that modality out (model / camera id then ignored).
 * Equivalent of constructing the objects and calling their SetUp() (region_modality.cpp:37-77,
 * depth_modality.cpp:34-60, optimizer.cpp:22-40). ------------------------------------------- */
int m3tb_set_body(m3tb_ctx* ctx, int body, const m3tb_region_params* region,
                  const m3tb_depth_params* depth, const m3tb_optimizer_params* optimizer,
                  int region_model, int depth_model, int color_camera, int depth_camera);
int m3tb_n_bodies(const m3tb_ctx* ctx);

/* Body::set_body2world_pose / body2world_pose (body.cpp:85-90) for bodies [first, first+count). */
int m3tb_set_poses(m3tb_ctx* ctx, int first, int count, const float* body2world);
int m3tb_get_poses(m3tb_ctx* ctx, int first, int count, float* body2world);

/* ColorHistograms::histogram_f_/histogram_b_ (color_histograms.h:96-97), n_bins^3 floats each. */
int m3tb_set_histograms(m3tb_ctx* ctx, int body, const float* histogram_f, const float* histogram_b);
int m3tb_get_histograms(m3tb_ctx* ctx, int body, float* histogram_f, float* histogram_b);

/* RegionModality::UseSharedColorHistograms / DoNotUseSharedColorHistograms (region_modality.cpp:168-179): `body` uses
 * the ColorHistograms object of `owner_body` (owner_body == -1: its own again). Members of a shared object only add their
 * line pixels in m3tb_start_modalities / m3tb_calculate_results; the object is initialised / updated ONCE from the sum of
 * all members' pixels (tracker.cpp:435-443, 507-515) with the owner's n_histogram_bins and learning rates (the shared
 * object's own parameters, color_histograms.h). The owner must not use another body's object itself; owner and members
 * need the same n_histogram_bins (checked at the next launch). m3tb_get_histograms of a member returns the shared
 * values, m3tb_set_histograms on any user sets them for all users. */
int m3tb_share_color_histograms(m3tb_ctx* ctx, int body, int owner_body);

/* ---- the hot path, fused: Tracker::ExecuteTrackingStep without CalculateResults (tracker.cpp:344-361)
 * for every body of the context: for corr in [0,n_corr): CalculateCorrespondences; for upd in
 * [0,n_update): CalculateGradientAndHessian + Optimizer::CalculateOptimization. One kernel launch. */
int m3tb_tracking_step(m3tb_ctx* ctx, int iteration, int n_corr_iterations, int n_update_iterations);
/* One correspondence iteration (the unit of BASELINE.json's metric): CalculateCorrespondences +
 * n_update x (CalculateGradientAndHessian + CalculateOptimization). */
int m3tb_corr_iteration(m3tb_ctx* ctx, int iteration, int corr_iteration, int n_update_iterations);

/* Tracker::StartModalities -> RegionModality::StartModality (region_modality.cpp:375-388):
 * first_iteration_ = iteration; histogram initialisation from the current pose and frame. */
int m3tb_start_modalities(m3tb_ctx* ctx, int iteration);
/* Tracker::CalculateResults -> RegionModality::CalculateResults (region_modality.cpp:572-583):
 * online histogram update with learning_rate_f/b. */
int m3tb_calculate_results(m3tb_ctx* ctx, int iteration);

/* ---- the hot path, fine-grained: mirrors the Modality / Optimizer methods 1:1 (parity, debugging,
 * and the CUDA Modality adapters driven by an unmodified m3t::Tracker). g/H may be NULL. ------- */
/* RegionModality::CalculateCorrespondences (region_modality.cpp:390-465), all bodies. */
int m3tb_region_correspondences(m3tb_ctx* ctx, int iteration, int corr_iteration);
/* RegionModality::CalculateGradientAndHessian (region_modality.cpp:485-558): g[n_bodies][6], H[n_bodies][36]. */
int m3tb_region_gradient_hessian(m3tb_ctx* ctx, int iteration, int corr_iteration, int opt_iteration,
                                 float* gradients, float* hessians);
/* DepthModality::CalculateCorrespondences (depth_modality.cpp:252-315). */
int m3tb_depth_correspondences(m3tb_ctx* ctx, int iteration, int corr_iteration);
/* DepthModality::CalculateGradientAndHessian (depth_modality.cpp:333-381). */
int m3tb_depth_gradient_hessian(m3tb_ctx* ctx, int iteration, int corr_iteration, int opt_iteration,
                                float* gradients, float* hessians);
/* Optimizer::CalculateOptimization (optimizer.cpp:144-167) for every body, using the gradients /
 * Hessians left on the device by the two calls above (Link::CalculateGradientAndHessian sums them,
 * link.cpp:184-193), then Link::UpdatePoses (link.cpp:205-241). */
int m3tb_calculate_optimization(m3tb_ctx* ctx, int iteration, int corr_iteration, int opt_iteration);

/* ---- kinematic structures (SURVEY §8 a13-a16, BASELINE config 5) --------------------------------------
 * One structure = one m3t::Optimizer with the Link tree below its root link, its Constraints and SoftConstraints
 * (Optimizer::Optimizer / AddConstraint / AddSoftConstraint + SetUp, M3T/src/optimizer.cpp:12-64). Links are listed in
 * Optimizer::ReferencedLinks() order (pre-order, optimizer.cpp:254-260), i.e. parent < own index; that is also the
 * order of the unknowns (DefineJacobians, optimizer.cpp:217-227). Structure ids are dense (0..n-1). Bodies that no
 * structure references keep the rigid-body optimiser of m3tb_set_body (one root link, body2joint = identity).
 * As soon as one structure exists, m3tb_tracking_step / m3tb_corr_iteration / m3tb_calculate_optimization run
 * Optimizer::CalculateOptimization per structure: Link::CalculateJacobian (link.cpp:159-182), SoftConstraint::
 * AddGradientsAndHessiansToLinks (soft_constraint.cpp:113-131), Constraint::CalculateResidualAndConstraintJacobian
 * (constraint.cpp:81-103), the (DoF + nc)^2 LDLT (optimizer.cpp:144-167) and Link::UpdatePoses (link.cpp:205-241).
 * Like Optimizer::SetUp, setting a structure makes the poses consistent (UpdatePoses with theta = 0). */
int m3tb_set_structure(m3tb_ctx* ctx, int structure, const m3tb_link* links, int n_links,
                       const m3tb_constraint* constraints, int n_constraints, const m3tb_optimizer_params* optimizer);
int m3tb_clear_structures(m3tb_ctx* ctx);
int m3tb_n_structures(const m3tb_ctx* ctx);
/* Link::ResetJointPoses (link.cpp:243-246) for every link: body2joint / joint2parent back to the values given to
 * m3tb_set_structure (the reference's default_*_pose_). One device-to-device copy, no synchronisation. */
int m3tb_reset_joint_poses(m3tb_ctx* ctx);
/* Optimizer::CalculateConsistentPoses (optimizer.cpp:133-142) for every structure. */
int m3tb_calculate_consistent_poses(m3tb_ctx* ctx);
/* Link::body2joint_pose / joint2parent_pose / link2world_pose of every link of one structure after the last update,
 * each [n_links][12]; any pointer may be NULL. */
int m3tb_get_link_poses(m3tb_ctx* ctx, int structure, float* body2joint, float* joint2parent, float* link2world);
/* theta of the last CalculateOptimization of one structure ([DoF + nc], debug / parity); *n_out = DoF + nc;
 * *updated = 0 when the NaN guard (optimizer.cpp:165) skipped the update. */
int m3tb_get_structure_theta(m3tb_ctx* ctx, int structure, float* theta, int capacity, int* n_out, int* updated);
/* Overwrites the gradient / Hessian a modality left on the device (what Modality::gradient() / hessian() return,
 * modality.h:132-137): modality 0 = region, 1 = depth; gradients[n_bodies][6], hessians[n_bodies][36] (symmetric).
 * For adapters that compute a modality elsewhere and for the parity tests of m3tb_calculate_optimization. */
int m3tb_set_gradient_hessian(m3tb_ctx* ctx, int modality, const float* gradients, const float* hessians);

/* ---- parity read-back of the per-line / per-point state (data_lines_, data_points_) ----------- */
/* `lines` must hold n_lines_max records; *n_out receives how many model points were processed. */
int m3tb_get_region_lines(m3tb_ctx* ctx, int body, m3tb_region_line* lines, int capacity, int* n_out);
int m3tb_get_depth_points(m3tb_ctx* ctx, int body, m3tb_depth_point* points, int capacity, int* n_out);
/* Index of the closest view chosen by the last *correspondences call (GetClosestView). */
int m3tb_get_closest_views(m3tb_ctx* ctx, int body, int* region_view, int* depth_view);

/* Optional frame prefetch (SURVEY f3: "overlap upload of frame t+1 with iterations of frame t"). Call it after the
 * pinned frames of the NEXT step have been handed over with m3tb_upload_* and while the current step may still be
 * running: the ROI ingest of those frames runs on a side stream into a second set of device buffers (the ROIs are
 * projected with the poses the last tracking launch started from), and the next tracking / histogram launch waits for
 * it. Results do not change (pixels outside a ROI are read from the pinned frame). It only takes effect when every
 * camera in use got a new pinned frame; otherwise, and for pageable frames, nothing happens and the frames are
 * ingested at the next launch as usual. The frames must stay unchanged until that next launch has completed. */
int m3tb_prefetch_frames(m3tb_ctx* ctx);
/* Bytes the last frame ingest (pinned-frame ROI fetch) moved host -> device; 0 if frames were copied in full. */
int m3tb_last_ingest_bytes(m3tb_ctx* ctx, unsigned long long* bytes);

/* Profiling aid (no reference counterpart): clock64() stamps taken by thread 0 of body `body` at the phase
 * boundaries of the last fused launch. Only available when the context was created with M3TB_TIMING=1 in the
 * environment. */
int m3tb_debug_phase_clocks(m3tb_ctx* ctx, int body, long long* out, int capacity);

/* Test aid (host only, no context, no GPU): RegionModel/DepthModel::GetClosestView (region_model.cpp:105-130) for
 * `n_queries` orientation vectors (R^T normalize(t), 3 floats each) over `n_views` view orientations, once by the
 * reference's full scan (`out_scan`) and once by the host restatement of the pruned search the kernels use
 * (`out_pruned`, started from view `prev[q]`; `out_evaluated[q]` = views it looked at). The two must be equal. */
int m3tb_debug_closest_view(const float* orientations, int n_views, const float* queries, int n_queries,
                            const int* prev, int* out_scan, int* out_pruned, int* out_evaluated);

#ifdef __cplusplus
}
#endif
#endif /* M3T_B200_H_ */
