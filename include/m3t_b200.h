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
 *  - a call that fails with M3TB_ERR_CUDA because a device / pinned allocation, stream or event could
 *    not be created leaves the context exactly as it was before the call: the same objects of the same
 *    sizes, the same host tables and the same renderer ids. Objects that are replaced (a model, a
 *    renderer's images, a grown table) are released only after their replacement exists. Calls that
 *    launch work (tracking, rendering, histogram updates) grow the device tables they need lazily, one
 *    set after another (structures, per-body state, renderer tables, shared-histogram groups): each set
 *    is replaced all or nothing, and a failure keeps the sets that were completed before it.
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
  /* Occlusion windows: an item whose window diameter is not finite or is negative (behind or level with the camera
   * that is scanned, or a non-finite pose) scans nothing and counts as unoccluded; items whose depth in the tracking
   * camera is not above 0 (NaN included) are dropped before any check. The reference's scans would not end there. */
  int32_t measure_occlusions;      /* 0 */
  float measured_depth_offset_radius; /* 0.01; must not exceed the model's max_radius_depth_offset nor round to a
                                         depth-offset id of 30 or more (M3TB_ERR_INVALID at the next launch) */
  float measured_occlusion_radius;    /* 0.01 */
  float measured_occlusion_threshold; /* 0.03 */
  int32_t n_unoccluded_iterations; /* 10 */
  int32_t min_n_unoccluded_lines;  /* 0 */
  /* checks that read renderer images (handed over with m3tb_upload_*_rendering), region_modality.h:424-431 */
  int32_t model_occlusions;        /* 0  RegionModality::ModelOcclusions (focused depth rendering) */
  float modeled_depth_offset_radius;  /* 0.01; the same limits as measured_depth_offset_radius */
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
  float considered_distances[M3TB_MAX_SCHEDULE]; /* {0.05,0.02,0.01}; finite, >= stride_length / 2, < 2^31 strides */
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

/* Parameters of m3t::TextureModality, defaults texture_modality.h:400-436. DescriptorType::ORB (32-byte binary
 * descriptors), BRISK and FREAK (64-byte binary descriptors), all NORM_HAMMING, and SIFT (128 floats) and DAISY
 * (1 .. 256 floats, 104 at M3T's defaults), both NORM_L2, are implemented; the detector's own settings stay with the
 * caller, who detects. */
#define M3TB_DESCRIPTOR_BRISK 0   /* TextureModality::DescriptorType::BRISK, texture_modality.h:153-162 */
#define M3TB_DESCRIPTOR_DAISY 1   /* TextureModality::DescriptorType::DAISY */
#define M3TB_DESCRIPTOR_FREAK 2   /* TextureModality::DescriptorType::FREAK */
#define M3TB_DESCRIPTOR_SIFT 3    /* TextureModality::DescriptorType::SIFT */
#define M3TB_DESCRIPTOR_ORB 4     /* TextureModality::DescriptorType::ORB */
typedef struct m3tb_texture_params {
  int32_t descriptor_type;                 /* M3TB_DESCRIPTOR_* (ORB_CUDA 5: M3TB_ERR_UNSUPPORTED) */
  int32_t focused_image_size;              /* 200 */
  float descriptor_distance_threshold;     /* 0.7 */
  float tukey_norm_constant;               /* 20 */
  int32_t n_standard_deviations;           /* 2 */
  float standard_deviations[M3TB_MAX_SCHEDULE]; /* {15, 5} */
  float max_keyframe_rotation_difference;  /* 10 deg, in radians */
  int32_t max_keyframe_age;                /* 100 */
  int32_t n_keyframes;                     /* 1 (1 .. 8) */
  int32_t measure_occlusions;              /* 0  (uses the body's depth camera, as the region modality does) */
  float measured_occlusion_radius;         /* 0.01 */
  float measured_occlusion_threshold;      /* 0.03 */
  int32_t model_occlusions;                /* 0  (needs a depth renderer attached with m3tb_attach_renderer) */
  float modeled_occlusion_radius;          /* 0.01 */
  float modeled_occlusion_threshold;       /* 0.03 */
  int32_t n_features_max;                  /* 512 (512 .. 4096): a device capacity, like n_lines_max; the reference
                                              has no counterpart and matches any number of features. The most
                                              keypoints one upload of the body may hand over; above 4096
                                              M3TB_ERR_UNSUPPORTED, below 512 M3TB_ERR_INVALID. */
} m3tb_texture_params;

/* TextureModality::DataPoint (texture_modality.h:136-141) - debug / parity read-back only. */
typedef struct m3tb_texture_point {
  float center_f_body[3];
  float correspondence_center[2];
  float center[2];
} m3tb_texture_point;

/* ---- defaults (the reference's in-class member initialisers) ------------------------------- */
void m3tb_region_params_default(m3tb_region_params* p);       /* region_modality.h:411-443 */
void m3tb_depth_params_default(m3tb_depth_params* p);         /* depth_modality.h:302-321 */
void m3tb_optimizer_params_default(m3tb_optimizer_params* p); /* optimizer.h:52-53 */
void m3tb_texture_params_default(m3tb_texture_params* p);     /* texture_modality.h:400-436 */

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
/* Both model setters refuse (M3TB_ERR_INVALID, the context unchanged) a stride_depth_offset that is not finite and
 * above 0, a max_radius_depth_offset that is not finite and >= 0, and int(max_radius_depth_offset /
 * stride_depth_offset + 1) above 30: what model generation refuses, and an infinite stride besides (every radius
 * would select depth offset 0 of a table the model cannot have been generated with). */
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

/* ---- device renderers: the focused renderers of the checks above, rendered on the device (k_render, DESIGN.md §3) so
 * that no OpenGL renderer and no image upload is needed. Rasterisation contract: DESIGN.md §3 "k_render".
 *
 * Body + RendererGeometry::AddBody (body.h, renderer_geometry.cpp): `triangles` is the body's triangle soup,
 * [n_triangles][3][3] floats in metres in the geometry frame, as RendererGeometry uploads it (after Body's unit scaling
 * and winding normalisation, body.cpp:201-249: counter-clockwise seen from outside); `geometry2body` the
 * Body::geometry2body_pose(); `enable_culling` Body::geometry_enable_culling(); body_id / region_id Body::body_id() /
 * region_id() (0..255). Independent of m3tb_set_body: a body that is only drawn (an occluder) needs only this and a pose. */
int m3tb_set_body_geometry(m3tb_ctx* ctx, int body, const float* triangles, int n_triangles,
                           const float geometry2body[12], float maximum_body_diameter, int enable_culling, int body_id,
                           int region_id);
/* FocusedBasicDepthRenderer / FocusedSilhouetteRenderer (basic_depth_renderer.h, silhouette_renderer.h; every device
 * renderer produces both images) of the colour (camera_kind 0) or depth (1) camera `camera`. `geometry_bodies` are drawn
 * in that order (RendererGeometry::render_data_bodies), `referenced_bodies` are the bodies the image focuses on
 * (FocusedRenderer::AddReferencedBody). Defaults (renderer.h:112-113,222): image_size 200, z_min 0.02, z_max 10.
 * id_type: 0 = IDType::BODY, 1 = IDType::REGION (the silhouette value). Renderer ids are dense (0..n). image_size above
 * 240 returns M3TB_ERR_UNSUPPORTED (the z-buffer lives in shared memory). A renderer attached to a modality cannot be
 * set again before it is detached. */
int m3tb_set_focused_renderer(m3tb_ctx* ctx, int renderer, int camera_kind, int camera, int image_size, float z_min,
                              float z_max, int id_type, const int* geometry_bodies, int n_geometry,
                              const int* referenced_bodies, int n_referenced);
/* RegionModality::ModelOcclusions / UseRegionChecking (region_modality.cpp:230-267) and DepthModality::ModelOcclusions /
 * UseSilhouetteChecking (depth_modality.cpp:128-161) with a device renderer: `modality` 0 region / 1 depth, `kind`
 * 0 depth image / 1 silhouette image; renderer -1 detaches (DoNot...). The renderer must render the modality's camera
 * and reference the body; a silhouette renderer must use id_type REGION for the region and BODY for the depth modality
 * (region_modality.cpp:66-86, depth_modality.cpp:56-76). The parameter flags (model_occlusions, use_region_checking,
 * use_silhouette_checking) still switch the checks. While a slot is attached, m3tb_upload_*_rendering on it fails.
 * With at least one slot attached, m3tb_tracking_step / m3tb_corr_iteration render every attached renderer before each
 * correspondence iteration (Tracker::CalculateCorrespondences, tracker.cpp:447-456), and m3tb_start_modalities /
 * m3tb_calculate_results first render the renderers attached to region modalities (tracker.cpp:430-434, 503-506).
 * Contexts without attached slots launch exactly what they launched before. */
int m3tb_attach_renderer(m3tb_ctx* ctx, int body, int modality, int kind, int renderer);
/* modality 2 = the body's TextureModality (m3tb_set_texture_modality) - its start and results renderers
 * (texture_modality.cpp:517-524): kind 1 the silhouette renderer, which SetUp requires and which must use id_type BODY
 * (Reconstruct3DPoint reads its silhouette and focused depth images), kind 0 the depth renderer of model_occlusions.
 * Both render the texture modality's colour camera and reference the body. m3tb_start_modalities and
 * m3tb_calculate_results render them before the texture modality's keyframe step. */
/* FocusedRenderer::StartRendering of every device renderer from the current poses (the fine-grained path calls it where
 * Tracker does). One kernel launch. */
int m3tb_render(m3tb_ctx* ctx);
/* Debug / parity read-back of one device renderer's last rendering: focused depth image (u16) and silhouette image (u8),
 * image_size x image_size, rows packed; corner_u / corner_v / scale, projection terms, and one
 * FocusedRenderer::IsBodyVisible flag per referenced body. Any pointer may be NULL. */
int m3tb_get_rendering(m3tb_ctx* ctx, int renderer, void* depth_u16, void* silhouette_u8, float* corner_u, float* corner_v,
                       float* scale, float* projection_term_a, float* projection_term_b, int* visible_flags);

/* ---- viewers (NormalColorViewer / NormalDepthViewer, normal_viewer.cpp; FullNormalRenderer, normal_renderer.cpp) ---
 * A viewer renders its geometry bodies over the whole camera image (width x height) with a full normal renderer
 * (FullRenderer::CalculateProjectionMatrix from the camera intrinsics, z range 0.02 .. 10, the defaults of the viewers'
 * renderers, normal_viewer.h:59,104) and alpha-blends the normal image over the camera frame (CalculateAlphaBlend).
 * DESIGN.md §3 "k_view_setup / k_view_raster / k_view_resolve" states what is computed. */
/* NormalColorViewer (kind 0, colour camera `camera`) or NormalDepthViewer (kind 1, depth camera `camera`) +
 * SetUp (normal_viewer.cpp:46-87,141-182): `geometry_bodies` are the RendererGeometry's bodies in draw order
 * (render_data_bodies), each with the geometry given by m3tb_set_body_geometry and its own culling flag; `opacity` is
 * set_opacity (reference default 0.5); min_depth / max_depth are the NormalDepthViewer's (defaults 0 and 1; ignored
 * for kind 0). Viewer ids are dense (0..n); setting an existing id replaces it. M3TB_ERR_INVALID for bad ids or kind,
 * an unset camera, a geometry body without geometry or a body listed twice. */
int m3tb_set_viewer(m3tb_ctx* ctx, int viewer, int kind, int camera, const int* geometry_bodies, int n_geometry,
                    float opacity, float min_depth, float max_depth);
/* Tracker::UpdateViewers (tracker.cpp:373) = UpdateViewer of every viewer (normal_viewer.cpp:97-113,192-211), from the
 * current poses, in stream order after any tracking launch: FullNormalRenderer::StartRendering + FetchNormalImage and
 * the alpha blend over the frame the camera holds (Camera::image(): the last upload; a pinned frame is read in place).
 * After m3tb_prefetch_frames the cameras already hold the next frames, so a caller who wants each frame paired with the
 * poses tracked on it updates the viewers before handing the next frames over. Three kernel launches for all viewers
 * together. m3tb_tracking_step never updates viewers. M3TB_ERR_NOT_SET_UP when a viewer's camera has never received a
 * frame; no viewer: nothing is launched. */
int m3tb_update_viewers(m3tb_ctx* ctx);
/* Read-back of viewer `viewer`'s last update: the blended BGR8 image (width x height, rows `pitch` bytes apart) and the
 * renderer's normal_image() (FullNormalRenderer::FetchNormalImage: BGRA8, GL_BGRA order with byte 0 = x, cleared to
 * 0, rows `normal_pitch` bytes apart). Either pointer may be NULL. M3TB_ERR_NOT_SET_UP before the first update since
 * the viewer was set or its camera changed size. */
int m3tb_get_viewer_image(m3tb_ctx* ctx, int viewer, uint8_t* bgr, size_t pitch, uint8_t* normal_bgra,
                          size_t normal_pitch);

/* ---- full renderers (FullBasicDepthRenderer / FullSilhouetteRenderer / FullNormalRenderer, renderer.cpp,
 * basic_depth_renderer.cpp, silhouette_renderer.cpp, normal_renderer.cpp) ---------------------------------------------
 * A full renderer draws its geometry bodies over the whole image of its camera (width x height, projection
 * FullRenderer::CalculateProjectionMatrix from the camera intrinsics and the renderer's own z range, world2camera from the
 * camera) with the viewers' rasteriser (DESIGN.md §3 "Full renderers"). Every full renderer produces all three images:
 * the depth image, the silhouette image and the normal image. */
/* FullBasicDepthRenderer / FullSilhouetteRenderer / FullNormalRenderer + SetUp of the colour (camera_kind 0) or depth
 * (1) camera `camera`: `geometry_bodies` are drawn in that order (RendererGeometry::render_data_bodies), each with the
 * geometry given by m3tb_set_body_geometry and its own culling flag. id_type: 0 = IDType::BODY, 1 = IDType::REGION (the
 * silhouette value). Full-renderer ids are dense (0..n) and separate from the focused renderers' and the viewers'; setting
 * an existing id replaces it. M3TB_ERR_INVALID for bad ids, kind, z range or id type, an unset camera, a geometry body
 * without geometry or a body listed twice. */
int m3tb_set_full_renderer(m3tb_ctx* ctx, int renderer, int camera_kind, int camera, float z_min, float z_max,
                           int id_type, const int* geometry_bodies, int n_geometry);
/* FullRenderer::StartRendering of every full renderer from the current poses, in stream order after any tracking
 * launch. Three kernel launches for all full renderers together, whatever their cameras and sizes. Never called by
 * m3tb_tracking_step or m3tb_update_viewers; no full renderer: nothing is launched. */
int m3tb_render_full(m3tb_ctx* ctx);
/* Read-back of full renderer `renderer`'s last render (width x height of its camera): FetchDepthImage (u16,
 * GL_DEPTH_COMPONENT16 as glReadPixels gives it, 65535 where nothing was drawn, row v = image row v), FetchSilhouetteImage
 * (u8, the drawn body's body_id or region_id, 0 for background) and FetchNormalImage (BGRA8 as m3tb_get_viewer_image),
 * rows `*_pitch` bytes apart, and FullDepthRenderer's projection terms (depth = a / (b - value), renderer.cpp:476-477).
 * Any pointer may be NULL. The images may go to host or device memory; the call waits for the copies only when one of
 * them goes to host memory. M3TB_ERR_NOT_SET_UP before the first render since the renderer was set or its camera
 * changed size. */
int m3tb_get_full_rendering(m3tb_ctx* ctx, int renderer, void* depth_u16, size_t depth_pitch, void* silhouette_u8,
                            size_t silhouette_pitch, void* normal_bgra, size_t normal_pitch, float* projection_term_a,
                            float* projection_term_b);

/* ---- focused normal renderers (FocusedNormalRenderer, normal_renderer.h:135-176, normal_renderer.cpp:295-423) -------
 * A focused normal renderer focuses on its referenced bodies as a focused renderer does
 * (FocusedRenderer::CalculateProjectionMatrix, renderer.cpp:348-405) and draws its geometry bodies into an
 * image_size x image_size depth image and normal image with the full renderers' rasteriser (DESIGN.md §3 "Focused normal
 * renderers"). Its depth image follows k_render's contract: up to the focused renderers' image_size limit of 240 it
 * equals, bit for bit, the depth image of a device focused renderer (m3tb_set_focused_renderer) with the same camera,
 * size, z range and bodies. */
/* FocusedNormalRenderer(name, renderer_geometry, camera, image_size, z_min, z_max) + AddReferencedBody + SetUp of the
 * colour (camera_kind 0) or depth (1) camera `camera`: `geometry_bodies` are drawn in that order
 * (RendererGeometry::render_data_bodies), each with the geometry given by m3tb_set_body_geometry and its own culling
 * flag; `referenced_bodies` are the bodies the image focuses on. Defaults (renderer.h:112-113,222): image_size 200, z_min
 * 0.02, z_max 10. Ids are dense (0..n) and separate from the focused renderers', the full renderers' and the viewers';
 * setting an existing id replaces it. M3TB_ERR_INVALID as for m3tb_set_focused_renderer; image_size above 4096 returns
 * M3TB_ERR_UNSUPPORTED (the z-buffer takes 8 bytes per pixel of device memory). */
int m3tb_set_focused_normal_renderer(m3tb_ctx* ctx, int renderer, int camera_kind, int camera, int image_size,
                                     float z_min, float z_max, const int* geometry_bodies, int n_geometry,
                                     const int* referenced_bodies, int n_referenced);
/* FocusedNormalRenderer::StartRendering (normal_renderer.cpp:361-369) of every focused normal renderer from the current
 * poses, in stream order after any tracking launch. Four kernel launches for all of them together. Never called by
 * m3tb_tracking_step, m3tb_render, m3tb_render_full or m3tb_update_viewers; none set: nothing is launched. */
int m3tb_render_focused_normals(m3tb_ctx* ctx);
/* Read-back of focused normal renderer `renderer`'s last render, image_size x image_size, rows packed:
 * FetchDepthImage (u16, GL_DEPTH_COMPONENT16, 65535 where nothing was drawn, row v = image row v), FetchNormalImage
 * (focused_normal_image(): BGRA8 as m3tb_get_full_rendering), corner_u / corner_v / scale, FocusedDepthRenderer's
 * projection terms (depth = a / (b - value)) and one FocusedRenderer::IsBodyVisible flag per referenced body. Any pointer
 * may be NULL. The images may go to host or device memory; the scalars and flags go to host memory. The call waits
 * unless every image goes to device memory and no scalar or flag is asked for. M3TB_ERR_NOT_SET_UP before the first
 * render since the renderer was set. */
int m3tb_get_focused_normal_rendering(m3tb_ctx* ctx, int renderer, void* depth_u16, void* normal_bgra, float* corner_u,
                                      float* corner_v, float* scale, float* projection_term_a,
                                      float* projection_term_b, int* visible_flags);

/* ---- normalised depth images (DepthCamera::NormalizedDepthImage, camera.cpp:108-115;
 * FullDepthRenderer::NormalizedDepthImage, renderer.cpp:407-427) ------------------------------------------------------ */
#define M3TB_NORMALIZED_DEPTH_CAMERA 0        /* source: depth camera `id` */
#define M3TB_NORMALIZED_DEPTH_FULL_RENDERER 1 /* source: full renderer `id` (m3tb_set_full_renderer) */
/* NormalizedDepthImage(min_depth, max_depth) as a u8 image of the source's size, rows `pitch` bytes apart, in host or
 * device memory (the call waits only for a host destination). One kernel launch.
 * - Depth camera: convertTo(CV_8UC1, alpha, beta) with alpha = 255 / ((max - min) / depth_scale) and
 *   beta = -(min / depth_scale) * alpha, as NormalDepthViewer computes it: one fused multiply-add, rounding half to even,
 *   saturation. It reads the frame the camera holds (the rectified frame when an undistortion is set; a pinned frame is
 *   read in place).
 * - Full renderer: per pixel uchar(min(max(a / (b - value) - min, 0), max - min) * 255 / (max - min)) of its last render.
 * M3TB_ERR_INVALID for a bad source, an unset camera or full renderer, max_depth <= min_depth (or NaN) and a pitch
 * smaller than a row; M3TB_ERR_NOT_SET_UP for a camera without a frame and a full renderer that has not rendered since
 * it was set or its camera changed size. */
int m3tb_get_normalized_depth_image(m3tb_ctx* ctx, int source, int id, float min_depth, float max_depth, void* dst,
                                    size_t pitch);

/* Loader-style batch ingest: `count` frames for cameras [first_cam, first_cam+count), frame k at
 * base + k*frame_stride bytes. Cameras of equal size share one device pool, so this is a single
 * host->device copy when the host frames are contiguous (frame_stride == height*pitch). */
int m3tb_upload_color_batch(m3tb_ctx* ctx, int first_cam, int count, const uint8_t* bgr,
                            size_t frame_stride, size_t pitch);
int m3tb_upload_depth_batch(m3tb_ctx* ctx, int first_cam, int count, const uint16_t* depth,
                            size_t frame_stride, size_t pitch);

/* ---- undistortion of raw frames as they are uploaded (AzureKinectColorCamera / AzureKinectDepthCamera::UpdateImage,
 * azure_kinect_camera.cpp:175-195, 321-345; k_undistort, DESIGN.md §3) --------------------------------------------- */
/* Host only (no context, no GPU), like m3tb_model_views: the map GetIntrinsicsAndDistortionMap builds
 * (azure_kinect_camera.cpp:234-265, 387-419): cv::initUndistortRectifyMap(CV_32FC1) with camera matrix `raw`, the
 * 8-coefficient rational model `distortion` in OpenCV order (k1, k2, p1, p2, k3, k4, k5, k6), R = I and new camera matrix
 * `rectified`, followed by cv::convertMaps(CV_16SC2, nninterpolation = true). `map_xy` receives height rows of width
 * (x, y) int16 pairs, `map_pitch` bytes apart. Every entry that lies inside the raw frame equals OpenCV's; entries far
 * outside it (|value| beyond the int16 range) may saturate differently and select the border value either way.
 * M3TB_ERR_INVALID for null pointers, raw and rectified sizes that differ or are not positive, non-finite intrinsics,
 * fu / fv <= 0, ppu / ppv < 0, non-finite coefficients or map_pitch < 4 * width. */
int m3tb_undistortion_map(const m3tb_intrinsics* raw, const float distortion[8], const m3tb_intrinsics* rectified,
                          int16_t* map_xy, size_t map_pitch);
/* Gives colour (camera_kind 0) or depth (1) camera `cam`, which must be set, a map (CV_16SC2 layout as above, the
 * camera's width x height, host or device memory, copied) that all its later uploads go through: the m3tb_upload_*
 * entry points then take the RAW frame, `channels` bytes per pixel for colour (4: the SDK's BGRA32, 3: BGR; the fourth
 * byte is dropped as COLOR_RGBA2RGB does) and u16 for depth (channels 1), pitch >= width * bytes per pixel, and leave
 * the rectified frame (cv::remap INTER_NEAREST, BORDER_CONSTANT: map entries outside the raw frame give 0) where an
 * upload always leaves it. Depth only: depth_value_offset (-32768 .. 32767, the reference's short(depth_offset /
 * depth_scale)) is added to every rectified pixel, border pixels included, with saturation to 0 .. 65535
 * (image_ += short); 0 adds nothing. A null map removes the undistortion (the camera keeps its last frame).
 * m3tb_set_*_camera with another width / height drops the undistortion; with the same size it is kept.
 * Each upload call to cameras with an undistortion adds one kernel launch (a batch: one for all of them); cameras
 * without one are uploaded exactly as before.
 *  - device frames are read in place; host frames, pageable or pinned, are copied whole into a staging buffer (grown
 *    lazily) and rectified from there, so the rectified camera refers to no host memory: m3tb_detach_frames has
 *    nothing to do for it, and m3tb_prefetch_frames, which needs pinned frames on every camera in use, does not
 *    prefetch while such a camera is in use;
 *  - LIFETIME of a pinned raw frame: it must stay unchanged until the stream has passed the upload (m3tb_synchronize,
 *    or any call that returns data to host memory).
 * A failed allocation leaves the context as it was. */
int m3tb_set_camera_undistortion(m3tb_ctx* ctx, int camera_kind, int cam, const int16_t* map_xy, size_t map_pitch,
                                 int channels, int32_t depth_value_offset);
/* Camera::image(): copies the frame camera `cam` (kind 0 colour BGR8, 1 depth u16) holds into `dst`, host or device
 * memory, rows `pitch` bytes apart (waits for the copy only when `dst` is host memory). A camera that still refers to a
 * pinned frame (ROI ingest) is read from that frame, so the result never depends on which rectangles were fetched.
 * M3TB_ERR_NOT_SET_UP before the camera's first upload. */
int m3tb_get_camera_image(m3tb_ctx* ctx, int camera_kind, int cam, void* dst, size_t pitch);

/* ---- bodies: one rigid body = Body + RegionModality and/or DepthModality + root Link + Optimizer.
 * region == NULL / depth == NULL leaves that modality out (model / camera id then ignored).
 * Equivalent of constructing the objects and calling their SetUp() (region_modality.cpp:37-77,
 * depth_modality.cpp:34-60, optimizer.cpp:22-40).
 * M3TB_ERR_INVALID, with nothing in the context changed, for a negative or non-finite measured / modeled occlusion
 * radius or depth-offset radius of either modality: it would stall the strided window scans (stride 0; the reference
 * loops forever) or index the depth-offset table below 0. ------------------------------------------- */
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

/* ---- texture modality (TextureModality, texture_modality.cpp; k_texture_keyframe / k_texture_match, DESIGN.md §3) -----
 * Feature detection stays with the caller, as the renderers once did (for ORB bodies m3tb_texture_detect_orb below runs
 * cv::ORB on the device instead): per frame it asks for each body's focus region,
 * crops and scales the grey image as DetectAndComputeCorrKeypoints does (texture_modality.cpp:866-868: cvtColor
 * BGR2GRAY, image(roi), resize by `scale` in both directions), runs cv::ORB, cv::SIFT or cv::xfeatures2d::DAISY on the
 * crop and hands the keypoints and descriptors over. Everything after detection runs on the device: keyframe
 * reconstruction from the device silhouette renderer with the occlusion checks, kNN matching with the ratio test
 * (Hamming for ORB, BRISK and FREAK, with k_texture_knn_hamming at correspondence iteration 0 for ORB bodies above 512
 * features and every BRISK / FREAK body; L2 for SIFT and DAISY, k_texture_knn_l2 at correspondence iteration 0), the
 * Tukey-weighted
 * reprojection gradient / Hessian in every update (inside k_track, added to the link after region and depth) and the
 * keyframe refresh. Bodies with a texture modality are tracked by k_track; contexts without one launch what they
 * launched before. A texture body may be the body of a link of a kinematic structure, or one of its extra bodies with
 * its own texture modality on its own camera (see m3tb_set_structure for the order of the link's sum). */
/* TextureModality + SetUp for body `body` (set with m3tb_set_body and m3tb_set_body_geometry, whose
 * maximum_body_diameter the focus region uses) on colour camera `color_camera`; NULL params remove the modality and
 * detach its renderers. Setting it again starts with an empty keyframe deque and, for SIFT / DAISY, clears the
 * descriptor length. M3TB_ERR_UNSUPPORTED for ORB_CUDA and for n_keyframes above 8, and for a change in place between
 * BRISK / FREAK and the other types: the binary upload and the keyframe read-back take no width, so a body that has a
 * texture modality of ORB, SIFT or DAISY gets BRISK or FREAK (or back) only after its removal (NULL params);
 * M3TB_ERR_INVALID for bad ids, an unset camera, a body without geometry, non-positive standard deviations or Tukey
 * constant, a negative or non-finite measured / modeled occlusion radius (a window stride of 0, a scan that never
 * ends), and measure_occlusions without the body's depth camera; a refused call changes nothing in the context.
 * M3TB_ERR_UNSUPPORTED for n_features_max above 4096 and M3TB_ERR_INVALID below 512.
 * Device memory: the tables hold C features per body slot for max_bodies, C the largest n_features_max any texture
 * body of the context has asked for (512 while every body keeps the default). The first call allocates the base
 * tables, 616 C bytes per slot (0.32 MB at 512, 2.5 MB at 4096); the first call with SIFT, DAISY, BRISK or FREAK adds
 * the wide descriptor tables and the match table, 9248 C bytes per slot (C frame and 8 x C keyframe rows of 256 words,
 * and 8 x C match results: 4.7 MB at 512, 37.9 MB at 4096; a BRISK / FREAK row uses 16 of its 256 words, so the
 * tables stay shared by every wide type); the first ORB body above 512 adds the match table alone
 * (32 C bytes per slot). A call that raises C remakes every table at the new C and keeps what the other bodies hold.
 * Each of these steps is all or nothing: on failure the context is as it was. */
int m3tb_set_texture_modality(m3tb_ctx* ctx, int body, const m3tb_texture_params* params, int color_camera);
/* TextureModality::CalculateScaleAndRegionOfInterest (texture_modality.cpp:890-931, margin 10 px) from the current
 * device poses, for bodies [first, first + count): roi[4 * k] = x, y, width, height, scale[k] the factor the crop is
 * resized by, valid[k] = 0 when the reference returns false (z < 1.5 r, an empty region) or the body has no texture
 * modality (roi and scale are then 0). Synchronises the stream. */
int m3tb_get_texture_focus(m3tb_ctx* ctx, int first, int count, int32_t* roi, float* scale, int32_t* valid);
/* The keypoints_ / descriptors_ of the current colour frame of one body: `n` (0 .. n_features_max) keypoints as (x, y) in crop
 * coordinates, which become roi + pt / scale in the image (texture_modality.cpp:884-887), and n binary descriptors of
 * the body's width: 32 bytes for ORB, 64 bytes for BRISK and FREAK, copied bit for bit. One upload per frame serves m3tb_start_modalities, correspondence iteration 0 (both detect on the same
 * frame at the same pose) and m3tb_calculate_results. A body whose camera received a newer frame since its last upload
 * has no features, as when the reference's detection returns early. M3TB_ERR_UNSUPPORTED above the body's
 * n_features_max features;
 * M3TB_ERR_INVALID for a SIFT / DAISY body (m3tb_upload_texture_float_features). The signature is ORB's; a BRISK or
 * FREAK body reads 64 n bytes from `descriptors`. */
int m3tb_upload_texture_features(m3tb_ctx* ctx, int body, const float* keypoints_xy, const uint8_t* descriptors, int n,
                                 int roi_x, int roi_y, float scale);
/* As m3tb_upload_texture_features for a SIFT or DAISY body: descriptors [n][length] floats, length 128 for SIFT and
 * 1 .. 256 for DAISY. The first upload after m3tb_set_texture_modality fixes the length; M3TB_ERR_INVALID for another
 * length later, for a non-finite descriptor value and for an ORB, BRISK or FREAK body. */
int m3tb_upload_texture_float_features(m3tb_ctx* ctx, int body, const float* keypoints_xy, const float* descriptors,
                                       int n, int length, int roi_x, int roi_y, float scale);
/* The focused grey images of bodies[0 .. count) on the device (k_texture_crop, one launch per 128 bodies): what
 * DetectAndComputeCorrKeypoints hands the detector (texture_modality.cpp:862-868),
 *   cv::cvtColor(color_camera_ptr_->image(), image, cv::COLOR_BGR2GRAY);
 *   cv::resize(image(roi), image, cv::Size(), scale, scale);   (INTER_LINEAR)
 * bit for bit as OpenCV computes it (DESIGN.md §3 "k_texture_crop"). roi and scale are m3tb_get_texture_focus's, from
 * the current device poses; the source is the camera's current frame wherever it is (a device copy, the rectified
 * frame of an undistorting camera, or a pinned frame read in place, whichever ROIs were fetched). Body k's crop is
 * size[2k] x size[2k + 1] bytes at out + k * body_stride, rows `pitch` bytes apart (device memory the caller owns),
 * size = saturate_cast<int>(roi.w * (double)scale) x ... as cv::resize sizes it; it grows with the distance of the
 * body. roi [count][4], scale [count], size [count][2] and valid [count] (0: no focus, nothing written) may be NULL.
 * The crop also records the body's roi, scale and frame for m3tb_upload_texture_features_device. M3TB_ERR_INVALID,
 * with nothing launched or recorded but the outputs filled, when a crop exceeds capacity_width x capacity_height;
 * M3TB_ERR_INVALID for a body without a texture modality or listed twice. Synchronises the stream once (poses). */
int m3tb_texture_crop(m3tb_ctx* ctx, const int* bodies, int count, uint8_t* out, size_t pitch, size_t body_stride,
                      int capacity_width, int capacity_height, int32_t* roi, float* scale, int32_t* size, int32_t* valid);
/* One body's features in device memory (cv::cuda::ORB's GpuMat keypoints and descriptors, a torch detector's
 * tensors): keypoint i at x[i * xy_stride], y[i * xy_stride] in crop coordinates (GpuMat rows: x and y rows of the
 * keypoint matrix, stride 1; interleaved xy: y = x + 1, stride 2); descriptor row i at descriptors + i *
 * descriptor_pitch bytes: with length 0 the binary width of the body's type (32 bytes for ORB, 64 for BRISK / FREAK;
 * descriptor_pitch at least that, no alignment needed, copied bit for bit and never checked as floats), or `length`
 * floats for SIFT / DAISY (4-byte aligned). */
typedef struct m3tb_device_features {
  int n;
  int length;
  const float* x;
  const float* y;
  int xy_stride;
  const void* descriptors;
  size_t descriptor_pitch;
} m3tb_device_features;
/* m3tb_upload_texture_features / _float_features for bodies[0 .. count) from device memory, in one k_texture_features
 * launch per 128 bodies and without synchronising: keypoints become float(roi_x) + x / scale with the roi and scale of
 * the body's last m3tb_texture_crop. Replaces, per body and frame, the host copy of the detector's output
 * (DetectAndComputeCorrKeypoints, texture_modality.cpp:870-887). Refusals as the host upload (M3TB_ERR_UNSUPPORTED
 * above the body's n_features_max features; M3TB_ERR_INVALID for the other descriptor kind, i.e. a nonzero length for a
 * binary body or 0 for a SIFT / DAISY body, a bad length and a length other than the first upload's), and
 * M3TB_ERR_INVALID for a body whose last crop is not of its camera's current frame; nothing is launched
 * when any body is refused. Float descriptors are checked on the device: a body with a non-finite value gets no
 * features this frame and its flag (m3tb_get_texture_feature_flags) is raised. The caller keeps the buffers unchanged
 * until the stream has passed the upload (any synchronising call). */
int m3tb_upload_texture_features_device(m3tb_ctx* ctx, const int* bodies, const m3tb_device_features* features,
                                        int count);
/* nonfinite[k] = 1 when body first + k's last m3tb_upload_texture_features_device held a non-finite descriptor
 * value (its features were dropped). Synchronises the stream. */
int m3tb_get_texture_feature_flags(m3tb_ctx* ctx, int first, int count, int32_t* nonfinite);
/* cv::ORB on the device (k_texture_orb, DESIGN.md §3 "k_texture_orb"). The detector settings M3T exposes
 * (texture_modality.h:410-412); everything else is cv::ORB's default, which M3T never changes: edgeThreshold 31,
 * firstLevel 0, WTA_K 2, HARRIS_SCORE, patchSize 31, fastThreshold 20. */
typedef struct m3tb_orb_params {
  int32_t n_features;   /* 300 (>= 1) */
  float scale_factor;   /* 1.2 (finite, > 1) */
  int32_t n_levels;     /* 3 (1 .. 8) */
} m3tb_orb_params;
void m3tb_orb_params_default(m3tb_orb_params* p);
/* DetectAndComputeCorrKeypoints (texture_modality.cpp:858-888) for the ORB bodies bodies[0 .. count), from the current
 * device poses and each body's camera's current frame: the focused crop (k_texture_crop, into context-owned scratch),
 * then cv::ORB detect and compute on it (k_texture_orb), the keypoints and descriptors stored in the body's feature
 * slot exactly as m3tb_upload_texture_features_device stores the same features in the same order (float(roi_x) +
 * x / scale). params [count] (NULL: m3tb_orb_params_default for every body). The result is bit-equal to OpenCV 4's
 * cv::ORB as a multiset of keypoints and descriptors. The order is canonical, not cv2's: level ascending, then
 * row-major by the keypoint's pixel in its level (cv2's order within a level comes from nth_element / partition).
 * cv::ORB can keep more than n_features keypoints, because its cuts keep every tie: a body that keeps more than its
 * n_features_max gets no features this frame (m3tb_get_texture_detections reports the count). A body without a focus
 * gets none either, as the reference returns early. Nor does a body whose pyramid has a level with a side of 0 pixels
 * (a small crop at a large scale_factor and many levels): cv::ORB builds every level before it detects and
 * cv::resize throws on the empty one, so cv::ORB returns no keypoints at all, the earlier levels' included; the
 * body's count is 0, with no read-back and no features, and the other bodies of the call are unaffected. Synchronises once (the poses); the counts stay on the device; two
 * launches per 128 bodies (one when none of them has a focus). Records the crop as m3tb_texture_crop does.
 * Refusals launch nothing and leave the context unchanged: M3TB_ERR_INVALID for a body without a texture modality, a
 * body whose descriptor type is not ORB, a body listed twice, n_features < 1, a scale_factor that is not finite or
 * not above 1 and n_levels < 1; M3TB_ERR_UNSUPPORTED for n_levels above 8 and n_features above 2^24;
 * M3TB_ERR_NOT_SET_UP without a colour frame.
 * Device memory: scratch of 16 bytes per pixel of the largest crop for up to 128 bodies (0.64 MB per body at
 * 200 x 200), grown on demand, and parity tables of 52 bytes per feature slot, made again when the feature capacity of
 * the context has grown (which forgets the other bodies' last detections); each growth is all or nothing. */
int m3tb_texture_detect_orb(m3tb_ctx* ctx, const int* bodies, int count, const m3tb_orb_params* params);
/* n_found[k]: the keypoints cv::ORB kept for body first + k at its last m3tb_texture_detect_orb (0 before one, and
 * after m3tb_set_texture_modality sets or removes the body's modality), which may exceed n_features (ties) and
 * n_features_max (the body then has no features). Synchronises the stream. */
int m3tb_get_texture_detections(m3tb_ctx* ctx, int first, int count, int32_t* n_found);
/* Parity read-back of body's last m3tb_texture_detect_orb, in the canonical order: xy [n][2] KeyPoint::pt in crop
 * (level-0) coordinates, angle [n] (degrees), response [n] (Harris), octave [n], descriptors [n][32]. The detection's
 * own copy: later feature uploads for the body do not change it. At most `capacity` keypoints; *n_out the number
 * stored (0 when the body kept more than its n_features_max, and when it has no detection: none yet, its texture
 * modality set or removed since, or the tables made again by a later detection of other bodies). Any output pointer
 * but n_out may be NULL. Synchronises the stream. */
int m3tb_get_texture_orb_keypoints(m3tb_ctx* ctx, int body, float* xy, float* angle, float* response, int32_t* octave,
                                   uint8_t* descriptors, int capacity, int* n_out);
/* TextureModality::CalculateCorrespondences (texture_modality.cpp:322-386) for every body with a texture modality:
 * matching at corr_iteration 0, the data points' projection (center) at every iteration. */
int m3tb_texture_correspondences(m3tb_ctx* ctx, int iteration, int corr_iteration);
/* TextureModality::CalculateGradientAndHessian (texture_modality.cpp:397-444): g[n_bodies][6], H[n_bodies][36] (zero
 * for bodies without a texture modality); the sums stay on the device for m3tb_calculate_optimization. The variance is
 * that of this call's corr_iteration, standard_deviations[min(corr_iteration, n_standard_deviations - 1)]; the
 * reference takes it from the last CalculateCorrespondences call, which in a tracking step has the same iteration. */
int m3tb_texture_gradient_hessian(m3tb_ctx* ctx, int iteration, int corr_iteration, int opt_iteration, float* gradients,
                                  float* hessians);
/* Parity read-back of the texture modality's data_points_ (at most `capacity`; *n_out receives the count). */
int m3tb_get_texture_points(m3tb_ctx* ctx, int body, m3tb_texture_point* points, int capacity, int* n_out);
/* Parity read-back of the keyframe deque, front to back: *n_keyframes deques entries, sizes[k] points each (sizes holds
 * 8 entries), their center_f_body [total][3] and descriptors (at most `capacity` points in all), the keyframe_age_ and
 * orientation_last_keyframe_[3]. Each descriptor is written at the body's width: [total][32] bytes for ORB,
 * [total][64] bytes for BRISK and FREAK, [total][length] floats (4 * length bytes) for SIFT and DAISY. Any output
 * pointer may be NULL. */
int m3tb_get_texture_keyframes(m3tb_ctx* ctx, int body, int* n_keyframes, int* sizes, float* points, uint8_t* descriptors,
                               int capacity, int* age, float* orientation);

/* ---- the hot path, fused: Tracker::ExecuteTrackingStep without CalculateResults (tracker.cpp:344-361)
 * for every body of the context: for corr in [0,n_corr): CalculateCorrespondences; for upd in
 * [0,n_update): CalculateGradientAndHessian + Optimizer::CalculateOptimization. One kernel launch. */
int m3tb_tracking_step(m3tb_ctx* ctx, int iteration, int n_corr_iterations, int n_update_iterations);
/* One correspondence iteration (the unit of BASELINE.json's metric): CalculateCorrespondences +
 * n_update x (CalculateGradientAndHessian + CalculateOptimization). */
int m3tb_corr_iteration(m3tb_ctx* ctx, int iteration, int corr_iteration, int n_update_iterations);

/* Tracker::StartModalities -> RegionModality::StartModality (region_modality.cpp:375-388):
 * first_iteration_ = iteration; histogram initialisation from the current pose and frame. Bodies with a texture
 * modality then run TextureModality::StartModality (texture_modality.cpp:314-320): a keyframe from the current pose. */
int m3tb_start_modalities(m3tb_ctx* ctx, int iteration);
/* Tracker::CalculateResults -> RegionModality::CalculateResults (region_modality.cpp:572-583):
 * online histogram update with learning_rate_f/b. Bodies with a texture modality then run
 * TextureModality::CalculateResults (texture_modality.cpp:456-472): like the reference, which does not call
 * PrecalculatePoseVariables there, the rotation rule and a new keyframe use the pose of the modality's last gradient
 * pass (the pose before the final update), while the renderers have drawn the final pose. */
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
 * Hessians left on the device by the calls above (Link::CalculateGradientAndHessian sums region, depth and texture,
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
 * A link's gradient / Hessian (Link::CalculateGradientAndHessian, link.cpp:184-193) is the sum over its modality sets:
 * its body's region, depth and texture terms (texture only where the body has a texture modality), then each extra
 * body's in the same order. An extra body is the same physical body seen by another camera set and may carry its own
 * texture modality on its own colour camera. With texture bodies, each update is one k_track launch (region, depth and
 * texture terms) and one k_structure launch; the texture match runs once per frame, at correspondence iteration 0.
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
/* Refiner::RefinePoses (refiner.cpp:76-117) for the rigid bodies `bodies` and the kinematic structures `structures`
 * (the Optimizers named). Defaults: n_corr_iterations 7, n_update_iterations 2 (refiner.h:40).
 * CalculateConsistentPoses of the named structures, then per correspondence iteration: render the start renderers of
 * the refined bodies, StartModality(0, corr) (first_iteration = 0, ClearMemory, line pixels, InitializeHistograms),
 * render their correspondence renderers, CalculateCorrespondences(0, corr) and n_update x (CalculateGradientAndHessian +
 * CalculateOptimization). A shared colour-histogram object with a refined member is initialised from the line pixels
 * of its refined members only, and every member reads the result. Every other body and structure is left exactly as
 * it was: poses, joint poses, histograms, lookup tables, per-line / per-point state, first_iteration, texture state and
 * the images of renderers that no refined body uses. The launches are those of the tracking step with one CTA per
 * refined body or structure (k_track, never k_track2; k_track once per run of consecutive refined bodies).
 * Both lists empty: M3TB_OK, nothing is launched. M3TB_ERR_INVALID: an id that is out of range or not set, an id listed
 * twice, a negative iteration count, or a body that is a link or an extra body of a structure (name the structure).
 * M3TB_ERR_UNSUPPORTED: a refined body, or a body of a refined structure, has a texture modality
 * (TextureModality::StartModality detects features before every correspondence iteration, which the caller does; for
 * ORB texture bodies m3tb_refine_poses_orb detects them on the device). */
int m3tb_refine_poses(m3tb_ctx* ctx, const int* bodies, int n_bodies, const int* structures, int n_structures,
                      int n_corr_iterations, int n_update_iterations);
/* m3tb_refine_poses with refined ORB texture bodies taking part, as Refiner::RefinePoses runs them: per correspondence
 * iteration, TextureModality::StartModality is DetectAndComputeCorrKeypoints on the device at the pose the iteration
 * starts from (m3tb_texture_detect_orb with orb_params[body]: one crop + ORB launch pair per 128 refined texture bodies)
 * and ComputeKeyframeData (k_texture_keyframe over the refined texture bodies: one new keyframe per iteration, at most
 * n_keyframes kept, age 0); their silhouette and depth renderers render with the start renderers. The bodies match
 * at correspondence iteration 0 only (texture_modality.cpp:332; kNN first where a body needs it), and every update adds
 * their texture term (k_track, or k_track + k_structure for structures). So a refined texture body ends with the
 * corr-0 data points and the features of the last iteration's detection. orb_params: NULL (m3tb_orb_params_default for
 * every body) or [m3tb_n_bodies(ctx)] entries by body id, of which only the refined texture bodies' are read.
 * A selection without texture bodies launches exactly what m3tb_refine_poses launches, with the same results.
 * Synchronises the host once per correspondence iteration with a texture body: detection reads the poses back to size
 * the focus crops. The detection scratch grows on demand, all or nothing; as the crop size follows the pose, it may
 * have to grow at a later iteration, and if that allocation fails the call returns M3TB_ERR_CUDA with the refined
 * bodies as the completed iterations left them (as the reference's loop returns false mid-way) and every other body
 * untouched; the context stays usable.
 * Refusals launch nothing and change nothing: every refusal of m3tb_refine_poses but the texture one;
 * M3TB_ERR_UNSUPPORTED for a refined texture body whose descriptor type is SIFT, DAISY, BRISK or FREAK (no device detector, and a
 * detection by the caller cannot run between the iterations of one call); the ORB-setting refusals of
 * m3tb_texture_detect_orb; M3TB_ERR_NOT_SET_UP when a refined texture body's camera has no colour frame, or the body
 * misses a renderer its texture modality needs. */
int m3tb_refine_poses_orb(m3tb_ctx* ctx, const int* bodies, int n_bodies, const int* structures, int n_structures,
                          int n_corr_iterations, int n_update_iterations, const m3tb_orb_params* orb_params);
/* Link::body2joint_pose / joint2parent_pose / link2world_pose of every link of one structure after the last update,
 * each [n_links][12]; any pointer may be NULL. */
int m3tb_get_link_poses(m3tb_ctx* ctx, int structure, float* body2joint, float* joint2parent, float* link2world);
/* theta of the last CalculateOptimization of one structure ([DoF + nc], debug / parity); *n_out = DoF + nc;
 * *updated = 0 when the NaN guard (optimizer.cpp:165) skipped the update. */
int m3tb_get_structure_theta(m3tb_ctx* ctx, int structure, float* theta, int capacity, int* n_out, int* updated);
/* Overwrites the gradient / Hessian a modality left on the device (what Modality::gradient() / hessian() return,
 * modality.h:132-137): modality 0 = region, 1 = depth, 2 = texture (once a texture modality has been set; only
 * bodies with one add it); gradients[n_bodies][6], hessians[n_bodies][36] (symmetric).
 * For adapters that compute a modality elsewhere and for the parity tests of m3tb_calculate_optimization. */
int m3tb_set_gradient_hessian(m3tb_ctx* ctx, int modality, const float* gradients, const float* hessians);
/* Test aid: Optimizer::CalculateOptimization + Link::UpdatePoses of n rigid bodies from given systems, through the
 * device's rigid-body solve on the shared-memory layout of k_track (solve 0) or of k_track2 (solve 1). a[n][36]: the normal matrix -H + diag(Tikhonov), only
 * its lower triangle is read; b[n][6]: the gradient; poses[n][12]: body2world, replaced by the updated pose (left as
 * it was when the NaN guard refuses the update); theta[n][6]: the solution before the guard; updated[n]: 1 if the
 * pose was updated. */
int m3tb_debug_rigid_solve(m3tb_ctx* ctx, int solve, int n, const float* a, const float* b, float* poses, float* theta,
                           int* updated);

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
 * camera in use got a new pinned frame; otherwise (a camera with an undistortion holds no pinned frame), and for
 * pageable frames, nothing happens and the frames are
 * ingested at the next launch as usual. The frames must stay unchanged until that next launch has completed. */
int m3tb_prefetch_frames(m3tb_ctx* ctx);
/* Bytes the last frame ingest (pinned-frame ROI fetch) moved host -> device; 0 if frames were copied in full. */
int m3tb_last_ingest_bytes(m3tb_ctx* ctx, unsigned long long* bytes);

/* Profiling aid (no reference counterpart): clock64() stamps taken by thread 0 of body `body` at the phase
 * boundaries of the last fused launch. Only available when the context was created with M3TB_TIMING=1 in the
 * environment. */
int m3tb_debug_phase_clocks(m3tb_ctx* ctx, int body, long long* out, int capacity);

/* Test aid (host only, no device work): which tracking-kernel variant the last tracking launch (m3tb_tracking_step,
 * m3tb_corr_iteration, the fine-grained correspondence / gradient calls) ran, so that a test can tell which code path
 * served it. All zero before the first tracking launch. */
typedef enum {
  M3TB_KERNEL_NONE = 0,
  M3TB_KERNEL_TRACK = 1,         /* k_track, the general kernel */
  M3TB_KERNEL_TRACK2 = 2         /* k_track2, the fused rigid-body kernel */
} m3tb_kernel;
typedef struct m3tb_launch_info {
  int32_t kernel;            /* m3tb_kernel */
  int32_t threads;           /* threads per body (CTA size) */
  int32_t items_per_thread;  /* lines and points each thread holds */
  int32_t lut_smem;          /* 1: the normalised LUT is staged in shared memory (every region body <= 16 bins) */
  int32_t occ;               /* 1: the variant with occlusion handling / renderer-image checks */
  int32_t tiles;             /* 1: ROI tiles are staged in shared memory */
  int32_t tma_mode;          /* k_track2: 0 legacy staging, 1 tensor maps as parameters, 2 in global memory; k_track: -1 */
} m3tb_launch_info;
int m3tb_debug_last_launch(m3tb_ctx* ctx, m3tb_launch_info* out);

/* Test aid: the histogram bin-index image of colour camera `cam` (one u16 lookup-table slot per pixel, the source of
 * k_track2's colour tiles) and the state that says which of its pixels are meant to be valid. Waits for the context's
 * stream and any prefetched ingest first. `out` (rows `out_pitch` bytes apart, width x height u16) may be null; nothing
 * is copied when the camera has no bin-index image (its frame is not in the shared pool, or the pool's width is not a
 * multiple of 4). info->rois (capacity info->roi_capacity, set by the caller) receives the colour ROI record of every
 * region body on the camera, in body order; info->n_rois is their number even when it exceeds the capacity. */
typedef struct m3tb_roi_record {
  int32_t body;
  int32_t x0, y0, x1, y1;    /* the rectangle k_ingest fetched: [x0, x1) x [y0, y1) */
  int32_t generation;        /* the camera generation it was fetched from, -1: never */
} m3tb_roi_record;
typedef struct m3tb_bin_image_info {
  int32_t state;             /* bit shift the image was written with; -1 none that matches the frame; -2 a pinned frame
                                whose bin indices the next ingest writes */
  int32_t pinned;            /* 1: the camera holds a pinned frame (device copy valid inside the ROIs only) */
  int32_t has_image;         /* 1: the camera has a bin-index image (and `out` received it) */
  int32_t width, height;
  int32_t generation;        /* the camera's frame generation */
  int32_t n_rois;
  int32_t roi_capacity;      /* in: capacity of rois */
  m3tb_roi_record* rois;     /* in: caller memory, may be null */
} m3tb_bin_image_info;
int m3tb_debug_bin_image(m3tb_ctx* ctx, int cam, uint16_t* out, size_t out_pitch, m3tb_bin_image_info* info);

/* Host only, meant for tests. *live (if not null) receives the number of CUDA resources the library holds across all
 * contexts: device allocations, pinned host allocations, streams and events. fail_after > 0 makes the fail_after-th
 * resource creation from now on fail as an allocation failure (cudaErrorMemoryAllocation) without calling CUDA;
 * 0 disarms that, a negative value only queries. */
int m3tb_debug_resources(int fail_after, long long* live);

/* ---- depth-model generation (DepthModel::GenerateModel, depth_model.cpp:144-213) -------------------------------- */
/* Model parameters (model.h:161-167). */
typedef struct m3tb_model_params {
  float sphere_radius;            /* distance of the virtual cameras from the body origin [m] */
  int32_t n_divides;              /* icosahedron subdivisions: 10 * 4^n_divides + 2 views */
  int32_t n_points;               /* surface points per view */
  float max_radius_depth_offset;  /* [m] */
  float stride_depth_offset;      /* [m]; max_radius / stride + 1 must not exceed 30 */
  int32_t use_random_seed;        /* must be 0: the reference seeds from the clock, which no test can reproduce */
  int32_t image_size;             /* full-frame render size [px], 21..8192 */
} m3tb_model_params;
/* sphere_radius 0.8, n_divides 4, n_points 200, max_radius_depth_offset 0.05, stride_depth_offset 0.002,
 * use_random_seed 0, image_size 2000 */
void m3tb_model_params_default(m3tb_model_params* p);
/* Generates depth model `model_id` of body `body` from the geometry given with m3tb_set_body_geometry: the geodesic
 * views are rendered on the device, each with the body alone (normal and depth image) and with the body in front of
 * the `n_occlusion_bodies` occlusion bodies (silhouette), all at body2world = I; a fresh std::mt19937{7} samples the
 * surface points of each view. The model then serves tracking exactly as if it had been uploaded with
 * m3tb_set_depth_model. Views whose silhouette is empty get zero-filled points. Returns M3TB_ERR_UNSUPPORTED for
 * use_random_seed != 0 and M3TB_ERR_INVALID for bad ids, a body without geometry, an offset ratio above 30 or a z_min
 * below 0.2 * sphere_radius (Model::SetUpRenderer / AddBodiesToRenderer); a refused call leaves the model as it was.
 * DESIGN.md §3 "k_model_raster / k_model_points" states what is computed. */
int m3tb_generate_depth_model(m3tb_ctx* ctx, int model_id, int body, const int* occlusion_bodies, int n_occlusion_bodies,
                              const m3tb_model_params* params);
/* Reads back a generated depth model; every output may be NULL: *n_views, *n_points, orientations [n_views][3],
 * surface_areas [n_views], points [n_views][n_points] x 144-B DataPoints (center_f_body[3], normal_f_body[3],
 * depth_offsets[30]), and the stride_depth_offset / max_radius_depth_offset it was generated with (what
 * m3tb_set_depth_model needs to rebuild the same depth-offset table). M3TB_ERR_NOT_SET_UP if the model was not
 * generated by m3tb_generate_depth_model. */
int m3tb_get_depth_model(m3tb_ctx* ctx, int model_id, int* n_views, int* n_points, float* orientations,
                         float* surface_areas, void* points, float* stride_depth_offset, float* max_radius_depth_offset);
/* Host only (no context, no GPU): the geodesic camera2body poses of a model (Model::GenerateGeodesicPoses,
 * model.cpp:386-454) as [n][12] row-major 3x4, in the order of the model's views; the view orientation is column 2.
 * *n_views receives the count; at most `capacity` (>= 0) poses are written (camera2body may be NULL). */
int m3tb_model_views(const m3tb_model_params* params, float* camera2body, int capacity, int* n_views);
/* Test aid: renders view `view` (geodesic order) of a depth-model generation with these arguments and returns its
 * normal image (image_size^2 x 4 B, GL_BGRA order, byte 0 = x), depth image (u16) and occlusion silhouette (u8);
 * any output may be NULL. Refusals as m3tb_generate_depth_model, plus a view index out of range. */
int m3tb_debug_render_model_view(m3tb_ctx* ctx, int body, const int* occlusion_bodies, int n_occlusion_bodies,
                                 const m3tb_model_params* params, int view, uint8_t* normal_bgra, uint16_t* depth,
                                 uint8_t* silhouette);

/* ---- region-model generation (RegionModel::GenerateModel, region_model.cpp:187-257) ------------------------------ */
/* RegionModel::AddAssociatedBody(body, movable, same_region), region_model.cpp:61-82: a fixed body (movable 0) is
 * drawn into the main silhouette with id 120 and its contour points are tested against its depth; a movable body
 * hides contour points it covers; a same-region body invalidates contour points next to it and extends the region
 * the line distances walk through. */
typedef struct m3tb_associated_body {
  int32_t body;
  int32_t movable;
  int32_t same_region;
} m3tb_associated_body;
/* Generates region model `model_id` of body `body` from the geometry given with m3tb_set_body_geometry, with the
 * `n_associated` associated bodies in insertion order (each of the four groups fixed, fixed same-region, movable,
 * movable same-region keeps that order, which is the draw order of the renderers). Every view is rendered on the
 * device with the renderers of the reference; the contours of the main silhouette are traced as
 * cv::findContours(RETR_LIST, CHAIN_APPROX_NONE) does, contours shorter than 15 points dropped, and a fresh
 * std::mt19937{7} samples the valid contour points. The model then serves tracking exactly as if it had been uploaded
 * with m3tb_set_region_model. Views without a valid contour point, and views whose sampling gives up after 101
 * consecutive rejections, get contour_length 0; points never produced are zero-filled. Refusals, which leave the model
 * as it was: M3TB_ERR_UNSUPPORTED for use_random_seed != 0 and for a view whose contours exceed 64 * image_size points;
 * M3TB_ERR_INVALID for bad ids, a body without geometry, the body listed as associated, a body listed twice, an
 * offset ratio above 30, any renderer's z_min below 0.2 * sphere_radius, or an image_size at which one view's z-buffers
 * (8 B per pixel and renderer) and contour scratch exceed the 1 GiB scratch bound (e.g. 5 renderers at 8192 px). DESIGN.md §3 "k_region_contours /
 * k_region_points" states what is computed. */
int m3tb_generate_region_model(m3tb_ctx* ctx, int model_id, int body, const m3tb_associated_body* associated,
                               int n_associated, const m3tb_model_params* params);
/* Reads back a generated region model like m3tb_get_depth_model; every output may be NULL: orientations [n_views][3],
 * contour_lengths [n_views], points [n_views][n_points] x 152-B DataPoints (center_f_body[3], normal_f_body[3],
 * foreground_distance, background_distance, depth_offsets[30]), stride / max radius of the depth offsets.
 * M3TB_ERR_NOT_SET_UP if the model was not generated by m3tb_generate_region_model. */
int m3tb_get_region_model(m3tb_ctx* ctx, int model_id, int* n_views, int* n_points, float* orientations,
                          float* contour_lengths, void* points, float* stride_depth_offset,
                          float* max_radius_depth_offset);
/* Test aid: renders view `view` of a region-model generation with these arguments and returns the silhouette image
 * (image_size^2 u8 each) of every renderer it uses, main first, then same-region, occlusion, foreground, background
 * (each only if used; *n_silhouettes receives the count), the main renderer's depth image (u16), and the contour list
 * as GenerateValidContours leaves it: *n_contour_points points as (x, y) int32 pairs in order, and *n_contours + 1
 * offsets into them. At most `capacity` points and capacity + 1 offsets are written; any output may be NULL.
 * Refusals as m3tb_generate_region_model, plus a view index out of range. */
int m3tb_debug_region_model_view(m3tb_ctx* ctx, int body, const m3tb_associated_body* associated, int n_associated,
                                 const m3tb_model_params* params, int view, uint8_t* silhouettes, int* n_silhouettes,
                                 uint16_t* depth, int32_t* contour_points, int32_t* contour_offsets, int capacity,
                                 int* n_contour_points, int* n_contours);

/* Test aid (host only, no context, no GPU): RegionModel/DepthModel::GetClosestView (region_model.cpp:105-130) for
 * `n_queries` orientation vectors (R^T normalize(t), 3 floats each) over `n_views` view orientations, once by the
 * reference's full scan (`out_scan`) and once by the host restatement of the pruned search the kernels use
 * (`out_pruned`, started from view `prev[q]`; `out_evaluated[q]` = views it looked at). The two must be equal. */
int m3tb_debug_closest_view(const float* orientations, int n_views, const float* queries, int n_queries,
                            const int* prev, int* out_scan, int* out_pruned, int* out_evaluated);

/* ---- pose scoring (the evaluators' CalculatePoseResults, examples/{ycb,rtb,opt,rbot}_evaluator.cpp) ---------------- */
#define M3TB_N_CURVE_VALUES 100  /* kNCurveValues of every evaluator */
/* Stores evaluation model `model` (ids dense: 0 .. the number set, below max_models; bodies share models): the full
 * vertex set `vertices` [n_vertices][3] in Body::vertices() order, which the nearest-neighbour search of ADD-S runs
 * against, and the reduced set of GenderateReducedVertices (ycb_evaluator.cpp:1222-1248): every vertex when
 * n_vertices_evaluation <= 0 or >= n_vertices, otherwise n_vertices_evaluation draws vertices[int(g() % n_vertices)]
 * of a fresh std::mt19937 g{7}. The reference's use_random_seed seeds from the clock and is not offered. Refused
 * (M3TB_ERR_INVALID, the model unchanged): bad id, NULL vertices, n_vertices < 1, a non-finite coordinate. */
int m3tb_set_evaluation_model(m3tb_ctx* ctx, int model, const float* vertices, int n_vertices, int n_vertices_evaluation);
/* Scores body `body` against evaluation model `model`; geometry2body (NULL: none) is the OPT evaluator's
 * kBody2Geometry2BodyPoseMap term of its delta pose. */
int m3tb_set_body_evaluation_model(m3tb_ctx* ctx, int body, int model, const float geometry2body[12]);
/* Reads the reduced set back: *n_vertices receives its size, at most `capacity` vertices [.][3] are written (vertices
 * may be NULL). */
int m3tb_get_evaluation_vertices(m3tb_ctx* ctx, int model, float* vertices, int capacity, int* n_vertices);

/* Curve and AUC scale, RBOT thresholds. YCB: threshold_max 0.1, curve_scale 1, auc_scale 1. OPT: threshold_max 0.2,
 * curve_scale = the body's diameter, auc_scale 0.2. RTB scores each body with threshold_max = ErrorThreshold and
 * averages on the host. */
typedef struct m3tb_score_params {
  float threshold_max;                /* 0.1 (YCBEvaluator::kThresholdMax) */
  float curve_scale;                  /* 1 */
  float auc_scale;                    /* 1 */
  float translation_error_threshold;  /* 0.05 m (rbot_evaluator.h:192) */
  float rotation_error_threshold;     /* 5 * kPi / 180 (rbot_evaluator.h:193) */
} m3tb_score_params;
void m3tb_score_params_default(m3tb_score_params* p);

typedef struct m3tb_pose_score {
  float add_error;          /* sum ||v - delta v|| / float(size) over the reduced set */
  float adds_error;         /* sum sqrt(min_w ||delta v - w||^2) / float(size), w over the full set */
  float add_auc;            /* auc_scale * (1 - std::min(error / (curve_scale * threshold_max), 1.0f)) */
  float adds_auc;
  float translation_error;  /* ||t - t_gt|| */
  float rotation_error;     /* acos((trace(R^T R_gt) - 1) / 2), R = Transform3fA::rotation() */
  float tracking_success;   /* 0 when either error is above its threshold, otherwise 1 (also for NaN errors) */
} m3tb_pose_score;
/* Scores the current device poses of bodies[0..n) against ground-truth body2world poses gt_body2world [n][12] (device
 * memory when gt_on_device != 0), on the context's stream after the work enqueued before it (no read-back of the
 * poses). delta = body2world.inverse() * gt, or (body2world * g2b).inverse() * gt * g2b with a geometry2body term. The
 * curves [n][M3TB_N_CURVE_VALUES] start at 1 and are 0 up to the first threshold
 * curve_scale * (threshold_max / 100) * (0.5 + i) the error falls below; add_curve / adds_curve may be NULL (both or
 * neither). out and the curves are device memory when out_on_device != 0; otherwise the call synchronises. A NaN error
 * gives a NaN AUC and a zero curve. As in nanoflann, a moved vertex whose distances are all NaN or infinite (a NaN or
 * infinite pose) takes FLT_MAX as its squared ADD-S distance. Refused (M3TB_ERR_INVALID, nothing launched): bad body ids, a body without an
 * evaluation model, n < 1, NULL gt / out / params, one curve pointer without the other, threshold_max or curve_scale
 * not finite and positive. DESIGN.md §3 "k_score / k_score_finish / k_diameter" states what is computed. */
int m3tb_score_poses(m3tb_ctx* ctx, const int* bodies, int n, const float* gt_body2world, int gt_on_device,
                     const m3tb_score_params* params, m3tb_pose_score* out, float* add_curve, float* adds_curve,
                     int out_on_device);
/* OPTEvaluator::CalculateDiameters (opt_evaluator.cpp:580-599): the largest (v_i - v_j).norm() over all pairs of each
 * model's full vertex set into out[n] (host memory; synchronises). Refused: bad or unset model ids, n < 1, NULL. */
int m3tb_calculate_diameters(m3tb_ctx* ctx, const int* models, int n, float* out);

#ifdef __cplusplus
}
#endif
#endif /* M3T_B200_H_ */
