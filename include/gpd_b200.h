/*
 * gpd_b200.h — C-ABI of libgpd_b200.so: the H100-native grasp-candidate hot path.
 *
 * This is the drop-in boundary for the ONE path of atenpas/gpd that this repo
 * accelerates (GraspDetector::detectGrasps steps 1-4, reference
 * src/gpd/grasp_detector.cpp:192-273):
 *
 *   sample index -> FrameEstimator local frame -> HandSearch/HandSet/FingerHand
 *   rotation sweep -> workspace/aperture filter -> ImageGenerator 60x60xC grasp
 *   image -> LeNet score.
 *
 * Conventions follow the reference's only C-ABI precedent,
 * src/detect_grasps_python.cpp:49-65,431-447,598-601: plain C structs and
 * pointers, return value = count (>= 0) or negative error code, no exceptions
 * cross the boundary, errors are also printed to stderr, the callee allocates
 * result arrays and the caller releases them with a library free function,
 * inputs are borrowed for the duration of the call only.
 *
 * Every entry point cites the reference interface it replaces. INTEGRATION.md
 * shows the reference-side bindings (a `CudaClassifier : net::Classifier`,
 * `HandSearch::searchHands`, `ImageGenerator::createImages`,
 * `GraspDetector::detectGrasps` shims) a maintainer would add.
 *
 * There is NO CPU fallback behind these symbols: every compute entry point
 * returns GPDB_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef GPD_B200_H_
#define GPD_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GPDB_VERSION 1

/* error codes (all negative; >= 0 is success / a count) */
#define GPDB_OK 0
#define GPDB_ERR_INVALID (-1)   /* bad argument / parameter                      */
#define GPDB_ERR_CUDA (-2)      /* CUDA runtime error or no usable device        */
#define GPDB_ERR_STATE (-3)     /* call order: cloud or weights not set          */
#define GPDB_ERR_IO (-4)        /* weight file missing or of the wrong size      */
#define GPDB_ERR_CAPACITY (-5)  /* a neighbourhood exceeded the on-chip tile     */

#define GPDB_MAX_CAMERAS 8
#define GPDB_MAX_HAND_AXES 3

/* pose_flags bits (one byte per (sample, axis, angle) pose) */
#define GPDB_POSE_VALID 1u     /* HandSet::is_valid_ after evalHands (hand_set.cpp:111)        */
#define GPDB_POSE_FILTERED 2u  /* survives filterGraspsWorkspace [+ filterGraspsDirection]     */
#define GPDB_POSE_HALF 4u      /* Hand::isHalfAntipodal (hand_set.cpp:255-261)                 */
#define GPDB_POSE_FULL 8u      /* Hand::isFullAntipodal                                        */

/* shadow_mode for the 15-channel occlusion channels (SURVEY.md 9.4, DESIGN.md) */
#define GPDB_SHADOW_DETERMINISTIC 0 /* counter-based draws; defined in include/gpd_b200_shadow.h */

/*
 * All parameters of the path. Field names are the reference's cfg keys; the
 * defaults are the reference's defaults (grasp_detector.cpp:48-86,130-185,
 * hand_geometry.cpp:25-30, image_geometry.cpp:24-28). gpdb_params_default()
 * fills them.
 */
typedef struct gpdb_params {
  /* candidate::HandGeometry (cfg/hand_geometry.cfg:8-12) */
  double finger_width;
  double hand_outer_diameter;
  double hand_depth;
  double hand_height;
  double init_bite;
  /* descriptor::ImageGeometry (cfg/image_geometry_15channels.cfg:8-12) */
  double volume_width;  /* ImageGeometry::outer_diameter_ */
  double volume_depth;
  double volume_height;
  int32_t image_size;
  int32_t image_num_channels; /* 1, 3, 12 or 15 */
  /* candidate::HandSearch::Parameters (grasp_detector.cpp:67-86) */
  double nn_radius; /* nn_radius_frames_ */
  int32_t num_orientations;
  int32_t num_finger_placements;
  int32_t num_hand_axes;
  int32_t hand_axes[GPDB_MAX_HAND_AXES];
  int32_t deepen_hand;
  double friction_coeff;
  int32_t min_viable;
  /* GraspDetector filters (grasp_detector.cpp:158-174) */
  double min_aperture;
  double max_aperture;
  double workspace_grasps[6];
  int32_t filter_approach_direction;
  double direction[3];
  double thresh_rad;
  /* net::Classifier (grasp_detector.cpp:130-138) */
  int32_t batch_size;       /* images per LeNet launch; 0 = library default          */
  int32_t relu_after_conv;  /* 0: Caffe/Eigen LeNet (no ReLU after conv, A14);        */
                            /* 1: the PyTorch/OpenVINO 12-channel net (pytorch/network.py:32-47) */
  /* library */
  int32_t shadow_mode;      /* GPDB_SHADOW_DETERMINISTIC                              */
  int32_t device;           /* CUDA device ordinal                                    */
  int32_t chunk_samples;    /* samples per device pass; 0 = library default           */
  int32_t keep_images;      /* gpdb_detect also returns the grasp images              */
  int32_t lenet_impl;       /* 0 = default (wgmma tensor cores), 1 = force SIMT fp32  */
} gpdb_params;

/* One grasp candidate = candidate::Hand (include/gpd/candidate/hand.h:267-276). */
typedef struct gpdb_pose {
  double sample[3];   /* Hand::sample_                                             */
  double frame[9];    /* Hand::orientation_, column-major: approach|binormal|axis  */
  double position[3]; /* Hand::position_ (hand.cpp:41-45)                          */
  double top;         /* BoundingBox::top_                                         */
  double bottom;
  double center;
  double width;       /* Hand::grasp_width_                                        */
  float score;        /* Label::score_ = logits[1] - logits[0] (eigen_classifier.cpp:74) */
  int32_t sample_index; /* index of the sample in the cloud                        */
  int32_t sample_slot;  /* position in the sample_idx array passed to the call     */
  int16_t pose_slot;    /* axis_i * num_orientations + angle_i                     */
  int16_t finger_idx;   /* Hand::finger_placement_index_                           */
  uint8_t half_antipodal;
  uint8_t full_antipodal;
  uint8_t pad_[6];    /* explicit tail padding (zero): sizeof(gpdb_pose) = 176 with no implicit bytes */
} gpdb_pose;

/* Result of gpdb_detect / gpdb_hand_search: callee-allocated, release with gpdb_free_result. */
typedef struct gpdb_result {
  int32_t n_samples;
  int32_t poses_per_sample; /* num_hand_axes * num_orientations                     */
  uint8_t *frame_valid;     /* [n_samples] 0 where calculateFrame found no neighbour */
  double *frames;           /* [n_samples*9] LocalFrame: normal|binormal|curvature_axis */
  uint8_t *pose_flags;      /* [n_samples*P] GPDB_POSE_* bits                        */
  float *pose_scores;       /* [n_samples*P] score, NaN where no image was classified */
  int32_t n_candidates;     /* poses with VALID and FILTERED set                     */
  gpdb_pose *candidates;    /* [n_candidates] in (sample slot, pose slot) order =    */
                            /* hands_out order of image_generator.cpp:91-98          */
  uint8_t *images;          /* [n_candidates*S*S*C] HWC uint8 (cv::Mat CV_8UC(C)) or NULL */
  double ms_candidates;     /* device time of "1. Candidate generation"  (grasp_detector.cpp:313) */
  double ms_images;         /*                "2. Descriptor extraction"                     */
  double ms_classify;       /*                "3. Classification"                            */
  int64_t kernel_launches;  /* CUDA kernels launched by this call                     */
  int32_t n_total_candidates; /* all poses with VALID and FILTERED set (= n_candidates except after gpdb_detect_select) */
  void *owner_;             /* library-private: the pinned host arena the arrays above live in (gpdb_free_result) */
} gpdb_result;

typedef struct gpdb_ctx gpdb_ctx;

/* Fill *p with the reference defaults (15-channel images, hand_axes = {2}). */
void gpdb_params_default(gpdb_params *p);

/* Replaces: GraspDetector::GraspDetector(cfg) (grasp_detector.cpp:5-190). One context = one
 * CUDA device + stream; calls on one context are serialised by the caller. */
int gpdb_create(const gpdb_params *params, gpdb_ctx **ctx_out);
void gpdb_destroy(gpdb_ctx *ctx);

/* Message of the last error on this context (or of the last failed gpdb_create when ctx==NULL). */
const char *gpdb_last_error(const gpdb_ctx *ctx);

/* Replaces: EigenClassifier::EigenClassifier weight loading (eigen_classifier.cpp:24-47).
 * `dir` is the `weights_file` cfg value: a directory (with trailing '/') holding
 * {conv1,conv2,ip1,ip2}_{weights,biases}.bin in the reference's raw float32 layout. */
int gpdb_load_weights_dir(gpdb_ctx *ctx, const char *dir);

/* Replaces: Classifier::create(model_file, weights_file, ...) weight loading for the reference's other backends
 * (classifier.cpp:33-61): `weights_file` may be a .bin parameter directory (trailing '/', as above), a Caffe
 * `.caffemodel` (layers conv1, conv2, ip1, ip2; caffe_classifier.cpp) or an OpenVINO IR `.bin` whose `.xml` is
 * `model_file` (or lies next to it; openvino_classifier.cpp:20-57). The blobs are converted to the .bin layout on the
 * host. An IR with ReLU after the convolutions needs a context created with relu_after_conv = 1. */
int gpdb_load_weights_file(gpdb_ctx *ctx, const char *model_file, const char *weights_file);
/* The host-side conversion alone (no device): fills eight caller-allocated arrays (sizes as gpdb_set_weights) in the
 * .bin layout; relu_layers_out = number of ReLU layers of an IR, -1 for a caffemodel; err_out receives the message. */
int gpdb_read_weights_file(const char *model_file, const char *weights_file, int32_t channels, float *const out[8],
                           int32_t *relu_layers_out, char *err_out, int32_t err_len);

/* Same, from memory, in the layout of the .bin files (A14): conv = OIHW row-major,
 * ip = column-major (out, in). Sizes: conv1 20*C*25, conv2 50*20*25, ip1 500*7200, ip2 2*500.
 * Any finite float32 weights are accepted. The tensor-core conv1 holds each filter as 24-bit integers times a float32
 * scale s_o ~ max|w_o| / 8.3e6; for max|w_o| below ~1e-36 that scale is subnormal, so s_o is rounded up until
 * max|w_o| / s_o <= 127 * 65536 + 127 * 257 (no digit overflows) and such a filter keeps fewer than 24 bits, down to its
 * weights' own subnormal resolution (s_o >= 2^-149). The power-of-two fp16 scale of the conv2 / ip1 weights is
 * held to 2^127 when their max|w| is below ~5e-38. The per-layer error bounds of both implementations are in
 * tests/lenet_layer_bounds.py. */
int gpdb_set_weights(gpdb_ctx *ctx, const float *conv1_w, const float *conv1_b,
                     const float *conv2_w, const float *conv2_b, const float *ip1_w,
                     const float *ip1_b, const float *ip2_w, const float *ip2_b);

/* Replaces: the util::Cloud accessors the path reads (include/gpd/util/cloud.h:300-366):
 *   xyz          getCloudProcessed() points, packed float32 x,y,z (3*N)
 *   normals      getNormals(), 3 x N float64 column-major
 *   cam_source   getCameraSource(), k x N int32 column-major (may be NULL: all ones)
 *   view_points  getViewPoints(), 3 x k float64 column-major
 * Builds the device neighbour grid (replaces the two KdTreeFLANN builds,
 * hand_search.cpp:29-31, image_generator.cpp:37-38). */
int gpdb_set_cloud(gpdb_ctx *ctx, const float *xyz, const double *normals,
                   const int32_t *cam_source, int32_t n_points, const double *view_points,
                   int32_t n_cams);

/* Replaces: Cloud::setSamples (cloud.cpp:662; used by SequentialImportanceSampling, sequential_importance_sampling.cpp:
 * 130-131,166-168): n arbitrary float64 sample positions (3 x n column-major) next to the installed cloud. Returns N, the
 * first sample index that addresses them: gpdb_detect / gpdb_frames / gpdb_hand_search / gpdb_detect_select accept sample
 * indices N .. N + n - 1 for these positions (indices < N keep addressing cloud points, Cloud::getSampleIndices). The
 * local frame and the radius searches use the float32 image of the position, the hand-frame transforms the float64
 * position, as the reference does; the shadow draws are seeded by the sample index as for cloud points. A new cloud
 * (gpdb_set_cloud / gpdb_preprocess) drops the positions. */
int gpdb_set_samples(gpdb_ctx *ctx, const double *samples_xyz, int32_t n_samples);

/* Replaces: GraspDetector::detectGrasps steps 1-4 (grasp_detector.cpp:222-273) for the
 * samples cloud.getSampleIndices() (cloud.h:345). Returns n_candidates or a negative error. */
int gpdb_detect(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n_samples, gpdb_result *out);

/* Replaces: GraspDetector::detectGrasps steps 1-4 followed by selectGrasps (grasp_detector.cpp:222-283,405-420): the
 * `num_selected` highest-scoring candidates, sorted by descending score (ties: (sample slot, pose slot) order), selected
 * ON THE DEVICE — only those pose records cross PCIe. out->candidates holds n_candidates = min(num_selected, total)
 * records, out->n_total_candidates the number of classified candidates; the per-sample / per-pose arrays
 * (frame_valid, frames, pose_flags, pose_scores, images) are NULL. Returns n_candidates or a negative error. */
int gpdb_detect_select(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n_samples, int32_t num_selected,
                       gpdb_result *out);

/* Device-resident variant of gpdb_detect: d_sample_idx [n], d_flags_out [n*P] and d_scores_out [n*P]
 * are DEVICE pointers on the context's device; no input or result crosses PCIe (only the per-chunk
 * candidate count is read back to size the image / classifier launches). `stats` receives
 * n_candidates, stage timings and the launch count; its array members stay NULL. The caller
 * guarantees 0 <= sample index < N. Used to measure the path with inputs resident in HBM. */
int gpdb_detect_resident(gpdb_ctx *ctx, const int32_t *d_sample_idx, int32_t n_samples, uint8_t *d_flags_out,
                         float *d_scores_out, gpdb_result *stats);

/* --- batches of clouds: many small scenes (views of objects, dataset evaluation, multi-camera cells) in one call -------
 * gpdb_set_clouds installs B processed clouds, concatenated: cloud b owns the points point_offsets[b] ..
 * point_offsets[b+1] - 1 of xyz (3 floats per point) and normals (3 doubles per point), its own n_cameras[b] = K_b <= 8
 * cameras (view_points: the 3 x K_b blocks of the clouds one after the other) and camera sources (cam_source: the
 * N_b x K_b int32 blocks one after the other, entries > 0 = seen, as gpdb_set_cloud; NULL = every camera sees every point).
 * Every cloud gets its own neighbour grid on the device; the batch is held beside the single cloud, and gpdb_set_cloud,
 * gpdb_preprocess, gpdb_detect and every other entry point behave as before whatever batch is installed. Empty clouds,
 * K_b outside 1..8, non-finite coordinates and malformed offsets are GPDB_ERR_INVALID; a failed call leaves no batch.
 * Returns B. gpdb_set_samples addresses the single cloud only: called while only a batch is installed, it is
 * GPDB_ERR_INVALID (a batch takes its positions from gpdb_set_clouds_samples). Raw views are preprocessed into a batch by
 * gpdb_preprocess_clouds. */
int gpdb_set_clouds(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *point_offsets, const float *xyz, const double *normals,
                    const int32_t *cam_source, const int32_t *n_cameras, const double *view_points);

/* gpdb_detect over every cloud of the batch in ONE call: sample_idx holds indices LOCAL to each cloud in CSR form (cloud b:
 * sample_idx[sample_offsets[b] .. sample_offsets[b+1]), an empty range is allowed). The result is one gpdb_result in
 * concatenated sample order: frames, flags and scores per sample of the whole stream; candidates (and images with
 * keep_images) grouped by cloud, cloud b's at cand_offsets_out[b] .. cand_offsets_out[b+1] - 1. Pose records carry the
 * cloud-local sample_index and sample_slot, so each cloud's slice equals gpdb_detect on that cloud alone, bit for bit.
 * sample_offsets and cand_offsets_out hold B + 1 entries for the B clouds of the installed batch (the call takes no
 * count: the caller keeps it from gpdb_set_clouds). A local index outside its cloud or malformed offsets:
 * GPDB_ERR_INVALID; a neighbourhood beyond the last tier anywhere: GPDB_ERR_CAPACITY for the whole call. The image limits of gpdb_detect apply to the largest K_b of the batch. */
int gpdb_detect_batch(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *sample_idx, gpdb_result *out,
                      int32_t *cand_offsets_out);

/* gpdb_detect_select applied to every cloud of the batch: the num_selected best candidates of each cloud (descending score,
 * ties in (sample slot, pose slot) order), chosen by one stable sort on the device; only they cross PCIe. Cloud b's
 * records are out->candidates[sel_offsets_out[b] .. sel_offsets_out[b+1]); out->n_total_candidates counts the classified
 * candidates of all clouds. */
int gpdb_detect_batch_select(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *sample_idx, int32_t num_selected,
                             gpdb_result *out, int32_t *sel_offsets_out);

/* Cloud::setSamples for every cloud of the installed batch (SequentialImportanceSampling over many views): cloud b owns
 * the columns pos_offsets[b] .. pos_offsets[b+1]-1 of samples_xyz (3 x M float64, column-major, as gpdb_set_samples;
 * pos_offsets has B + 1 entries, starts at 0 and never decreases; an empty range is allowed). In gpdb_detect_batch,
 * gpdb_detect_batch_select and gpdb_hand_search_batch the local index N_b + j then addresses position j of cloud b
 * (indices below N_b keep addressing points), and each cloud's results equal gpdb_set_cloud + gpdb_set_samples + the
 * single-cloud call on that cloud, bit for bit (shadow draws are seeded by the cloud-local index). Each call replaces all
 * positions; a failed call, and any gpdb_set_clouds / gpdb_preprocess_clouds, successful or not, leaves none. The single
 * cloud's positions (gpdb_set_samples) and these never touch each other. Returns M; GPDB_ERR_STATE when no batch is
 * installed, GPDB_ERR_INVALID for malformed offsets. */
int gpdb_set_clouds_samples(gpdb_ctx *ctx, const int32_t *pos_offsets, const double *samples_xyz);

/* gpdb_hand_search over every cloud of the batch in ONE call: inputs and output layout of gpdb_detect_batch (cloud b's
 * candidates at cand_offsets_out[b] .. cand_offsets_out[b+1] - 1), no images, pose_scores NaN. Needs no weights. */
int gpdb_hand_search_batch(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *sample_idx, gpdb_result *out,
                           int32_t *cand_offsets_out);

/* Run all work of this context on an existing CUDA stream (cudaStream_t passed as void*), e.g. the
 * host framework's current stream, instead of the context's own stream. */
int gpdb_set_stream(gpdb_ctx *ctx, void *cuda_stream);

/* The chunk pipeline runs the hand search of the chunks ahead on a second stream, concurrently with the image stage and
 * the classifier of the current chunk (default: on; environment GPD_B200_OVERLAP=0 turns the default off). With
 * enable = 0 every kernel of a call runs on the context's stream, one after the other: the stage timers of
 * gpdb_last_timings are then exclusive per stage (bench.py takes its per-kernel times from such a pass). Results are
 * identical either way. */
int gpdb_set_overlap(gpdb_ctx *ctx, int32_t enable);

/* Stage-level entry points (used by the parity tests and by partial drop-ins). */

/* Replaces: FrameEstimator::calculateLocalFrames (frame_estimator.cpp:6-35).
 * frames_out [n*9] normal|binormal|curvature_axis, valid_out [n]. */
int gpdb_frames(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n_samples, double *frames_out,
                uint8_t *valid_out);

/* Replaces: HandSearch::searchHands (hand_search.cpp:24-64) + filterGraspsWorkspace /
 * filterGraspsDirection (grasp_detector.cpp:334-398,422-456). No images, no scores. */
int gpdb_hand_search(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n_samples,
                     gpdb_result *out);

/* Replaces: ImageGenerator::createImages (image_generator.cpp:17-70) for given hands.
 * images_out [n_poses * S*S*C] HWC uint8. */
int gpdb_images(gpdb_ctx *ctx, const gpdb_pose *poses, int32_t n_poses, uint8_t *images_out);

/* Replaces: Classifier::classifyImages (classifier.h:72-73; eigen_classifier.cpp:59-79).
 * images_hwc [n * S*S*C] continuous cv::Mat data; scores_out [n]; logits_out [n*2] or NULL. */
int gpdb_classify(gpdb_ctx *ctx, const uint8_t *images_hwc, int32_t n_images, float *scores_out,
                  float *logits_out);

/* --- cloud preprocessing (SURVEY.md 8(f).1: the step immediately before the path) -------------- */

/* Parameters of CandidatesGenerator::preprocessPointCloud (candidates_generator.cpp:14-37); field names are
 * the reference's cfg keys (grasp_detector.cpp:50-66, cfg/eigen_params.cfg:16-21). */
typedef struct gpdb_preprocess_params {
  double workspace[6];      /* cfg `workspace`: min_x max_x min_y max_y min_z max_z, strict inequalities   */
  double voxel_size;        /* cfg `voxel_size`; Cloud::voxelizeCloud(float cell_size) rounds it to float  */
  double normals_radius;    /* cfg `normals_radius`                                                        */
  int32_t voxelize;         /* cfg `voxelize`                                                              */
  int32_t estimate_normals; /* 1: Cloud::calculateNormalsOMP + reverseNormals (cloud.cpp:497-535,573-604); */
                            /* 0: keep the caller's normals (voxel-averaged, cloud.cpp:307-311,331-333)    */
} gpdb_preprocess_params;

/* Reference defaults: workspace -1..1, voxelize, voxel_size 0.003, normals_radius 0.03, estimate normals. */
void gpdb_preprocess_params_default(gpdb_preprocess_params *p);

/* Replaces: CandidatesGenerator::preprocessPointCloud steps removeNans -> filterWorkspace -> voxelizeCloud ->
 * calculateNormals (candidates_generator.cpp:18-26; cloud.cpp:154-164,207-266,286-348,458-484,497-535,573-604)
 * on the device, and installs the processed cloud in the context exactly as gpdb_set_cloud would (the neighbour
 * grid is built from the device copy). Inputs as gpdb_set_cloud (raw cloud, n_points may be millions); `normals`
 * may be NULL when estimate_normals = 1. Returns the number of processed points N' (>= 0) or a negative error.
 * A camera sees a point when its cam_source entry is exactly 1, as in the reference's voxelisation and normal
 * estimation (cloud.cpp:327,581,611); with voxelize = 0 any entry other than 0 or 1 is GPDB_ERR_INVALID (the
 * reference would keep it raw and read it as == 1 for the normals but >= 1 in the grasp path). More than 8 192
 * neighbours within normals_radius at one point is GPDB_ERR_CAPACITY; a voxel index of 2^21 or more on any axis
 * (cloud extent / voxel_size) is GPDB_ERR_INVALID. After either error, or a rejected cam_source, the context holds
 * no cloud until the next successful gpdb_set_cloud / gpdb_preprocess.
 * Not covered: remove_outliers, refine_normals_k and sample_above_plane (separate steps: gpdb_remove_outliers, which the
 * reference's preprocessing never runs although its cfg parses the key, gpdb_refine_normals, then gpdb_segment_plane) and
 * Cloud::subsample (host-side RNG; the sample indices are an input of gpdb_detect; a batch draws them on the device with
 * gpdb_subsample_clouds).
 * Semantics that differ from the reference by specification (DESIGN.md "preprocessing"): the voxel set is an
 * exact set (the reference's std::set comparator is not a strict weak order), output order = descending index
 * of each voxel's first point (the reference's iteration order whenever its de-duplication succeeds). */
int gpdb_preprocess(gpdb_ctx *ctx, const float *xyz, const double *normals, const int32_t *cam_source,
                    int32_t n_points, const double *view_points, int32_t n_cams,
                    const gpdb_preprocess_params *pp);

/* Reads back the cloud currently installed in the context (after gpdb_preprocess or gpdb_set_cloud):
 * xyz_out [3*N] float32, normals_out [3*N] float64 (3 x N column-major), cam_source_out [k*N] int32 (k x N
 * column-major); any output may be NULL. Returns N. These are the util::Cloud members the reference's
 * preprocessing leaves behind (cloud_processed_, normals_, camera_source_; cloud.h:300-333). */
int gpdb_get_cloud(gpdb_ctx *ctx, float *xyz_out, double *normals_out, int32_t *cam_source_out);

/* After gpdb_preprocess: src_out [N] = index into the RAW cloud of the point that represents each processed point
 * (the first point of its voxel, cloud.cpp:304-310 `(*res.first)(3)`). Returns N. */
int gpdb_get_cloud_source_index(gpdb_ctx *ctx, int32_t *src_out);

/* CandidatesGenerator::preprocessPointCloud for every cloud of a batch in ONE call (the gpdb_preprocess steps, each cloud
 * on its own), leaving the processed clouds installed as the batch, exactly as gpdb_set_clouds would install them.
 * Raw cloud b: points point_offsets[b] .. point_offsets[b+1]-1 of xyz (normals likewise, may be NULL when
 * estimate_normals = 1), n_cameras[b] cameras, view points and cam_source blocks as gpdb_set_clouds (cam_source NULL:
 * every camera sees every point). One gpdb_preprocess_params for all clouds. processed_offsets_out[B+1] receives the
 * processed point offsets. Returns B or a negative error; a failed call leaves no batch, the single cloud is never touched.
 * Every processed cloud is bit-equal to gpdb_preprocess on that raw cloud alone (points, camera sources, source indices,
 * normals). Camera sources follow gpdb_preprocess: an entry counts as seen when it is exactly 1, and with voxelize = 0
 * an entry other than 0 or 1 is GPDB_ERR_INVALID. A raw cloud must hold at least one point; a cloud the filter empties
 * stays in the batch with no points (equal processed offsets: it takes only an empty sample range in
 * gpdb_detect_batch). Malformed offsets, K_b outside 1..8, missing normals with estimate_normals = 0 and a
 * non-positive voxel_size or normals_radius are GPDB_ERR_INVALID before any device work; a voxel index of 2^21 or more
 * in any cloud is GPDB_ERR_INVALID (the message names the cloud); more than 8 192 neighbours within normals_radius at
 * one point is GPDB_ERR_CAPACITY. */
int gpdb_preprocess_clouds(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *point_offsets, const float *xyz,
                           const double *normals, const int32_t *cam_source, const int32_t *n_cameras,
                           const double *view_points, const gpdb_preprocess_params *pp, int32_t *processed_offsets_out);

/* Reads back the installed batch (after gpdb_preprocess_clouds or gpdb_set_clouds), concatenated in cloud order:
 * xyz_out [3*N], normals_out [3*N], cam_source_out (the N_b x K_b int32 blocks one after the other), src_out [N] =
 * index into cloud b's RAW points of the point that represents each processed point (gpdb_preprocess_clouds only;
 * GPDB_ERR_STATE after gpdb_set_clouds). Any output may be NULL. Returns N; GPDB_ERR_STATE when no batch is installed. */
int gpdb_get_clouds(gpdb_ctx *ctx, float *xyz_out, double *normals_out, int32_t *cam_source_out, int32_t *src_out);

/* Device time (ms, CUDA events) of the stages of the last gpdb_preprocess or gpdb_preprocess_clouds call (for a batch:
 * all clouds together): ms[0] upload, ms[1] NaN/workspace filter, ms[2] voxelise, ms[3] grid build, ms[4] normals,
 * ms[5] whole call. */
int gpdb_preprocess_timings(const gpdb_ctx *ctx, double ms_out[6]);

/* Replaces: HandSearch::reevaluateHypotheses (hand_search.cpp:66-134; GraspDetector::evalGroundTruth,
 * grasp_detector.cpp:523-527): the given hands (sample, frame, top, finger_idx are read) are re-labelled against the cloud
 * installed in the context — radius search around the hand's sample, its own frame, evaluateFingers at its own depth and
 * finger placement, closing region, Antipodal::evaluateGrasp. labels_out[i] = 1 for a full antipodal grasp, else 0; the
 * half_antipodal / full_antipodal fields of the records are updated in place. Returns n. */
int gpdb_reevaluate(gpdb_ctx *ctx, gpdb_pose *hands, int32_t n_hands, int32_t *labels_out);

/* HandSearch::reevaluateHypotheses for every cloud of the installed batch in one call: group b, hands[hand_offsets[b] ..
 * hand_offsets[b+1]), is re-labelled against cloud b (hand_offsets: B + 1 host entries starting at 0, never decreasing;
 * an empty group is allowed). Fields read and written as gpdb_reevaluate; group b's records and labels are bit-equal to
 * gpdb_reevaluate on those hands with cloud b installed alone. The hands may come from anywhere, e.g. the candidates of
 * camera views detected in another context, labelled here against ground-truth clouds installed once. The call only
 * reads the store: the batch, its sample positions and the SIS record are unchanged. Returns hand_offsets[B];
 * GPDB_ERR_STATE when no batch is installed; malformed offsets or NULL arrays for a non-empty call are GPDB_ERR_INVALID
 * before any device work, with the outputs untouched. */
int gpdb_reevaluate_batch(gpdb_ctx *ctx, const int32_t *hand_offsets, gpdb_pose *hands, int32_t *labels_out);

/* Replaces: Clustering::findClusters(hand_list, remove_inliers = false) (clustering.cpp:5-105; GraspDetector::detectGrasps
 * step 6, grasp_detector.cpp:283-301; SequentialImportanceSampling step 4) on the device: one warp per hand over the n
 * hands (n <= num_selected in detectGrasps), inliers folded in index order so that the running mean / variance are the
 * reference's. hands [n] are host records (score, position, frame read); clusters_out has room for n records and receives
 * the clusters in the order of their seed hands (position = mean inlier position, score = lower 99 % confidence bound).
 * Returns the number of clusters. */
int gpdb_find_clusters(gpdb_ctx *ctx, const gpdb_pose *hands, int32_t n_hands, int32_t min_inliers, gpdb_pose *clusters_out);

/* gpdb_find_clusters on each of n_groups groups of hands independently, in one call (step 6 of detectGrasps over a batch
 * of clouds): group g is hands[hand_offsets[g] .. hand_offsets[g+1]) (hand_offsets: n_groups + 1 entries starting at 0,
 * never decreasing; an empty group is allowed). Group g's clusters are clusters_out[cluster_offsets_out[g] ..
 * cluster_offsets_out[g+1]) (cluster_offsets_out: n_groups + 1 entries), in seed-hand order, bit-equal to
 * gpdb_find_clusters on that group alone; clusters_out has room for hand_offsets[n_groups] records. Needs no cloud.
 * Returns the number of clusters of all groups. */
int gpdb_find_clusters_batch(gpdb_ctx *ctx, int32_t n_groups, const int32_t *hand_offsets, const gpdb_pose *hands,
                             int32_t min_inliers, gpdb_pose *clusters_out, int32_t *cluster_offsets_out);

/* --- device-resident batches: clouds, samples and results that live in GPU memory ------------------------------------
 * The batch calls above from device memory, with no bulk PCIe traffic: preprocess (or install), detect + select and
 * cluster a batch whose arrays a framework produced on the GPU (simulated depth cameras, device depth-to-cloud); install
 * sample positions a model drew on the GPU, return every hand with its pose flags and scores, and make and classify
 * grasp images for a classifier of the caller's.
 * Sizes and offsets stay on the host (B, point / sample / hand offsets, n_cameras, view_points, the preprocessing
 * parameters; the library sizes its launches from them). Arguments named d_* are device pointers on the context's device:
 * any non-NULL d_* argument that cudaPointerGetAttributes does not report as device or managed memory of that device is
 * GPDB_ERR_INVALID, before any device work. The library reads and writes them in order on the context's stream
 * (gpdb_set_stream: e.g. the framework's current stream, so that inputs made ready on it need no synchronisation) and, as
 * every entry point, returns once its outputs are complete: they may then be used on any stream.
 * Each call has the semantics, error codes, messages and failure rules of its host twin (a failed install leaves no batch,
 * the single cloud is never touched); its checks are the host twin's, on the device (non-finite coordinates, cam_source
 * entries, sample indices), and report the first offending point / entry / position. */

/* gpdb_preprocess_clouds from device arrays: d_xyz [3M] float32, d_normals [3M] float64 or NULL, d_cam_source (the
 * N_b x K_b int32 blocks) or NULL; the raw arrays are read in place and the camera masks packed on the device. */
int gpdb_preprocess_clouds_device(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *point_offsets, const float *d_xyz,
                                  const double *d_normals, const int32_t *d_cam_source, const int32_t *n_cameras,
                                  const double *view_points, const gpdb_preprocess_params *pp,
                                  int32_t *processed_offsets_out);

/* gpdb_set_clouds from device arrays (d_xyz [3N], d_normals [3N], d_cam_source or NULL): copied device to device into
 * the batch; the finiteness check and the camera masks run on the device. Returns B. */
int gpdb_set_clouds_device(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *point_offsets, const float *d_xyz,
                           const double *d_normals, const int32_t *d_cam_source, const int32_t *n_cameras,
                           const double *view_points);

/* gpdb_detect_batch_select with device sample indices (d_sample_idx [sample_offsets[B]], cloud-local, checked on the
 * device) and a device result: d_selected_out has room for B * num_selected records and receives them exactly as
 * gpdb_detect_batch_select returns them (cloud-local sample_slot; cloud b's at sel_offsets_out[b] ..
 * sel_offsets_out[b+1]); sel_offsets_out [B + 1] is a host array. stats receives the counts (n_candidates = records
 * written, n_total_candidates), the stage timings and the launch count; its array members stay NULL and it needs no
 * gpdb_free_result. Returns the number of records. */
int gpdb_detect_batch_select_device(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *d_sample_idx,
                                    int32_t num_selected, gpdb_pose *d_selected_out, int32_t *sel_offsets_out,
                                    gpdb_result *stats);

/* gpdb_find_clusters_batch with device hands (d_hands [hand_offsets[G]]) and clusters (d_clusters_out, room for
 * hand_offsets[G] records); hand_offsets and cluster_offsets_out [G + 1] are host arrays. */
int gpdb_find_clusters_batch_device(gpdb_ctx *ctx, int32_t n_groups, const int32_t *hand_offsets, const gpdb_pose *d_hands,
                                    int32_t min_inliers, gpdb_pose *d_clusters_out, int32_t *cluster_offsets_out);

/* gpdb_set_clouds_samples with the positions in device memory: d_samples_xyz (3 x M float64, column-major, M =
 * pos_offsets[B]) is copied device to device into the batch's sample arena. Same rules: the values are not checked, each
 * call replaces all positions, a failed call and any new batch leave none, GPDB_ERR_STATE without a batch. Returns M. */
int gpdb_set_clouds_samples_device(gpdb_ctx *ctx, const int32_t *pos_offsets, const double *d_samples_xyz);

/* gpdb_hand_search_batch with device sample indices (d_sample_idx [n = sample_offsets[B]], checked on the device) and
 * device results: d_hands_out has room for n * P records and receives every VALID|FILTERED record exactly as
 * gpdb_hand_search_batch returns them (grouped by cloud, cloud-local sample_slot; cloud b's at cand_offsets_out[b] ..
 * cand_offsets_out[b+1], a host array of B + 1 entries); d_flags_out [n * P] receives the pose flags (may be NULL).
 * stats receives the counts, timings and launch count; its array members stay NULL. Needs no weights. Returns the number
 * of records. */
int gpdb_hand_search_batch_device(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *d_sample_idx,
                                  uint8_t *d_flags_out, gpdb_pose *d_hands_out, int32_t *cand_offsets_out, gpdb_result *stats);

/* gpdb_detect_batch the same way: d_candidates_out (room for n * P records) receives the scored records as
 * gpdb_detect_batch returns them, d_flags_out / d_scores_out [n * P] the pose flags and scores (NaN where no image was
 * classified; either may be NULL). No images: size d_images_out of gpdb_images_batch_device from cand_offsets_out. */
int gpdb_detect_batch_device(gpdb_ctx *ctx, const int32_t *sample_offsets, const int32_t *d_sample_idx, uint8_t *d_flags_out,
                             float *d_scores_out, gpdb_pose *d_candidates_out, int32_t *cand_offsets_out, gpdb_result *stats);

/* ImageGenerator::createImages (gpdb_images) for given hands of the installed batch: group b, d_hands[hand_offsets[b] ..
 * hand_offsets[b+1]), belongs to cloud b (hand_offsets: B + 1 host entries starting at 0, never decreasing). d_images_out
 * receives hand_offsets[B] images of S*S*C bytes, HWC uint8 (the cv::Mat layout of gpdb_images), byte-identical to
 * gpdb_detect_batch with keep_images = 1 for the same records. The records' sample_slot is ignored; sample_index seeds the
 * shadow draws. Returns the number of images. */
int gpdb_images_batch_device(gpdb_ctx *ctx, const int32_t *hand_offsets, const gpdb_pose *d_hands, uint8_t *d_images_out);

/* gpdb_classify on n images in device memory (d_images_hwc [n * S*S*C], HWC uint8): d_scores_out [n] and d_logits_out
 * [n * 2] (may be NULL) are written by the classifier directly. Bit-equal to gpdb_classify, for both lenet_impl values. */
int gpdb_classify_device(gpdb_ctx *ctx, const uint8_t *d_images_hwc, int32_t n, float *d_scores_out, float *d_logits_out);

/* gpdb_reevaluate_batch on device records: d_hands [hand_offsets[B]] are re-labelled in place and d_labels_out
 * [hand_offsets[B]] receives the labels, bit-equal to the host twin. With images_batch_device this keeps the images and
 * the labels of many views on the GPU (training data, INTEGRATION.md). */
int gpdb_reevaluate_batch_device(gpdb_ctx *ctx, const int32_t *hand_offsets, gpdb_pose *d_hands, int32_t *d_labels_out);

/* --- sequential importance sampling: SequentialImportanceSampling::detectGrasps on the device ----------------------------
 * (sequential_importance_sampling.cpp:54-270) over every cloud of the installed batch (gpdb_set_clouds[_device] /
 * gpdb_preprocess_clouds[_device]; a single cloud is a batch of one) in ONE call: the initial hand search, every round's
 * draws (include/gpd_b200_sis.h), hand search and kept-set bookkeeping, the final classification at all kept positions, the
 * score filter and the clustering run on the device; a round reads back B counts. Field names are the reference's SIS cfg
 * keys (:19-31). */
typedef struct gpdb_sis_params {
  int32_t num_iterations;            /* rounds (5)                                                            */
  int32_t num_samples_per_iteration; /* positions drawn per round and cloud (50)                              */
  double prob_rand_samples;          /* share of uniform positions (0.3): num_rand = (int)(prob * S)          */
  double standard_deviation;         /* sigma of the Gaussian proposals (0.02)                                */
  int32_t sampling_method;           /* 0 sum of Gaussians, 1 max of Gaussians (rejection)                    */
  double workspace[6];               /* uniform positions: inclusive bounds min_x max_x min_y max_y min_z max_z */
  double min_score;                  /* keep hands with score > min_score (pruneGraspCandidates)              */
  int32_t min_inliers;               /* > 0: return the clusters (findClusters); 0: the kept hands            */
  uint64_t seed;                     /* cloud b draws with key seed + b                                       */
} gpdb_sis_params;

/* The reference defaults above, workspace -1..1, min_score 0, min_inliers 1, seed 0. */
void gpdb_sis_params_default(gpdb_sis_params *p);

/* init_idx: cloud-local point indices in CSR form (cloud b: init_idx[init_offsets[b] .. init_offsets[b+1]), B + 1
 * offsets), drawn by the caller (Cloud::subsample). A cloud whose initial search finds no hand is inactive: no rounds, no
 * output. The result holds per cloud the hands with score > min_score at the kept positions, in the order
 * gpdb_detect_batch returns them there (cloud-local sample slots), or their clusters in seed order when min_inliers > 0;
 * cloud b's records are out->candidates[hand_offsets_out[b] .. hand_offsets_out[b+1]). The per-sample arrays are NULL,
 * n_samples counts the kept positions and n_total_candidates the classified candidates. Afterwards the batch holds the
 * kept positions as gpdb_set_clouds_samples would install them; a failed call leaves none, the single cloud is never
 * touched. Needs weights (GPDB_ERR_STATE). Negative counts, prob_rand_samples outside [0, 1], a sigma that is not finite
 * and positive, a sampling_method other than 0 / 1, malformed offsets and an init index outside its cloud are
 * GPDB_ERR_INVALID before any device work. Returns the number of records. */
int gpdb_sis_batch(gpdb_ctx *ctx, const gpdb_sis_params *sp, const int32_t *init_offsets, const int32_t *init_idx,
                   gpdb_result *out, int32_t *hand_offsets_out);
/* The same from device memory (the rules of the device-resident family above): d_init_idx is checked on the device,
 * d_hands_out has room for (init_offsets[B] + B * num_iterations * num_samples_per_iteration) * P records and receives
 * them; stats receives the counts, timings and launches, its array members stay NULL. Bit-equal to gpdb_sis_batch. */
int gpdb_sis_batch_device(gpdb_ctx *ctx, const gpdb_sis_params *sp, const int32_t *init_offsets, const int32_t *d_init_idx,
                          gpdb_pose *d_hands_out, int32_t *hand_offsets_out, gpdb_result *stats);
/* What the last successful SIS call evaluated and kept (host arrays, any may be NULL): eval_offsets_out [B+1] and
 * eval_xyz_out [3 x total] the positions of every round, per cloud in round order, eval_round_counts_out [B * iterations]
 * (cloud-major) the positions of each round (fewer than drawn when a proposal loop ran out); kept_offsets_out [B+1] and
 * kept_xyz_out the positions of every sample that carried a VALID|FILTERED pose, the initial samples first, then the
 * rounds, in sample order. The arrays are sized by the batch of that call. Returns B; GPDB_ERR_STATE when none ran, the
 * last one failed, or a batch was installed since (gpdb_set_clouds[_device], gpdb_preprocess_clouds[_device]). */
int gpdb_sis_positions(gpdb_ctx *ctx, int32_t *eval_offsets_out, int32_t *eval_round_counts_out, double *eval_xyz_out,
                       int32_t *kept_offsets_out, double *kept_xyz_out);

/* --- depth images and Cloud::subsample on the device (include/gpd_b200_depth.h) -----------------------------------------
 * The two steps in front of and behind preprocessing that a depth-camera or simulator user would otherwise write: depth
 * images -> gpdb_preprocess_depth[_device] -> gpdb_subsample_clouds[_device] -> gpdb_detect_batch_select[_device] ->
 * gpdb_find_clusters_batch[_device], without leaving the GPU. The camera struct, the arithmetic, the raw-cloud numbering
 * and the sampling rule are specified in gpd_b200_depth.h. */
typedef struct gpdb_depth_camera gpdb_depth_camera;

/* gpdb_preprocess_clouds of n_views views given as depth images: view b has n_cameras[b] cameras (1..8); cameras holds
 * the sum of n_cameras host descriptions, view by view, and depth every camera's image back to back in the same order,
 * all of one format (GPDB_DEPTH_U16 / GPDB_DEPTH_F32). View b's raw cloud is the concatenation of its cameras' pixels
 * (gpd_b200_depth.h 3), and the call installs exactly what gpdb_preprocess_clouds installs from it (processed offsets
 * to processed_offsets_out [B+1]; gpdb_get_clouds' src_out = pixel index into the view's concatenated images). The raw
 * cloud is never built: back-projection runs inside the NaN / workspace filter. Failure rules of gpdb_preprocess_clouds
 * (a failed call leaves no batch, drops the SIS record and the sample positions, never touches the single cloud). These
 * are GPDB_ERR_INVALID before any device work, the message naming the view and camera: K_b outside 1..8, a width or
 * height < 1, non-finite intrinsics or pose, fx or fy <= 0, depth_scale <= 0, min_depth < 0, max_depth <= min_depth, an
 * unknown format, estimate_normals = 0, 2^31 or more pixels in the call, and the gpdb_preprocess_clouds parameter
 * checks. The rotation of a pose is not checked for orthonormality. Returns B. */
int gpdb_preprocess_depth(gpdb_ctx *ctx, int32_t n_views, const int32_t *n_cameras, const gpdb_depth_camera *cameras,
                          int32_t depth_format, const void *depth, const gpdb_preprocess_params *pp,
                          int32_t *processed_offsets_out);
/* The same with the images in device memory (d_depth on the context's device, read in place on the context's stream). */
int gpdb_preprocess_depth_device(gpdb_ctx *ctx, int32_t n_views, const int32_t *n_cameras, const gpdb_depth_camera *cameras,
                                 int32_t depth_format, const void *d_depth, const gpdb_preprocess_params *pp,
                                 int32_t *processed_offsets_out);

/* --- organized clouds: Cloud::calculateNormalsOrganized on the device (include/gpd_b200_organized.h) ------------------
 * pcl::IntegralImageNormalEstimation (COVARIANCE_MATRIX, smoothing size 20, PCL's defaults otherwise), the method the
 * reference's calculateNormals picks for an organized cloud: each normal comes from a pixel window of at most 20 x 20
 * that shrinks towards depth discontinuities, so it does not smooth across object silhouettes, and its cost per pixel
 * does not depend on how many neighbours a point has. The reference's preprocessing never reaches it (its workspace
 * filter makes the cloud unorganized), so it is a call of its own. */

/* Normals of n_clouds organized clouds by the rules of gpd_b200_organized.h: cloud b is heights[b] x widths[b] float32
 * points, row-major, NaN coordinates for a missing point, with view point view_points[3b .. 3b+2] (float32, host);
 * the clouds lie back to back in xyz. normals_out [3 * points] receives the float32 normals (NaN where rule 5 gives none:
 * the 20-pixel border, non-finite depth, a distance map value <= 2), distance_out [points] (may be NULL) the rule-3
 * distance map. Nothing installed changes. GPDB_ERR_INVALID before any device work: n_clouds <= 0, a null array, a
 * width or height < 1, 2^31 or more points in the call. Returns n_clouds. */
int gpdb_normals_organized(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *widths, const int32_t *heights, const float *xyz,
                           const float *view_points, float *normals_out, float *distance_out);
/* The same with xyz and the outputs in device memory (widths, heights and view_points stay host arrays). */
int gpdb_normals_organized_device(gpdb_ctx *ctx, int32_t n_clouds, const int32_t *widths, const int32_t *heights,
                                  const float *d_xyz, const float *view_points, float *d_normals_out,
                                  float *d_distance_out);
/* gpdb_preprocess_depth with the normals of gpd_b200_organized.h rule 7: a processed point whose representative pixel
 * (gpdb_get_clouds' src) has a finite integral-image normal in its camera's image (camera frame, rotated to the world by
 * the pose's R) takes it, with reverseNormals applied; every other point (a fallback: the image border, silhouettes,
 * holes) keeps exactly the radius estimate gpdb_preprocess_depth gives it, so estimate_normals must be nonzero and
 * normals_radius > 0. Points, camera sources, source indices and offsets are those of gpdb_preprocess_depth bit for bit,
 * and so are the failure rules. n_fallback_out [B] (may be NULL) receives each view's fallback points.
 * gpdb_preprocess_timings' ms[4] covers both normal methods. Returns B. */
int gpdb_preprocess_depth_organized(gpdb_ctx *ctx, int32_t n_views, const int32_t *n_cameras,
                                    const gpdb_depth_camera *cameras, int32_t depth_format, const void *depth,
                                    const gpdb_preprocess_params *pp, int32_t *processed_offsets_out,
                                    int32_t *n_fallback_out);
/* The same with the images in device memory. */
int gpdb_preprocess_depth_organized_device(gpdb_ctx *ctx, int32_t n_views, const int32_t *n_cameras,
                                           const gpdb_depth_camera *cameras, int32_t depth_format, const void *d_depth,
                                           const gpdb_preprocess_params *pp, int32_t *processed_offsets_out,
                                           int32_t *n_fallback_out);

/* Replaces: Cloud::subsample (cloud.cpp:350-370) for every cloud of the installed batch, by the rule of gpd_b200_depth.h
 * 5: cloud b draws min(num_samples, eligible points) cloud-local point indices without replacement, in ascending order
 * (num_samples = 0: every eligible point). mask (may be NULL) holds one byte per raw point of the preprocessing call that
 * installed the batch (gpdb_preprocess_clouds[_device] / gpdb_preprocess_depth[_device]), concatenated by view; a point
 * is eligible when the byte of its source raw point is nonzero. sample_idx_out has room for sum over b of min(num_samples,
 * N_b) entries (N_b when num_samples = 0) and receives cloud b's draw at sample_offsets_out[b] .. sample_offsets_out[b+1]
 * (B + 1 host entries): the CSR lists gpdb_detect_batch[_select][_device], gpdb_hand_search_batch[_device] and
 * gpdb_sis_batch[_device] take. The batch is not changed. No batch, or a mask after gpdb_set_clouds[_device] (no source
 * indices), is GPDB_ERR_STATE; a negative num_samples is GPDB_ERR_INVALID. Returns the number of indices. */
int gpdb_subsample_clouds(gpdb_ctx *ctx, int32_t num_samples, uint64_t seed, const uint8_t *mask, int32_t *sample_idx_out,
                          int32_t *sample_offsets_out);
/* The same with the mask and the indices in device memory (sample_offsets_out stays a host array). */
int gpdb_subsample_clouds_device(gpdb_ctx *ctx, int32_t num_samples, uint64_t seed, const uint8_t *d_mask,
                                 int32_t *d_sample_idx_out, int32_t *sample_offsets_out);

/* --- the support plane: Cloud::sampleAbovePlane on the device (include/gpd_b200_plane.h) --------------------------------
 * pcl::SACSegmentation's RANSAC plane fit with refit (cloud.cpp:407-435), restated with counter-based draws: fit the
 * table plane of each installed cloud and mark the points off it, so that samples land on the objects. The recipe of a
 * tabletop view: gpdb_preprocess_depth[_device] -> gpdb_segment_planes[_device] -> gpdb_subsample_clouds_points[_device]
 * (the eligible bytes as the mask) -> gpdb_detect_batch_select[_device]. */
typedef struct gpdb_plane_params {
  double distance_threshold; /* inlier iff the point's distance is < this (0.01, cloud.cpp:418)                     */
  int32_t max_iterations;    /* at most max_iterations + 1 hypotheses (50, SACSegmentation's default), 1..1024    */
  double probability;        /* RANSAC's stop probability (0.99), in (0, 1)                                      */
  uint64_t seed;             /* cloud b draws with key seed + b (the single cloud: seed)                         */
} gpdb_plane_params;

/* The values above. */
void gpdb_plane_params_default(gpdb_plane_params *p);

/* Segments the single installed cloud (gpdb_set_cloud / gpdb_preprocess) by the rules of gpd_b200_plane.h: plane_out[4]
 * = (a, b, c, d) with ax + by + cz + d = 0 (all NaN when the fit failed: fewer than 3 points or no good sample),
 * *n_inliers_out = the points within distance_threshold of it (0 when the fit failed), eligible_out [N] (may be NULL) = 1
 * for every point off the plane, and 1 for every point when the fit failed or no point is off the plane. Nothing
 * installed changes. No cloud is GPDB_ERR_STATE; a threshold that is not finite and positive, max_iterations outside
 * 1..1024 and probability outside (0, 1) are GPDB_ERR_INVALID before any device work. Equal to gpdb_segment_planes on a
 * batch of one. Returns 1. */
int gpdb_segment_plane(gpdb_ctx *ctx, const gpdb_plane_params *pl, float plane_out[4], int32_t *n_inliers_out,
                       uint8_t *eligible_out);
/* The same for every cloud of the installed batch (cloud b with key seed + b; its result depends on nothing else):
 * planes_out [4B], n_inliers_out [B], n_hypotheses_out [B] (may be NULL) = RANSAC hypotheses evaluated, eligible_out [N]
 * (may be NULL, concatenated by cloud). No batch is GPDB_ERR_STATE. Nothing installed changes: the clouds, sample
 * positions and SIS record stay. Returns B. */
int gpdb_segment_planes(gpdb_ctx *ctx, const gpdb_plane_params *pl, float *planes_out, int32_t *n_inliers_out,
                        int32_t *n_hypotheses_out, uint8_t *eligible_out);
/* The same with d_eligible_out in device memory (the rules of the device-resident family); planes and counts stay host
 * arrays. */
int gpdb_segment_planes_device(gpdb_ctx *ctx, const gpdb_plane_params *pl, float *planes_out, int32_t *n_inliers_out,
                               int32_t *n_hypotheses_out, uint8_t *d_eligible_out);

/* --- the normal refinement: Cloud::refineNormals on the device (include/gpd_b200_refine.h) -----------------------------
 * refine_normals_k > 0 (candidates_generator.cpp:28-30): every normal becomes the normalised sum of the normals of its
 * point's k nearest neighbours, repeated until the mean change is small (pcl::NormalRefinement's defaults), so that noisy
 * normals, those of depth images in particular, are smoothed before the local frames, the antipodal test and the
 * normals channels of the images read them. The reference runs it between calculateNormals and sampleAbovePlane: e.g.
 * gpdb_preprocess_depth[_device] -> gpdb_refine_normals_clouds -> gpdb_segment_planes[_device] -> ... */

/* Refines the normals of the single installed cloud (any install: gpdb_set_cloud, gpdb_preprocess) in place by the
 * rules of gpd_b200_refine.h with k nearest neighbours (the point itself included; every point when the cloud has fewer
 * than k). *iterations_out (may be NULL) = iterations run (1..15; 0 for an empty cloud). gpdb_get_cloud reads the
 * refined normals back; the store's other content derived from the normals (the per-cloud flag of normals not of unit
 * length, which decides how the image stage folds a cell) is recomputed by the rule every install applies, so a refined
 * cloud behaves as one installed with the refined normals. The call is not an install: sample positions stay, and the
 * batch is untouched. k outside 1..128 (GPDB_REFINE_MAX_K: the neighbour lists take N * k int32 of device memory) is
 * GPDB_ERR_INVALID, no cloud GPDB_ERR_STATE; after any error the stored normals are unchanged. Returns 1. */
int gpdb_refine_normals(gpdb_ctx *ctx, int32_t k, int32_t *iterations_out);
/* The same for every cloud of the installed batch (any install: gpdb_set_clouds[_device], gpdb_preprocess_clouds[_device],
 * gpdb_preprocess_depth[_device]), each cloud on its own: its own neighbour lists, stop decision and iteration count,
 * iterations_out [B] (may be NULL). Sample positions and the SIS record stay; the single cloud is untouched. No batch is
 * GPDB_ERR_STATE. Returns B. */
int gpdb_refine_normals_clouds(gpdb_ctx *ctx, int32_t k, int32_t *iterations_out);

/* --- the statistical outlier removal: Cloud::removeStatisticalOutliers on the device (include/gpd_b200_outliers.h) ------
 * Removes the points whose mean distance to their mean_k nearest neighbours lies more than stddev_mul standard
 * deviations above the cloud's mean of that distance (pcl::StatisticalOutlierRemoval; the reference's
 * removeStatisticalOutliers uses mean_k = 50, stddev_mul = 1.0). Depth images are where such points come from: flying
 * pixels at depth edges and isolated speckle, each a sample that finds no grasp, a point in the fingers' way and occupied
 * cells in the grasp images. E.g. gpdb_preprocess_depth[_device] -> gpdb_remove_outliers_clouds ->
 * gpdb_refine_normals_clouds -> gpdb_segment_planes[_device] -> ...
 *
 * The call is an install of the kept points: they keep their order, normals, camera masks and (after a preprocessing
 * install) source indices, which still index the raw points, so per-pixel masks keep working; the grids, the nonunit
 * flags and the flag of clouds whose every point every camera sees are recomputed as gpdb_set_clouds computes them, so
 * the store behaves as one installed with the kept points. Sample positions are dropped. mean_k outside 1..127
 * (GPDB_OUTLIERS_MAX_K) or a non-finite stddev_mul is GPDB_ERR_INVALID and no cloud GPDB_ERR_STATE; these errors change
 * nothing. Any other error (a CUDA error, e.g. no device memory for the neighbour lists) leaves no cloud (the batch
 * call: no batch, no sample positions, no SIS record), as a failed install does. A cloud of at most mean_k points keeps
 * every point and reports NaN statistics (gpd_b200_outliers.h rule 5). */

/* The single installed cloud (any install: gpdb_set_cloud, gpdb_preprocess); the batch is untouched. stats_out (may be
 * NULL) = {mean, stddev, threshold}; kept_out (may be NULL) one byte per point before the call, 1 = kept. Returns the
 * number of kept points; when none is kept the context holds no cloud, as after gpdb_preprocess keeping none. */
int gpdb_remove_outliers(gpdb_ctx *ctx, int32_t mean_k, double stddev_mul, double stats_out[3], uint8_t *kept_out);
/* Every cloud of the installed batch (any install: gpdb_set_clouds[_device], gpdb_preprocess_clouds[_device],
 * gpdb_preprocess_depth[_device]), each on its own; the single cloud is untouched. offsets_out [B+1] (may be NULL) = the
 * new point offsets, stats_out [3B] (may be NULL) each cloud's {mean, stddev, threshold}, kept_out [N before] (may be
 * NULL) the kept bytes. The SIS record is dropped (gpdb_sis_positions is then GPDB_ERR_STATE). No batch is GPDB_ERR_STATE.
 * Returns B. */
int gpdb_remove_outliers_clouds(gpdb_ctx *ctx, int32_t mean_k, double stddev_mul, int32_t *offsets_out,
                                double *stats_out, uint8_t *kept_out);

/* gpdb_subsample_clouds with the mask over the INSTALLED points: point_mask [N] (may be NULL) holds one byte per point of
 * the batch, concatenated by cloud (the eligible bytes of gpdb_segment_planes), so it also works after
 * gpdb_set_clouds[_device]. The draw rule is gpd_b200_depth.h 5 unchanged; point_mask = NULL equals gpdb_subsample_clouds
 * with mask = NULL bit for bit. */
int gpdb_subsample_clouds_points(gpdb_ctx *ctx, int32_t num_samples, uint64_t seed, const uint8_t *point_mask,
                                 int32_t *sample_idx_out, int32_t *sample_offsets_out);
/* The same with the mask and the indices in device memory (sample_offsets_out stays a host array). */
int gpdb_subsample_clouds_points_device(gpdb_ctx *ctx, int32_t num_samples, uint64_t seed, const uint8_t *d_point_mask,
                                        int32_t *d_sample_idx_out, int32_t *sample_offsets_out);

/* --- training views from triangle meshes (include/gpd_b200_render.h) ----------------------------------------------------
 * Depth images of mesh scenes in the layout gpdb_preprocess_depth[_device] consumes, and dense ground-truth clouds sampled
 * from the same surfaces for gpdb_reevaluate_batch[_device]: meshes -> views -> candidates -> labels -> images -> weights
 * with no dataset on disk. Neither call installs anything: the single cloud, the batch, its sample positions and the SIS
 * record are untouched. The rules are specified in gpd_b200_render.h. */

/* Renders n_views mesh scenes: view b has the float32 xyz vertices vertex_offsets[b] .. vertex_offsets[b+1]-1 of vertices
 * (world frame) and the int32 index triples face_offsets[b] .. face_offsets[b+1]-1 of faces (0-based, into the view's own
 * vertices); it is seen by n_cameras[b] (1..8) cameras, the sum of n_cameras host descriptions in cameras, view by view.
 * depth_out receives every camera's image back to back in the same order (gpd_b200_render.h 5; format GPDB_DEPTH_U16 or
 * GPDB_DEPTH_F32), face_out (may be NULL) one int32 per pixel: the view-local index of the face the pixel's return hit,
 * -1 where it has none. GPDB_ERR_INVALID, the message naming the view, with nothing written: malformed offsets, a face
 * index outside its view's vertices, a non-finite vertex, the camera checks of gpdb_preprocess_depth, an unknown format,
 * 2^31 or more pixels in the call. Returns n_views. */
int gpdb_render_depth(gpdb_ctx *ctx, int32_t n_views, const int32_t *vertex_offsets, const float *vertices,
                      const int32_t *face_offsets, const int32_t *faces, const int32_t *n_cameras,
                      const gpdb_depth_camera *cameras, int32_t depth_format, void *depth_out, int32_t *face_out);
/* The same with vertices, faces and the outputs in device memory (offsets and cameras stay host arrays), on the context's
 * stream. */
int gpdb_render_depth_device(gpdb_ctx *ctx, int32_t n_views, const int32_t *vertex_offsets, const float *d_vertices,
                             const int32_t *face_offsets, const int32_t *d_faces, const int32_t *n_cameras,
                             const gpdb_depth_camera *cameras, int32_t depth_format, void *d_depth_out,
                             int32_t *d_face_out);
/* Samples the surfaces of n_meshes meshes (laid out as the views of gpdb_render_depth) at density points per square metre,
 * mesh b with the key seed + b (gpd_b200_render.h 6). point_offsets_out [B+1] (host) always receives the point offsets;
 * xyz_out = NULL only counts, else xyz_out [3n] receives the float32 points, normals_out [3n] (may be NULL) the float64
 * unit face normals that gpdb_set_clouds[_device] takes, face_out [n] (may be NULL) each point's mesh-local face. The call
 * is deterministic, so a count followed by a fill agrees. GPDB_ERR_INVALID, the message naming the mesh, with nothing
 * written: malformed offsets, a face index outside its mesh's vertices, a non-finite vertex, a density that is not
 * finite and > 0, 2^31 or more points. Returns the number of points n. */
int gpdb_sample_meshes(gpdb_ctx *ctx, int32_t n_meshes, const int32_t *vertex_offsets, const float *vertices,
                       const int32_t *face_offsets, const int32_t *faces, double density, uint64_t seed,
                       int32_t *point_offsets_out, float *xyz_out, double *normals_out, int32_t *face_out);
/* The same with vertices, faces and the point arrays in device memory (the offsets stay host arrays). */
int gpdb_sample_meshes_device(gpdb_ctx *ctx, int32_t n_meshes, const int32_t *vertex_offsets, const float *d_vertices,
                              const int32_t *face_offsets, const int32_t *d_faces, double density, uint64_t seed,
                              int32_t *point_offsets_out, float *d_xyz_out, double *d_normals_out, int32_t *d_face_out);

/* The structured-light sensor model of gpdb_render_sensor_depth[_device] (rules in gpd_b200_sensor.h). Every field 0
 * (gpdb_sensor_params_default) is a clean render. */
typedef struct gpdb_sensor_params {
  double baseline;          /* metres from the camera to the projector along the camera's +x; 0 disables rules 5, 6 */
  double lateral_sigma;     /* pixels: the spread of the pixel each return is read from (rule 3)                  */
  double disparity_sigma;   /* pixels: the spread of the disparity (rule 6)                                       */
  double disparity_step;    /* pixels: the disparity quantum; 0 means no quantisation (rule 6)                    */
  double min_cos_incidence; /* no return below this cosine of the incidence angle; 0 disables rule 4             */
  double shadow_tolerance;  /* relative depth slack of the projector's visibility test (rule 5), < 1             */
  double dropout;           /* the probability in [0, 1] of dropping a return (rule 7)                            */
} gpdb_sensor_params;

/* Every field 0: a clean render. */
void gpdb_sensor_params_default(gpdb_sensor_params *p);

/* gpdb_render_depth's arguments, then the sensor model and the seed: the same images seen as a structured-light sensor
 * sees them (projector shadows, grazing-angle dropouts, quantised disparity noise, lateral jitter, dropout), view b with
 * the key seed + b (gpd_b200_sensor.h). With every sensor field 0 the outputs equal gpdb_render_depth's bit for bit.
 * GPDB_ERR_INVALID, nothing written: gpdb_render_depth's errors, sensor NULL, and the parameter rules of
 * gpd_b200_sensor.h 9. Returns n_views. */
int gpdb_render_sensor_depth(gpdb_ctx *ctx, int32_t n_views, const int32_t *vertex_offsets, const float *vertices,
                             const int32_t *face_offsets, const int32_t *faces, const int32_t *n_cameras,
                             const gpdb_depth_camera *cameras, int32_t depth_format, void *depth_out, int32_t *face_out,
                             const gpdb_sensor_params *sensor, uint64_t seed);
/* The same with vertices, faces and the outputs in device memory (offsets, cameras and the sensor model stay host
 * memory), on the context's stream. */
int gpdb_render_sensor_depth_device(gpdb_ctx *ctx, int32_t n_views, const int32_t *vertex_offsets, const float *d_vertices,
                                    const int32_t *face_offsets, const int32_t *d_faces, const int32_t *n_cameras,
                                    const gpdb_depth_camera *cameras, int32_t depth_format, void *d_depth_out,
                                    int32_t *d_face_out, const gpdb_sensor_params *sensor, uint64_t seed);
/* Development aid: the float64 inverse-normal table of gpd_b200_sensor.h rule 2 (table_out [4097], host), the bytes the
 * device interpolates. Needs no device. Returns 4097. */
int gpdb_debug_sensor_table(double *table_out);

/* Replaces: freeMemoryGrasps (detect_grasps_python.cpp:598-601). The arrays of a result live in page-locked host memory
 * owned by the library (the device writes them directly, overlapped with compute); gpdb_free_result hands that memory
 * back for the next call. A result may outlive its context. */
void gpdb_free_result(gpdb_result *r);

/* --- multi-GPU (SURVEY.md 8(e)): one context per GPU, one process or thread per context ------------------------------
 * The path shards by sample: every rank runs steps 1-4 on the contiguous slice [r*n/R, (r+1)*n/R) of the sample-index
 * array over its own copy of the cloud (reference parallel loops: hand_search.cpp:168-182, image_generator.cpp:83-89,
 * eigen_classifier.cpp:67-76); the only exchange is ONE ncclAllGather of fixed-stride {score f32, flags u8} slots.
 * NCCL is loaded at run time (libnccl.so.2; the copy already in the process, e.g. PyTorch's, is reused). */
#define GPDB_COMM_ID_BYTES 128
/* ncclGetUniqueId: call on one rank, distribute the 128 bytes to the others by any means (MPI, torch.distributed, a pipe). */
int gpdb_comm_unique_id(char id_out[GPDB_COMM_ID_BYTES]);
/* ncclCommInitRank on the context's device and stream (collective: every rank calls it). nranks == 1 is allowed. */
int gpdb_comm_init(gpdb_ctx *ctx, const char id[GPDB_COMM_ID_BYTES], int32_t rank, int32_t nranks);
int gpdb_comm_destroy(gpdb_ctx *ctx);
/* Slice of rank `rank` of `nranks` over n samples and the fixed slot size (largest slice) of the all-gather. */
void gpdb_shard_bounds(int32_t n, int32_t rank, int32_t nranks, int32_t *lo, int32_t *hi, int32_t *slot_samples);
/* gpdb_set_cloud on every rank from rank `root`'s host arrays (ncclBroadcast of the device copies over NVLink; the other
 * ranks pass NULL arrays and any sizes). Every rank then builds its own neighbour grid. Returns N. */
int gpdb_set_cloud_bcast(gpdb_ctx *ctx, int32_t root, const float *xyz, const double *normals, const int32_t *cam_source,
                         int32_t n_points, const double *view_points, int32_t n_cams);
/* gpdb_detect over sharded samples: every rank passes the SAME sample_idx[n]; on return out->pose_flags / out->pose_scores
 * [n*P] hold the gathered results of ALL ranks (identical everywhere), out->candidates the pose records of this rank's
 * slice (sample_slot = position in the full array), out->n_total_candidates the global count; frames / frame_valid
 * are NULL. Returns this rank's candidate count. */
int gpdb_detect_sharded(gpdb_ctx *ctx, const int32_t *sample_idx, int32_t n_samples, gpdb_result *out);
/* Device-resident variant (measurement with inputs in HBM): d_sample_idx_local [n_local] = this rank's slice,
 * d_gathered = nranks slots of gpdb_slot_bytes(slot_samples, P) bytes each: [scores f32 slot_samples*P][flags u8
 * slot_samples*P, padded to 16 B]; this rank's results are written into slot `rank` and all-gathered in place. */
int gpdb_detect_sharded_resident(gpdb_ctx *ctx, const int32_t *d_sample_idx_local, int32_t n_local, int32_t slot_samples,
                                 uint8_t *d_gathered, gpdb_result *stats);
int64_t gpdb_slot_bytes(int32_t slot_samples, int32_t poses_per_sample);

/* --- introspection ------------------------------------------------------------------------- */
/* Device-side stage timings of the last gpdb_detect call, CUDA events on the context stream:
 * ms[0] frames, ms[1] hand search + compaction, ms[2] images, ms[3] LeNet, ms[4] whole call,
 * ms[5] conv1+pool, ms[6] conv2+pool, ms[7] ip1+ip2. */
int gpdb_last_timings(const gpdb_ctx *ctx, double ms_out[8]);
/* Development aid: per-phase SM-cycle counters of the image kernel (thread 0 of every CTA, summed over CTAs).
 * enable != 0 allocates / clears the counters, enable == 0 frees them; cycles_out (may be NULL) receives the
 * counters accumulated so far: [2] ball scan, [3] point channels, [4] shadow setup, [5] shadow casting,
 * [6] shadow bitmap pass, [7] shadow channels, [8] output flush. Event counts of the fast image kernel: [0] shadow
 * cell-sum entries of projection 2 whose low word carried, [1] the most shadow voxels summed into one cell of
 * projection 2, [14] shadow casts that walked the grid because the in-ball list was full. Sub-phases of the shadow
 * (cycles as above; the draw evaluation is [5] - [16] - [17], the voxel evaluation [6] - [18]): [16] casting: cull +
 * work-list append (both image kernels), [17] casting: window test (both); k_images2: [18] voxel pass: bitmap
 * intersection + expansion, [19] the shadow_channel passes, [20] the projection-2 stash sum, [21] the tile clears,
 * [22] the scan behind [1] (only while the counters are on); [23] event: shadow cell-sum entries whose cell another
 * active lane of the same warp hits in the same update. */
int gpdb_debug_phase_cycles(gpdb_ctx *ctx, int enable, uint64_t cycles_out[32]);
/* Development aid: how often the geometry kernels left their first choice of list for a larger tier or an in-place
 * fallback, counted while gpdb_debug_phase_cycles(ctx, 1, ...) has the counters enabled (summed since then; all zero when
 * they are off). counts_out receives:
 *  [0] k_frames samples re-run by tier 1 (ball over 128 keys)  [1] ... by tier 2 (over 1 024 keys)
 *  [2] k_hands samples moved to the 12 800-point tile (staged list over 2 176 points)  [3] ... to the global-memory tier
 *      (over 12 800)  [4] k_hands poses whose Antipodal passes walked the whole staged list (closing region over 1 024
 *      points, or a staged list over 65 535)
 *  [5] k_images2 images handed to k_images because the box holds over 1 024 points  [6] ... because a box point has a
 *      normal of other than unit length  [7] k_images images redone by the global-memory box list (over 2 048 points)
 *  [8] k_images2 shadow points cast in place (work list full)  [9] ... draws evaluated in place (draw list full)
 *  [10] ... images whose shadow voxel stash overflowed
 *  [11] k_images shadow points cast in place  [12] ... draws evaluated in place  [13] ... images whose shadow voxel
 *       list overflowed  [14] ... shadow casts that walked the grid because the in-ball record (tile C) was full
 *  [15] gpdb_reevaluate[_batch][_device] hands whose Antipodal passes walked the grid because the closing region held over
 *       1 024 points (the neighbour-0 padding is not counted) */
int gpdb_debug_path_counts(gpdb_ctx *ctx, uint64_t counts_out[16]);
/* Development aid: gpdb_classify (same batching, same kernels of the implementation lenet_impl selects) that also returns
 * what each LeNet layer computed, in one layout for both implementations. images_hwc as gpdb_classify; outputs:
 *  pool1_out [n][20][28][28]  conv1 + bias (+ReLU) + 2x2 max-pool, NCHW
 *  pool2_out [n][7200]        k = c + 50 j: exactly the values ip1 multiplies (the tensor cores' fp16 hi + lo operand,
 *                             unscaled, hence float64)
 *  ip1_out   [n][500]         ip1 + bias + ReLU
 *  logits_out [n][2]
 * Any output may be NULL. Returns n. */
int gpdb_debug_lenet_layers(gpdb_ctx *ctx, const uint8_t *images_hwc, int32_t n, float *pool1_out, double *pool2_out,
                            float *ip1_out, float *logits_out);

/* ---- Training the classifier on the device (rules in include/gpd_b200_train.h) ------------------------------------------
 * The context's network (image_num_channels, relu_after_conv, image_size 60) trained in float32 on the CUDA cores: the
 * forward pass is gpdb_classify's with lenet_impl = 1, bit for bit. Training keeps its own weights: gpdb_classify uses
 * the loaded ones until the caller passes gpdb_train_weights to gpdb_set_weights. */
typedef struct gpdb_train_params {
  int32_t optimizer;                /* 0 = SGD (torch.optim.SGD, dampening 0), 1 = Adam (torch.optim.Adam, L2 decay) */
  float lr, momentum, weight_decay; /* momentum: SGD only */
  float beta1, beta2, eps;          /* Adam only */
} gpdb_train_params;
/* Starts (or restarts) training: init = the eight arrays in the gpdb_set_weights layout, or NULL for the context's loaded
 * weights (GPDB_ERR_STATE if none). Zeroes the optimiser state and the step count. Bad params (unknown optimizer, a
 * non-finite or negative lr / momentum / weight_decay / eps, betas outside [0, 1)) or a NULL array: GPDB_ERR_INVALID,
 * nothing changed. */
int gpdb_train_begin(gpdb_ctx *ctx, const gpdb_train_params *p, const float *const init[8]);
/* One optimiser step on the mean cross-entropy of n >= 1 images (HWC uint8, as gpdb_classify) and labels in {0, 1}; the
 * step's loss to *loss_out (may be NULL). Before gpdb_train_begin: GPDB_ERR_STATE. n <= 0, a NULL array, image_size other
 * than 60 or a label outside {0, 1} (checked on the device, the message names the first): GPDB_ERR_INVALID. A failed step
 * changes neither the weights, nor the optimiser state, nor the step count. */
int gpdb_train_step(gpdb_ctx *ctx, const uint8_t *images_hwc, const int32_t *labels, int32_t n, float *loss_out);
/* gpdb_train_step on device arrays; d_loss_out (may be NULL) is a device float. */
int gpdb_train_step_device(gpdb_ctx *ctx, const uint8_t *d_images_hwc, const int32_t *d_labels, int32_t n,
                           float *d_loss_out);
/* The current trained weights, in the .bin layout (what gpdb_set_weights reads), to eight host arrays. */
int gpdb_train_weights(gpdb_ctx *ctx, float *const out[8]);
/* Writes {conv1,conv2,ip1,ip2}_{weights,biases}.bin into the directory dir (which must exist; a trailing '/' is optional):
 * what gpdb_load_weights_dir and the reference's EigenClassifier read. Host only. channels other than 1, 3, 12, 15
 * or a NULL argument: GPDB_ERR_INVALID; a file that cannot be written: GPDB_ERR_IO. */
int gpdb_write_weights_dir(const char *dir, int32_t channels, const float *const w[8]);
/* Development aid, like gpdb_debug_lenet_layers: one step's forward state, backward intermediates and gradients, nothing
 * updated. Any n >= 1: a step of more than GPDB_TRAIN_CHUNK images (include/gpd_b200_train.h) runs in chunks as
 * gpdb_train_step does, and each chunk's per-image arrays are copied out at their image offset before the next chunk
 * runs; the gradients are those of the whole step. Every output host memory, any of them NULL; a NULL struct:
 * GPDB_ERR_INVALID. */
typedef struct gpdb_train_debug {
  float *pool1;      /* [n][20][28][28]  as gpdb_debug_lenet_layers */
  float *pool2;      /* [n][7200]        k = c + 50 j */
  float *ip1;        /* [n][500] */
  float *logits;     /* [n][2] */
  uint8_t *choice1;  /* [n][20][28][28]  pooling choice of each pool1 value, 0..3 in row-major window order */
  uint8_t *choice2;  /* [n][7200]        ... of each pool2 value, k = c + 50 j */
  float *loss;       /* [n]              per-image losses */
  float *dlogits;    /* [n][2] */
  float *dip1;       /* [n][500]         d ip1 output, ReLU mask applied */
  float *dpool2;     /* [n][7200]        d pool2 (before its mask), k = c + 50 j */
  float *dpool1;     /* [n][20][28][28]  d pool1 (before its mask) */
  float *grad[8];    /* the eight gradients, .bin layouts */
} gpdb_train_debug;
int gpdb_debug_train_step(gpdb_ctx *ctx, const uint8_t *images_hwc, const int32_t *labels, int32_t n,
                          gpdb_train_debug *out);

/* Version / build info string (arch, lenet implementation). */
const char *gpdb_build_info(void);

#ifdef __cplusplus
}
#endif
#endif /* GPD_B200_H_ */
