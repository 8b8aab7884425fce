// common.cuh — shared declarations of libgpd_b200.so (sm_90a only).
//
// HBM layout of one context (see DESIGN.md "data layout"): two cloud stores (CloudSet), `one` for the single cloud and
// `many` for a batch, each holding the concatenated points of its clouds:
//   store   pts4   float4[N]  points SORTED BY (CLOUD, GRID CELL): x,y,z + cloud-local index bits  (4.8 MB @300k)
//           xyz    float[3N]  points by concatenated index (nb0 lookups)
//           nrm    double[3N] normals by concatenated index, 3xN column-major as the ABI gives them
//           cam    uint8[N]   bit k set when camera k of the point's cloud sees the point
//           cell_start int[ncell+1]   one uniform grid per cloud, x fastest: a run of cells along x is ONE
//                                     contiguous segment of pts4
//           desc   CloudDesc[n]       per cloud: grid, point range, cameras
//   per chunk of samples: frames double[9n], dense pose records gpdb_pose[n*P], flags uint8[n*P],
//           compact candidate list gpdb_pose[nc], images uint8[nc*S*S*C] (HWC, the cv::Mat layout),
//           LeNet activations.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <initializer_list>
#include <utility>
#include <vector>

#include "../../include/gpd_b200.h"
#include "../../include/gpd_b200_shadow.h"

#define GPDB_MAX_ORIENT 32
#define GPDB_MAX_SLOTS 32   // 2 * num_finger_placements
#define GPDB_MAX_DEEPEN 64  // deepen steps
#define GPDB_MAX_NSP 128    // shadow draws per point

// Everything the kernels need, resident in global memory (uniform, L1/L2-cached loads).
struct DevParams {
  // hand geometry / search (cfg/hand_geometry.cfg, grasp_detector.cpp:67-86)
  double finger_width, hand_outer_diameter, hand_depth, hand_height, init_bite;
  int P, n_axes, n_orient, nfp;
  int axes[GPDB_MAX_HAND_AXES];
  int deepen, slots_disjoint, all_axes_z;
  double inv_slot_step;        // 1 / spacing of the finger slots (index estimate in slot_mask)
  double fs[GPDB_MAX_SLOTS];   // FingerHand::finger_spacing_ (finger_hand.cpp:12-19)
  double fsw[GPDB_MAX_SLOTS];  // fs + finger_width
  int J;                       // deepen steps d_j = init_bite + j*0.005 accumulated in double (finger_hand.cpp:120-121)
  double topj[GPDB_MAX_DEEPEN], botj[GPDB_MAX_DEEPEN];
  double cosf;                 // cos(friction_coeff * pi / 180) (antipodal.cpp:28)
  int min_viable;
  // filters (grasp_detector.cpp:334-456)
  double min_ap, max_ap, ws[6];
  int filt_dir;
  double dir[3], thresh;
  double dir_keep;             // smallest dot in [-1, 1] the direction filter keeps (host acos(dot) <= thresh); 2: none
  // rotations (hand_set.cpp:52-53,68-69): rotb = AngleAxis(pi, UnitY); rot[a*n_orient+i]
  double rotb[9];
  double rot[GPDB_MAX_HAND_AXES * GPDB_MAX_ORIENT][9];
  // image geometry (cfg/image_geometry_*.cfg)
  double vol_w, vol_d, vol_h;
  int S, C;
  // shadow (hand_set.cpp:118-233, include/gpd_b200_shadow.h)
  double shadow_length, vox_mult;
  int nsp;                     // num_shadow_points
  int bm_dim;                  // bitmap edge (voxels)
  unsigned lcgA[GPDB_MAX_NSP], lcgC[GPDB_MAX_NSP];  // LCG skip-ahead: seed after t+1 steps = lcgA[t]*seed0 + lcgC[t]
  // radii: float32 predicates (dist < r2) and search extents
  float r2_lrf, r2_hs, r2_img;
  float rf_lrf, rf_hs, rf_img;
  // LeNet
  int relu_after_conv;
};

// A normal of unit length up to float32 rounding. createNormalsImage folds every point of a grasp-image cell into the
// cell as v += (|n| - v) / ||v|| (image_strategy.cpp:136-141); while every normal has unit length the result is the last
// writer's |n|, which is what the image kernels store. A zero normal (a point no camera sees) or a voxel average of
// supplied normals is not of unit length, and neither is a NaN normal (the fold keeps a cell NaN once a NaN writer
// reached it); images holding one replay the fold exactly.
__host__ __device__ __forceinline__ bool unit_normal(const double *n) {
  const double l2 = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
  return fabs(l2 - 1.0) <= 1e-5;
}

struct DevCloud {
  const float4 *pts4;
  const float *xyz;
  const double *nrm;
  const uint8_t *cam;
  const int *cell_start;
  // Cloud::setSamples (gpdb_set_samples): float64 positions addressed by sample indices >= n_points
  const double *samples;
  int n_points;
};

// One cloud of a store: its grid, its range of the concatenated arrays and its cameras. pts4 is sorted by (cloud, cell)
// and its w bits hold the CLOUD-LOCAL index, so keys, shadow seeds and pose records of a cloud do not depend on the
// clouds stored beside it.
struct CloudDesc {
  float lo[3], inv_cell;
  int dim[3];
  int cell_base;              // first entry of this cloud's cells in the store's cell_start
  int off, N, K;              // first point in the concatenated arrays, points, cameras
  int all_seen;               // every point is seen by every camera (cam mask complete): the per-point masks need not be read
  int nonunit;                // some normal is not of unit length (unit_normal): images holding one fold their cells exactly
  int pos;                    // first of this cloud's sample positions in the store's samples (gpdb_set_clouds_samples)
  double vp[GPDB_MAX_CAMERAS][3];
};
// The clouds of a store as the kernels see them: d[n] descriptors, soff[n+1] the CSR offsets of the running batch call's
// samples per cloud (a sample's position in the call = its sample slot).
struct CloudTable {
  const CloudDesc *d;
  const int *soff;
  int n;
};

// A store of clouds. Its arrays are grow-only arenas (repeated installs, one per camera frame, do not pay cudaMalloc /
// cudaFree); n == 0: nothing installed. The context keeps two, `one` and `many`, and a call on one never touches the other.
struct CloudSet {
  float4 *pts4;
  float *xyz;
  double *nrm;
  uint8_t *cam;
  int *src;             // cloud-local raw index of each point (valid after preprocessing: has_src)
  int *cell_start;
  CloudDesc *desc;      // [n] on the device
  int *soff;            // [n + 1] sample offsets of the running batch call (device; the hand offsets of
                        // gpdb_images_batch_device)
  int *off;             // [n + 1] point offsets (host)
  int *sel;             // [n + 1] per-cloud offsets of the records the last batch call left on the device (host)
  int *pos;             // [n + 1] per-cloud offsets of the sample positions while n_samples > 0 (host; the batch only)
  int *raw_off;         // [n + 1] raw point offsets of the preprocessing call that installed the clouds (host, with src)
  size_t point_cap, cell_cap, desc_cap;
  int n, maxk;          // clouds installed, largest camera count
  bool has_src;
  double *samples;      // sample positions (3 x n_samples): gpdb_set_samples (single cloud) / gpdb_set_clouds_samples (batch,
  int n_samples;        // cloud b's at pos[b] .. pos[b+1]-1), or nullptr; a grow-only arena of samples_cap positions
  size_t samples_cap;
  int positions(int b) const { return n_samples ? pos[b + 1] - pos[b] : 0; }  // sample positions of cloud b
  DevCloud view;        // the concatenated arrays as the kernels read them
  int points() const { return n ? off[n] : 0; }
  CloudTable table() const { return CloudTable{desc, soff, n}; }
};

// device error counters: [0] LRF capacity, [1] hand-search capacity (final tier), [2] image box list,
// [3] hand-search tier-1 overflow count (informational), [4] normal-estimation capacity (final tier)
#define GPDB_NERR 8

// path counters (gpdb_debug_path_counts): d_prof[GPDB_PROF_PATH + e], counted only while the counters are on; the events
// are listed in include/gpd_b200.h
#define GPDB_PROF_PATH 16
// sub-phase cycles and events of the shadow half of the image kernels: d_prof[GPDB_PROF_SUB + i], returned by
// gpdb_debug_phase_cycles as cycles_out[16 + i] (the slots are listed in include/gpd_b200.h)
#define GPDB_PROF_SUB 32
#define GPDB_PROF_SLOTS 48
enum PathEvent {
  PATH_FRAMES_T1, PATH_FRAMES_T2, PATH_HANDS_T2, PATH_HANDS_T3, PATH_HANDS_SLAB, PATH_IMG2_BOX, PATH_IMG2_NONUNIT, PATH_IMG_GL,
  PATH_IMG2_CAST, PATH_IMG2_DRAW, PATH_IMG2_STASH, PATH_IMG_CAST, PATH_IMG_DRAW, PATH_IMG_STASH, PATH_IMG_BALL, PATH_LABEL_WALK
};

#define CUDA_TRY(expr)                                                                        \
  do {                                                                                        \
    cudaError_t e__ = (expr);                                                                 \
    if (e__ != cudaSuccess) {                                                                 \
      gpdb_set_error(ctx, GPDB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,         \
                     cudaGetErrorString(e__));                                                \
      return GPDB_ERR_CUDA;                                                                   \
    }                                                                                         \
  } while (0)

// after each kernel launch: counts it in ctx->launches and turns a launch error into GPDB_ERR_CUDA
#define LAUNCH_CHECK()                                                                                    \
  do {                                                                                                    \
    ctx->launches++;                                                                                      \
    cudaError_t e__ = cudaGetLastError();                                                                 \
    if (e__ != cudaSuccess) {                                                                             \
      gpdb_set_error(ctx, GPDB_ERR_CUDA, "%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return GPDB_ERR_CUDA;                                                                               \
    }                                                                                                     \
  } while (0)

struct LenetWeights {  // device pointers, layouts documented in lenet_simt.cu
  float *c1w, *c1b, *c2w, *c2b, *i1w, *i1b, *i2w, *i2b;
  int C;
  bool set;
};

struct C1Affine {  // conv1 epilogue: per-filter weight scale and bias (kernel parameter = constant bank)
  float scale[20], bias[20];
};
struct LenetTc {  // tensor-core (wgmma) weight blobs, lenet_tc.cu
  void *b1, *b2, *b3;
  C1Affine c1_aff;
  int npl, nch1;
  float w2_scale, a2_scale, w3_scale, x3_scale;
  bool ready;
};

struct StageTimes;  // api.cu
struct PipeState;   // api.cu: copy stream, events and the pinned result arenas of the chunk pipeline
struct CommState;   // comm.cu: NCCL communicator (multi-GPU sharding)
struct SisState;    // sis.cu: host-side record of the last gpdb_sis_batch call (gpdb_sis_positions)
struct TrainState;  // train.cu: the trained weights, the optimiser state and the step count (gpdb_train_begin)

// The scratch buffers of a context (gpdb_scratch), each grown on demand and never shrunk. This enum is the whole slot
// map: a buffer is addressed by its enumerator only, and a buffer several stages share is named for what it is, not for
// one of its users. Two users of one buffer must never run at the same time. Outside the chunk pipeline all work of a
// context is ordered on its one stream; the pipeline (gpdb_run_pipeline) drains its streams before it returns, and while
// it runs it is the only place with two users live at once. Its rule is:
//
//   while the main stream is inside images / LeNet / score scatter of chunk i, the hand-search stream runs the hand
//   search and compaction of chunk i + 1. The two sets of buffers must stay disjoint:
//     hand-search stream writes  SCR_CUB, SCR_OVF, SCR_KEYS, SCR_POSES, SCR_CAND (its half), SCR_COUNT, SCR_HANDS_GL,
//                                and chunk i + 1's range of SCR_FLAGS
//     main stream writes         SCR_P16, SCR_WORK_A / B / C, SCR_SCORES, SCR_HWC, SCR_IMG_GL, SCR_IMG_OVF2, SCR_IMG_OVF,
//                                chunk i's range of SCR_PSCORES and (ordered by events) chunk i's half of SCR_CAND
//   both read SCR_SIDX, SCR_FRAMES and SCR_VALID, complete before the hand-search stream starts. The frames stage, the
//   selection after the last chunk and every other entry point run on the main stream alone and may use either set.
//   A stage that joins one of the two concurrent phases takes its buffers from that phase's set or gets a new one.
enum ScratchSlot {
  // main stream: images in the P16 layout (pipeline, gpdb_images, gpdb_classify); cell ids of the grid build
  SCR_P16,
  // cub temporary storage: the compaction on the hand-search stream; select, grid build and preprocessing otherwise
  SCR_CUB,
  // overflow lists of k_frames / k_hands (frames finish before the hand-search stream starts); of the normal estimation
  SCR_OVF,
  // compaction flags and positions (hand-search stream; the pixel filter of gpdb_preprocess_depth and the eligible points of
  // gpdb_subsample_clouds); sort keys and values of the selection
  SCR_KEYS,
  // stage workspaces. LeNet: pool1 / pool2 / ip1 (main stream). Preprocessing: header, filter flags + filtered points,
  // voxel sort buffers. B is also the cell counts of the grid build; in the sharded calls A is the broadcast header and
  // B the all-gather buffer
  SCR_WORK_A, SCR_WORK_B, SCR_WORK_C,
  // sample indices of a call (gpdb_subsample_clouds: its output); the raw upload / the device camera masks of preprocessing
  SCR_SIDX,
  // per call: frames, frame validity, dense per-pose flags, dense per-pose scores
  SCR_FRAMES, SCR_VALID, SCR_FLAGS, SCR_PSCORES,
  // dense pose records of one chunk (hand-search stream); the selection output after the last chunk
  SCR_POSES,
  // double-buffered candidate lists (gpdb_images: the uploaded poses); candidate counts [2] + the cluster count
  SCR_CAND, SCR_COUNT,
  // main stream: candidate scores (+ logits in gpdb_classify); images in the cv::Mat layout
  SCR_SCORES, SCR_HWC,
  // gpdb_reevaluate[_batch]: hands, labels. Clustering: dense + compacted records (+ uploaded hands); group offsets, counts, keep flags
  SCR_HANDS, SCR_LABELS,
  // global-memory fallbacks of the capacity tiers. Image stage (main stream): the box lists of k_images' last tier and
  // the overflow list of its shared-memory tier
  SCR_IMG_GL, SCR_IMG_OVF2,
  // k_hands last tier: the staged neighbourhoods (hand-search stream)
  SCR_HANDS_GL,
  // overflow list of k_images2 (main stream; not SCR_OVF, which the hand search of the next chunk is writing)
  SCR_IMG_OVF,
  // k_frames last tier: the staged neighbourhood keys
  SCR_FRAMES_GL,
  // the device-side input checks (first_bad): the check word, then the per-cloud arrays of the check
  SCR_CHECK,
  // gpdb_sis_batch: kept / evaluated positions, the round's sample lists and counts (main stream, between pipeline calls;
  // read again by gpdb_sis_positions)
  SCR_SIS,
  // host twins of gpdb_preprocess_depth / gpdb_subsample_clouds[_points] / gpdb_segment_plane[s]: the uploaded depth
  // images, the uploaded mask, the eligible bytes on their way back; host installs and preprocessing calls: the
  // uploaded camera-source matrices
  SCR_UPLOAD,
  // gpdb_segment_plane[s]: hypotheses, their inlier counts, the picked and refined planes (plane.cu)
  SCR_PLANE,
  // gpdb_refine_normals[_clouds]: the two float32 iterates, the errors, done flags and counts (refine.cu)
  SCR_REFINE,
  // the k-nearest-neighbour lists (refine_knn_lists, N * k int32) of gpdb_refine_normals[_clouds] and
  // gpdb_remove_outliers[_clouds]: one grow-only buffer for both, the largest part of their memory
  SCR_NBR,
  // gpdb_remove_outliers[_clouds]: mean distances, statistics, keep flags and their scan, per-cloud counts and camera
  // flags, the kept points gathered before they go back into the store (outliers.cu)
  SCR_OUTLIERS,
  // gpdb_normals_organized[_device]: one group of images at a time, its image table, points, distance map, normals and
  // integral tables (organized.cu)
  SCR_ORGANIZED,
  // gpdb_preprocess_depth_organized[_device]: the camera table, the views' first cameras, the fallback counts and the
  // per-point organized flags (organized.cu)
  SCR_ORGANIZED_DEPTH,
  // gpdb_train_step[_device] / gpdb_debug_train_step: one chunk's forward state, backward intermediates and per-image
  // gradient partials (train.cu, train_scratch_bytes)
  SCR_TRAIN,
  // gpdb_render_depth[_device]: one group of cameras at a time, its camera table, camera-frame vertices, face records,
  // tile rectangles, running minimum and per-tile lists; gpdb_sample_meshes[_device]: the offsets, counts and their scan
  // (render.cu)
  SCR_RENDER,
  SCR_N
};

struct gpdb_ctx {
  gpdb_params prm;
  DevParams hp;       // host copy
  DevParams *dp;      // device copy
  int device;
  cudaStream_t stream;
  bool own_stream;
  bool overlap_hands;  // hand search of the chunks ahead on its own stream (gpdb_set_overlap)
  StageTimes *st;
  PipeState *pipe;
  CommState *comm;
  SisState *sis;
  TrainState *train;
  int sm_count;
  int smem_optin;  // largest shared memory (dynamic + static) one block may opt in to, in bytes
  char err[512];
  CloudSet one;       // the single cloud (gpdb_set_cloud / gpdb_preprocess): a store of one cloud
  CloudSet many;      // the batch of clouds (gpdb_set_clouds / gpdb_preprocess_clouds)
  double *d_qtab;
  // weights
  LenetWeights w;
  LenetTc tc;
  // scratch (grown on demand), addressed through gpdb_scratch only
  void *scratch[SCR_N];
  size_t scratch_sz[SCR_N];
  int *d_err;
  unsigned long long *d_prof;  // optional phase counters (gpdb_debug_phase_cycles, GPDB_PROF_SLOTS slots), nullptr = off
  int64_t launches;
  double last_ms[8];
  double pre_ms[6];   // gpdb_preprocess stage timings
  gpdb_pose *d_sel;   // gpdb_detect_select: all classified candidates of a call (grown on demand)
  size_t sel_cap;
  cudaEvent_t ev[6];  // stage boundaries of a preprocessing call (pre_ms)
};

void gpdb_set_error(gpdb_ctx *ctx, int code, const char *fmt, ...);
// device-side stage timers (CUDA events on the context stream). stages: 0 frames, 1 hand search +
// compaction, 2 images, 3 LeNet, 4 whole call, 5 conv1, 6 conv2, 7 ip1+ip2
cudaEvent_t gpdb_st_begin(gpdb_ctx *ctx);
void gpdb_st_end(gpdb_ctx *ctx, int stage, cudaEvent_t begin);
void *gpdb_scratch(gpdb_ctx *ctx, ScratchSlot slot, size_t bytes);  // returns nullptr on failure (error set)

// Several arrays in one buffer, each stated once. A layout is a callable that takes its arrays from a Carve, in order:
// run with a null base it only adds up the bytes (carve_bytes), run over a buffer it assigns the pointers (carve_at),
// so the size and the pointers cannot disagree. Each array starts at the alignment of its type, or at `align`.
struct Carve {
  unsigned char *base;
  size_t at;
  template <class T> T *take(size_t n, size_t align = alignof(T)) {
    at = (at + align - 1) / align * align;
    T *p = base ? reinterpret_cast<T *>(base + at) : nullptr;
    at += sizeof(T) * n;
    return p;
  }
};
template <class Layout> size_t carve_bytes(Layout &&layout) {
  Carve c{nullptr, 0};
  layout(c);
  return c.at;
}
template <class Layout> void carve_at(void *base, Layout &&layout) {
  Carve c{static_cast<unsigned char *>(base), 0};
  layout(c);
}
// scratch slot `slot` grown to the layout's bytes, then carved by it; false: no memory (error set)
template <class Layout> bool gpdb_carve(gpdb_ctx *ctx, ScratchSlot slot, Layout &&layout) {
  void *base = gpdb_scratch(ctx, slot, carve_bytes(layout));
  if (!base) return false;
  carve_at(base, layout);
  return true;
}

// api.cu
int gpdb_pipe_create(gpdb_ctx *ctx);
void gpdb_pipe_destroy(gpdb_ctx *ctx);
int gpdb_check_state(gpdb_ctx *ctx, bool need_cloud, bool need_weights);
void *gpdb_result_extra(gpdb_result *r, size_t bytes);  // pinned host memory owned by the result (freed with it)
// Where the results of a pipeline call go. The result struct always receives the counts and timings.
enum PipeDest {
  PIPE_TO_HOST,      // the per-sample / per-pose arrays and every candidate record (+ images if kept) to the host arena
  PIPE_TOP_HOST,     // the select_k best records (per_cloud: of every cloud, sample slots cloud-local) to the host arena
  PIPE_TOP_DEVICE,   // the same selection of a per_cloud call to d_selected on the device; nothing to the host
  PIPE_STAY,         // nothing leaves the device: the caller reads the dense flags and scores there
  PIPE_ALL_DEVICE,   // PIPE_STAY, and every scored candidate record stays in ctx->d_sel (sample-slot order, stream slots)
  PIPE_ALL_CALLER    // every candidate record of a per_cloud call to d_selected (room for n * P), grouped by cloud with
                     // cloud-local sample slots; store->sel (host) receives the per-cloud offsets
};
// One call of the chunked device pipeline (see api.cu): where its inputs are and where its outputs go.
struct PipeRequest {
  CloudSet *store;            // the clouds the samples address
  const int32_t *sample_idx;  // n sample indices, in host or device memory
  int32_t n;
  bool samples_on_device;
  bool per_cloud;             // the samples are the CSR stream of a batch call (offsets in store->soff, checked by the
                              // caller); else they address the one cloud of the store and host samples are checked here
  bool classify;              // images + LeNet scores; false: the hand search alone
  uint8_t *d_flags;           // dense per-pose flags and scores [n * P] on the device. In: the caller's arrays, or null for
  float *d_scores;            // the pipeline's scratch. Out: the arrays that were used, valid until the next call
  PipeDest dest;
  int select_k;               // PIPE_TOP_*: records to keep (per cloud when per_cloud)
  gpdb_pose *d_selected;      // PIPE_TOP_DEVICE, PIPE_ALL_CALLER: receives them
  int slot_base;              // added to every sample_slot (rank offset of a sharded call)
};
int gpdb_run_pipeline(gpdb_ctx *ctx, PipeRequest &rq, gpdb_result *out);
// (re)allocates the arenas of store s for at least n points and n_clouds clouds
int gpdb_cloud_reserve(gpdb_ctx *ctx, CloudSet &s, size_t n, int n_clouds);
// Installs the B clouds whose points the arrays of s already hold (cloud b: off[b] .. off[b+1]-1, host offsets): desc[b]
// (host) carries K / vp / all_seen and receives the point range; uploads the descriptors and builds the grids. nonunit:
// also set the descriptors' nonunit flags from the stored normals (false: the caller sets them once the normals exist).
int gpdb_install_clouds(gpdb_ctx *ctx, CloudSet &s, CloudDesc *desc, const int *off, int B, bool nonunit);
// The points of B clouds (cloud b: off[b] .. off[b+1]-1, host offsets) into store s, ready for gpdb_install_clouds:
// reserves s, copies xyz and normals into it, then on the device refuses a non-finite coordinate (naming the first
// point) and packs the camera-source matrices (cloud b: n_cameras[b] entries per point, concatenated; null: every
// camera sees every point) into s.cam, a camera seeing a point when its entry is > 0; desc[b] receives K / vp /
// all_seen. device: xyz, normals and cam_source are the caller's device arrays, else host arrays uploaded here
// (cam_source into SCR_UPLOAD).
int gpdb_stage_clouds(gpdb_ctx *ctx, CloudSet &s, const char *name, int B, const int32_t *off, const float *xyz,
                      const double *normals, const int32_t *cam_source, const int32_t *n_cameras,
                      const double *view_points, bool device, CloudDesc *desc);
// every non-null pointer must be device (or managed) memory of the context's device; runs before any device work
int gpdb_check_device_ptrs(gpdb_ctx *ctx, const char *name,
                           std::initializer_list<std::pair<const char *, const void *>> ptrs);
static const unsigned long long NO_BAD = ~0ull;  // the check word when no position offends
// The check-word protocol of the device-side checks. The word, at the head of SCR_CHECK, is set to all ones;
// enqueue(d_bad, d_extra) queues the kernel that lowers it to the first offending position, with `extra` bytes behind the
// word for the check's own arrays; *bad receives the word (NO_BAD: nothing offends) once the stream has drained.
template <class Enqueue>
static int first_bad(gpdb_ctx *ctx, size_t extra, unsigned long long *bad, Enqueue enqueue) {
  unsigned long long *d_bad = (unsigned long long *)gpdb_scratch(ctx, SCR_CHECK, sizeof(*d_bad) + extra);
  if (!d_bad) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemsetAsync(d_bad, 0xFF, sizeof(*d_bad), ctx->stream));
  const int rc = enqueue(d_bad, d_bad + 1);
  if (rc != GPDB_OK) return rc;
  CUDA_TRY(cudaMemcpyAsync(bad, d_bad, sizeof(*bad), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return GPDB_OK;
}
// what every call that installs a batch does first: a failed call leaves no batch, no sample positions and no SIS record
// behind (the SIS positions describe clouds that are gone); the single cloud is never touched
void gpdb_drop_batch(gpdb_ctx *ctx);
// GPDB_ERR_STATE unless a batch is installed; hint names the calls that install one
int gpdb_need_batch(gpdb_ctx *ctx, const char *name, const char *hint);
// CSR offsets off[B+1] (the array `label`) from the host: they start at 0 and never decrease; entry b belongs to the b-th
// `unit` (cloud or group). A call whose start message lists other arguments too checks the start itself first.
int gpdb_check_offsets(gpdb_ctx *ctx, const char *name, const char *label, const int32_t *off, int B, const char *unit);
// The cloud-local indices d_idx[off[b] .. off[b+1]) of cloud b of the installed batch must lie in [0, N_b + M_b), M_b
// its sample positions. The list d_idx and its offsets d_off are in device memory, off is the host copy of d_off;
// batch_check_samples finds the first offending position, which the message names. init: the initial indices of
// gpdb_sis_batch, which has dropped the positions (M_b = 0) and names the indices so.
int gpdb_check_cloud_indices(gpdb_ctx *ctx, const char *name, bool init, const int32_t *off, const int32_t *d_idx,
                             const int *d_off);
// the preprocessing parameters, against the caller's normals (null: none)
int gpdb_check_preprocess_params(gpdb_ctx *ctx, const char *name, const gpdb_preprocess_params *pp, const double *normals);
// The steps of a preprocessing call after the filter and voxelisation (store s holds the processed points, poff[B+1] their
// offsets, desc[B] the camera fields): install with one grid per cloud, normals, nonunit flags, stage timings, and the
// raw offsets roff[B+1] the source indices refer to. after_normals (may be empty) runs between the normal estimation and
// the nonunit flags, inside the normals' stage timing. A failure leaves no cloud in s.
int gpdb_preprocess_install(gpdb_ctx *ctx, CloudSet &s, CloudDesc *desc, int B, const int32_t *roff,
                            const gpdb_preprocess_params *pp, int32_t *poff,
                            const std::function<int()> &after_normals = nullptr);
// drops the sample positions of store s and makes its arena hold n positions (grown, never shrunk)
int gpdb_reserve_samples(gpdb_ctx *ctx, CloudSet &s, int n);
// gpdb_find_clusters_batch after the argument checks (gpdb_find_clusters: one group): the clusters of all G groups in one
// k_clusters launch, compacted in hand order, so group g's are clusters_out[cluster_offsets_out[g] ..
// cluster_offsets_out[g+1]); returns their total. device: hands are device arrays (no copy of the hands); clusters_out
// may be host or device memory
int gpdb_cluster_groups(gpdb_ctx *ctx, int G, const int32_t *hand_offsets, const gpdb_pose *hands, int min_inliers,
                        gpdb_pose *clusters_out, int32_t *cluster_offsets_out, bool device = false);

// largest b in [0, n) with a[b] <= x, for a non-decreasing a with a[0] <= x: the cloud that owns position x of a CSR array
__device__ __forceinline__ int csr_owner(const int *a, int n, long long x) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] <= x) lo = mid; else hi = mid;
  }
  return lo;
}

// One sequential fold over v[0 .. n) per CTA of THREADS threads: thread 0 applies add(v[j]) for j = 0, 1, .., n - 1
// from one half of `stage` (double-buffered chunks of CHUNK values in shared memory, 16-byte aligned) while warps 1..
// stage the next chunk into the other half, so the chain waits on shared loads only. Every thread of the CTA calls it;
// it returns with the CTA synchronised.
template <int THREADS, int CHUNK, class Add>
__device__ __forceinline__ void ordered_fold(const float *v, int n, float (*stage)[CHUNK], Add &&add) {
  const int nc = (n + CHUNK - 1) / CHUNK;
  for (int j = threadIdx.x; j < min(n, CHUNK); j += THREADS) stage[0][j] = __ldg(v + j);
  __syncthreads();
  for (int c = 0; c < nc; c++) {
    const int base = c * CHUNK;
    if (threadIdx.x == 0) {
      const float *p = stage[c & 1];
      const int len = min(CHUNK, n - base);
      int j = 0;
#pragma unroll 4
      for (; j + 4 <= len; j += 4) {
        const float4 q = *reinterpret_cast<const float4 *>(p + j);
        add(q.x);
        add(q.y);
        add(q.z);
        add(q.w);
      }
      for (; j < len; j++) add(p[j]);
    } else if (threadIdx.x >= 32 && c + 1 < nc) {
      const int nb = base + CHUNK, nl = min(CHUNK, n - nb);
      for (int j = threadIdx.x - 32; j < nl; j += THREADS - 32) stage[(c + 1) & 1][j] = __ldg(v + nb + j);
    }
    __syncthreads();
  }
}

// batch_device.cu (the installs and batch entry points, host and device twins). The checks lower *d_first_bad (set to
// all ones by the caller) to the first offending position.
// camera masks of N points in B clouds (point offsets d_off[B+1]; cloud b's N_b x K_b int32 block starts at entry
// d_row_off[b] of d_rows, K_b = d_k[b]; d_rows null: every camera sees every point), seen as == 1 (eq1) or > 0;
// d_all_seen[b] (1 on entry) drops to 0 when a point of cloud b misses a camera; strict01: first entry other than 0 / 1
int batch_pack_cameras(gpdb_ctx *ctx, const int32_t *d_rows, const int *d_off, const long long *d_row_off, const int *d_k,
                       int B, int N, bool eq1, bool strict01, uint8_t *d_cam, int *d_all_seen,
                       unsigned long long *d_first_bad);
// first point (float index / 3) of d_v[n] with a non-finite coordinate
int batch_first_nonfinite(gpdb_ctx *ctx, const float *d_v, long long n, unsigned long long *d_first_bad);
// first position i of the CSR sample list (cloud b: d_soff[b] .. d_soff[b+1]-1) with d_sidx[i] outside [0, d_lim[b])
int batch_check_samples(gpdb_ctx *ctx, const int *d_sidx, int n, const int *d_soff, int B, const int *d_lim,
                        unsigned long long *d_first_bad);
// d_out[j] = d_in[j] with its sample slot made local to the cloud whose slots d_soff assigns it (d_in may equal d_out)
int batch_local_slots(gpdb_ctx *ctx, const gpdb_pose *d_in, int n, const int *d_soff, int B, gpdb_pose *d_out);
// d_out[j] = d_in[j] with sample slot base + j: the image kernels then find hand j's cloud from the hand offsets held in
// the store's soff (gpdb_images_batch_device)
int batch_image_hands(gpdb_ctx *ctx, const gpdb_pose *d_in, int n, int base, gpdb_pose *d_out);

// sis.cu (gpdb_sis_batch[_device], gpdb_sis_positions; include/gpd_b200_sis.h)
// a new batch, or a SIS call that fails, leaves nothing for gpdb_sis_positions to read
void sis_forget(gpdb_ctx *ctx);
void sis_free(gpdb_ctx *ctx);  // gpdb_destroy: the SIS record

// geometry.cu
// builds the per-cloud grids of store s (its s.n descriptors hold off / N) and fills the descriptors' grid fields
int geo_build_grid_batch(gpdb_ctx *ctx, CloudSet &s);
// the top k of every cloud of the running batch (store s) among the n candidate records (sample-slot order, scores
// filled) -> *d_out (device scratch); s.sel[s.n + 1] (host) receives the per-cloud output offsets. Returns the total or
// an error.
int geo_select_batch(gpdb_ctx *ctx, CloudSet &s, const gpdb_pose *d_cand, int n, int k, gpdb_pose **d_out);
// the per-cloud offsets of the n candidate records of the running batch (store s; sample-slot order, stream slots) ->
// cand_off[s.n + 1] (host), once the stream has drained
int geo_batch_cand_off(gpdb_ctx *ctx, const CloudSet &s, const gpdb_pose *d_cand, int n, int *cand_off);
int geo_frames(gpdb_ctx *ctx, const CloudSet &s, const int *d_sidx, int n, double *d_frames, uint8_t *d_valid);
int geo_hands(gpdb_ctx *ctx, const CloudSet &s, const int *d_sidx, int n, int slot0, const double *d_frames,
              const uint8_t *d_valid, gpdb_pose *d_poses, uint8_t *d_flags);
// compacts poses with VALID|FILTERED into d_cand (in (sample,pose) order); *d_count receives the count
int geo_compact(gpdb_ctx *ctx, const gpdb_pose *d_poses, const uint8_t *d_flags, int n_poses, gpdb_pose *d_cand,
                int *d_count);
// grasp images in the P16 layout: S*S pixels of 16 bytes (channels 0..C-1, zero padded) per image = conv1's operand
int geo_images(gpdb_ctx *ctx, const CloudSet &s, const gpdb_pose *d_cand, int nc, uint8_t *d_p16);
int geo_p16_to_hwc(gpdb_ctx *ctx, const uint8_t *d_p16, int n, uint8_t *d_hwc);  // -> cv::Mat layout (C bytes per pixel)
int geo_hwc_to_p16(gpdb_ctx *ctx, const uint8_t *d_hwc, int n, uint8_t *d_p16);
int geo_scatter_scores(gpdb_ctx *ctx, const gpdb_pose *d_cand, const float *d_scores, int nc, int slot0, int P,
                       float *d_pose_scores, gpdb_pose *d_cand_out);

// HandSearch::reevaluateHypotheses: labels + half / full flags of the given hands, hand i against the cloud of store s
// whose group holds it (group offsets in s.soff, uploaded by the caller; a store of one cloud reads no offsets)
int geo_label(gpdb_ctx *ctx, const CloudSet &s, gpdb_pose *d_hands, int n, int *d_labels);
// Clustering::findClusters (remove_inliers = false) on each of G groups of hands (group g: d_goff[g] .. d_goff[g+1]-1,
// device offsets): dense per-hand cluster records + keep flags (3 = cluster), for geo_compact; d_gcount[G] (zeroed here)
// receives the clusters per group
int geo_clusters(gpdb_ctx *ctx, const gpdb_pose *d_hands, int n, const int *d_goff, int G, int min_inliers, gpdb_pose *d_dense,
                 uint8_t *d_keep, int *d_gcount);
// the k highest-scoring of the n candidate records (scores filled), descending, stable -> d_out[k]
int geo_select(gpdb_ctx *ctx, const gpdb_pose *d_cand, int n, int k, gpdb_pose *d_out);

// preprocess.cu (cloud preprocessing, SURVEY.md 8(f).1)
// per-cloud bounds of xyz (cloud b: points d_off[b] .. d_off[b+1]-1, device offsets; `largest` points in the largest
// cloud) -> bounds[6b .. 6b+5] (min x y z, max x y z as order-preserving ints; an empty cloud keeps INT_MAX / INT_MIN)
int pre_bounds_batch(gpdb_ctx *ctx, const float *xyz, const int *d_off, int B, int largest, int *bounds);
// the exclusive scan of n compaction flags: flag holds n + 1 ints (flag[n] is zeroed here), pos[0 .. n] receives the
// positions and pos[n] the number of flagged entries; counts its 2 launches
int scan_flags(gpdb_ctx *ctx, int *flag, int *pos, int n);
// filters + voxelises a raw batch into the arenas of store s (reserved inside); poff[B+1] (host) = processed offsets
int pre_filter_voxelize_batch(gpdb_ctx *ctx, CloudSet &s, const float *d_xyz_raw, const uint8_t *d_cam_raw,
                              const double *d_nrm_raw, int M, int B, const int *roff, const gpdb_preprocess_params &pp,
                              int *poff, cudaEvent_t ev_filter_done);
// the two halves of pre_filter_voxelize_batch, for a front that filters its own way (depth.cu). PreBatch: the device
// header of one call (SCR_WORK_A): workspace, raw / filtered / processed offsets, bounds, voxel error words, and `extra`
// bytes for the front
struct PreBatch {
  double *ws;
  int *roff, *foff, *poff, *bounds, *verr;
  unsigned char *extra;
};
int pre_batch_header(gpdb_ctx *ctx, int B, const int *roff, const gpdb_preprocess_params &pp, size_t extra, PreBatch &h);
// h.foff from the exclusive scan pos of the filter flags (M + 1 entries): foff[b] = pos[roff[b]]
int pre_filter_offsets(gpdb_ctx *ctx, const int *pos, const PreBatch &h, int B);
// the filtered points (host offsets foff[B+1]; keep = raw index in the call's numbering, xyz1 the coordinates) voxelised
// (or gathered) into store s; poff[B+1] (host) = processed offsets
int pre_voxelize_back(gpdb_ctx *ctx, CloudSet &s, const PreBatch &h, const int *foff, const int *keep, const float *xyz1,
                      const uint8_t *d_cam_raw, const double *d_nrm_raw, int B, const gpdb_preprocess_params &pp, int *poff);

// depth.cu (include/gpd_b200_depth.h)
// the depth format of gpdb_preprocess_depth[_device] and gpdb_render_depth[_device]: GPDB_DEPTH_U16 or GPDB_DEPTH_F32
int check_depth_format(gpdb_ctx *ctx, const char *name, int32_t format);
// The camera checks of gpdb_preprocess_depth[_device] and gpdb_render_depth[_device]: view b has n_cameras[b] (1..8)
// cameras, each of them well formed, and the call holds fewer than 2^31 pixels; roff[B+1] receives the raw offsets
// (cumulative pixels per view)
int check_depth_cameras(gpdb_ctx *ctx, const char *name, int32_t B, const int32_t *n_cameras,
                        const gpdb_depth_camera *cams, std::vector<int> &roff);

// refine.cu (include/gpd_b200_refine.h): rule 1 alone. nbr[g*k + r], r < min(k, N_b): the cloud-local index of the r-th
// neighbour of concatenated point g of store s (device memory of N * k int32; k in 1..128).
int refine_knn_lists(gpdb_ctx *ctx, const CloudSet &s, int k, int *nbr);
// organized.cu (include/gpd_b200_organized.h). Rules 6 and 7 on store s, just installed with radius normals by
// gpdb_preprocess_depth from the depth images d_depth (device) of the B views with n_cameras[b] cameras cams: each point
// whose representative pixel has a finite organized normal takes it in s.nrm; n_fallback[B] (host, may be null) receives
// the other points per view. The nonunit flags are the caller's.
int org_depth_normals(gpdb_ctx *ctx, const char *name, CloudSet &s, const void *d_depth, int format,
                      const gpdb_depth_camera *cams, const int *n_cameras, int B, int *n_fallback);
int pre_normals_batch(gpdb_ctx *ctx, CloudSet &s, double radius);  // normals of the installed store (grids built)
int pre_nonunit_batch(gpdb_ctx *ctx, CloudSet &s);                 // per-cloud nonunit flags of the store, in the descriptors

// lenet_simt.cu
int lenet_upload(gpdb_ctx *ctx, const float *const w[8]);
// Host buffers that receive the layer outputs of a forward pass (gpdb_debug_lenet_layers), any of them null:
// pool1 [n][20][28][28], pool2 [n][7200] (k = c + 50 j, the values ip1 multiplies), ip1 [n][500]
struct LenetLayers {
  float *pool1;
  double *pool2;
  float *ip1;
};
// layers == nullptr (every production call): the kernels alone, nothing is read back
int lenet_forward(gpdb_ctx *ctx, const uint8_t *d_images, int n, float *d_scores, float *d_logits,
                  const LenetLayers *layers = nullptr);

// The float32 SIMT forward (lenet_impl = 1) with the weights w (lenet_upload's layouts): pool1 p1 [n][20][28][28], pool2
// p2 [n][7200] (k = c + 50 j), ip1 h3 [n][500], scores and logits. lenet_forward and the training forward both run it.
int lenet_simt_run(gpdb_ctx *ctx, const LenetWeights &w, const uint8_t *d_images, int n, float *p1, float *p2, float *h3,
                   float *d_scores, float *d_logits);

// train.cu (include/gpd_b200_train.h)
void train_free(gpdb_ctx *ctx);

// lenet_tc.cu (wgmma conv1 / conv2 / ip1)
int lenet_tc_upload(gpdb_ctx *ctx, const float *const w[8]);
struct __half;
int lenet_tc_forward(gpdb_ctx *ctx, const uint8_t *d_images, int n, float *p1, __half *xc, float *h3);
size_t lenet_tc_xc_bytes(int n);
// pool1 and pool2 of the last lenet_tc_forward (device p1 / xc, stream synchronised) in the LenetLayers layout
int lenet_tc_read_layers(gpdb_ctx *ctx, int n, const float *p1, const __half *xc, const LenetLayers &out);
