// render.cu — depth images of triangle-mesh scenes and surface samples of the same meshes (include/gpd_b200_render.h):
// gpdb_render_depth[_device] and gpdb_sample_meshes[_device].
//
// Rendering, per group of cameras:
//   k_rnd_xform    one float64 camera-frame copy per (camera, vertex) (rule 2)
//   k_rnd_setup    m0..m2, n and h once per (camera, face) (rule 4), and the screen tiles the face's conservative pixel
//                  bounds touch
//   k_rnd_bin      the (face, tile) pairs counted per tile, then, after an exact scan, filled into per-tile lists with
//                  integer atomics: the list order is arbitrary, the resolve does not depend on it
//   k_rnd_resolve  one CTA per (camera, tile), one thread per pixel: the lexicographic minimum of (t, face) over the
//                  tile's list (rule 5), then the depth and face images
// The cameras of a call are processed in groups whose per-camera arrays fit RND_GROUP_BYTES; a group's (face, tile)
// pairs are resolved in chunks of at most the carved list length, the running minimum kept per pixel between chunks, so a
// face covering every tile (a table) costs one list entry per tile and memory stays bounded.
//
// Sensor views (include/gpd_b200_sensor.h): with a baseline every camera is followed by its projector, a camera of the
// same intrinsics whose pose is shifted along the camera's +x, and the two always share a group, so the projector's
// image counts toward the group's bytes. Every chunk's resolve then keeps the running minimum, and after the group's
// last chunk
//   k_sensor       one thread per camera pixel: rules 1-8, reading the camera's and the projector's (t, face) minima and
//                  the hit face's vertices, then the depth and face images
//
// Sampling: k_mesh_count per face (rule 6's count, a 64-bit total), scan_flags over the counts once the total is known
// to lie below 2^31, then k_mesh_write per point. Scratch: SCR_RENDER. Compiled with -fmad=false: every float64
// operation is rounded on its own.
//
// The entry points gpdb_render_depth[_device], gpdb_render_sensor_depth[_device] and gpdb_sample_meshes[_device], with
// their checks and the host twins' uploads, follow the kernels.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/gpd_b200_render.h"
#include "../../include/gpd_b200_sensor.h"
#include "common.cuh"

namespace {

constexpr int RND_TILE = 16;                                 // tile edge in pixels: one thread per pixel
constexpr int RND_THREADS = RND_TILE * RND_TILE;
constexpr int RND_STAGE = 64;                                // face records a resolve CTA stages in shared memory at once
constexpr size_t RND_GROUP_BYTES = size_t(256) << 20;        // per-camera arrays of one group
constexpr long long RND_LIST_CAP = 32ll << 20;               // (face, tile) entries one chunk may hold
constexpr double RND_PROJ_LIMIT = 16777216.0;                // 2^24: projected bounds beyond this take every tile

// One camera of a group. Its vertices are xv .. xv + nv - 1 of the group's camera-frame vertices, its faces the items
// item .. item + nf - 1, its tiles tile .. tile + tx*ty - 1; pix is its first pixel in the call's images.
struct RndCam {
  double pose[12];
  double fx, fy, cx, cy, scale;
  int W, H, tx, ty;
  int vbase, nv, fbase, nf;
  int xv, item, tile, pad;
  long long pix;
};

// rule 2: q[i] for every (camera, vertex) of the group; xv_off[G+1] the cameras' first entries
__global__ void k_rnd_xform(const RndCam *cams, const int *xv_off, int G, int n, const float *vtx, double *q) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const RndCam &c = cams[csr_owner(xv_off, G, i)];
  const long long v = (long long)c.vbase + (i - c.xv);
  const float p[3] = {vtx[3 * v], vtx[3 * v + 1], vtx[3 * v + 2]};
  double o[3];
  gpdb_render_to_camera(c.pose, p, o);
  q[3 * (size_t)i] = o[0];
  q[3 * (size_t)i + 1] = o[1];
  q[3 * (size_t)i + 2] = o[2];
}

// The tiles a face may cover, inclusive, as (tx0, ty0, tx1, ty1); tx0 > tx1: none. Every tile of the image when a vertex
// lies at or behind the camera plane, a projected bound is not finite or beyond 2^24 pixels, or an edge runs so close to
// a ray through the eye that its m is within rounding of zero. Otherwise the projected bounding box grown by one pixel:
// the coverage test of rule 4 is exact up to float64 roundings, many orders of magnitude below a pixel there.
__device__ int4 rnd_tiles(const RndCam &c, const double *A, const double *B, const double *C, const double *rec) {
  const int4 all = make_int4(0, 0, c.tx - 1, c.ty - 1);
  const int4 none = make_int4(1, 0, 0, 0);
  if (rec[9] == 0.0 && rec[10] == 0.0 && rec[11] == 0.0) return none;  // n = 0: s = 0 for every ray
  const double *V[3] = {A, B, C};
  double umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
  for (int k = 0; k < 3; k++) {
    const double *P = V[k], *Q = V[(k + 1) % 3], *m = rec + 3 * k;
    if (!(P[2] > 0.0)) return all;
    const double pm = fmax(fabs(P[0]), fmax(fabs(P[1]), fabs(P[2]))), qm = fmax(fabs(Q[0]), fmax(fabs(Q[1]), fabs(Q[2])));
    const double mm = fmax(fabs(m[0]), fmax(fabs(m[1]), fabs(m[2])));
    if (!(mm > 1.4901161193847656e-8 * (pm * qm))) return all;  // 2^-26
    const double u = c.cx + c.fx * (P[0] / P[2]), v = c.cy + c.fy * (P[1] / P[2]);
    umin = fmin(umin, u);
    umax = fmax(umax, u);
    vmin = fmin(vmin, v);
    vmax = fmax(vmax, v);
  }
  if (!(fabs(umin) < RND_PROJ_LIMIT && fabs(umax) < RND_PROJ_LIMIT && fabs(vmin) < RND_PROJ_LIMIT &&
        fabs(vmax) < RND_PROJ_LIMIT))
    return all;
  const int u0 = max((int)floor(umin) - 1, 0), u1 = min((int)ceil(umax) + 1, c.W - 1);
  const int v0 = max((int)floor(vmin) - 1, 0), v1 = min((int)ceil(vmax) + 1, c.H - 1);
  if (u0 > u1 || v0 > v1) return none;
  return make_int4(u0 / RND_TILE, v0 / RND_TILE, u1 / RND_TILE, v1 / RND_TILE);
}

// rule 4's setup of every (camera, face) item of the group, its tile rectangle and its (face, tile) pairs; *pairs (zeroed
// by the caller) receives their sum
__global__ void k_rnd_setup(const RndCam *cams, const int *item_off, int G, int n, const int *faces, const double *q,
                            double *rec, int4 *rect, int *count, unsigned long long *pairs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const RndCam &c = cams[csr_owner(item_off, G, i)];
  const long long f = (long long)c.fbase + (i - c.item);
  const double *A = q + 3 * ((size_t)c.xv + faces[3 * f]);
  const double *B = q + 3 * ((size_t)c.xv + faces[3 * f + 1]);
  const double *C = q + 3 * ((size_t)c.xv + faces[3 * f + 2]);
  double r[GPDB_RENDER_REC];
  gpdb_render_setup(A, B, C, r);
  for (int k = 0; k < GPDB_RENDER_REC; k++) rec[(size_t)GPDB_RENDER_REC * i + k] = r[k];
  const int4 t = rnd_tiles(c, A, B, C, r);
  rect[i] = t;
  const int cnt = t.x > t.z ? 0 : (t.z - t.x + 1) * (t.w - t.y + 1);
  count[i] = cnt;
  if (cnt) atomicAdd(pairs, (unsigned long long)cnt);
}

// the (face, tile) pairs of items i0 .. i1-1: fill = false counts them per tile (cnt); fill = true writes item i into
// tile t's list at pos[t] + atomicAdd(cnt[t], 1), cnt zeroed again by the caller
__global__ void k_rnd_bin(const RndCam *cams, const int *item_off, int G, int i0, int i1, const int4 *rect, int *cnt,
                          const int *pos, int *list, bool fill) {
  const int i = i0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= i1) return;
  const RndCam &c = cams[csr_owner(item_off, G, i)];
  const int4 r = rect[i];
  for (int y = r.y; y <= r.w; y++)
    for (int x = r.x; x <= r.z; x++) {
      const int t = c.tile + y * c.tx + x;
      const int k = atomicAdd(cnt + t, 1);
      if (fill) list[pos[t] + k] = i;
    }
}

// One CTA per tile of the group: each thread keeps the lexicographic minimum of (t, face) of its pixel over the tile's
// list, starting from none (first chunk) or from the running minimum (best_t / best_f), and writes either the running
// minimum back or, after the last chunk, the depth and face images (rule 5).
__global__ void __launch_bounds__(RND_THREADS) k_rnd_resolve(const RndCam *cams, const int *tile_off, int G,
                                                             const double *rec, const int *pos, const int *list,
                                                             bool first, bool last, double *best_t, int *best_f,
                                                             const long long *pix_off, int format, void *depth,
                                                             int *face_out) {
  __shared__ double s_rec[RND_STAGE][GPDB_RENDER_REC];
  __shared__ int s_face[RND_STAGE];
  const int tile = blockIdx.x;
  const int g = csr_owner(tile_off, G, tile);
  const RndCam &c = cams[g];
  const int lt = tile - c.tile;
  const int u = (lt % c.tx) * RND_TILE + threadIdx.x % RND_TILE, v = (lt / c.tx) * RND_TILE + threadIdx.x / RND_TILE;
  const bool in = u < c.W && v < c.H;
  const long long gp = pix_off[g] + (long long)v * c.W + u;  // the pixel in the group's running minimum
  double d[2];
  gpdb_render_ray(u, v, c.fx, c.fy, c.cx, c.cy, d);
  double bt = INFINITY;
  int bf = -1;
  if (!first && in) {
    bt = best_t[gp];
    bf = best_f[gp];
  }
  const int e0 = pos[tile], e1 = pos[tile + 1];
  for (int base = e0; base < e1; base += RND_STAGE) {
    const int m = min(RND_STAGE, e1 - base);
    __syncthreads();
    for (int k = threadIdx.x; k < m * GPDB_RENDER_REC; k += RND_THREADS) {
      const int r = k / GPDB_RENDER_REC, w = k % GPDB_RENDER_REC;
      s_rec[r][w] = rec[(size_t)GPDB_RENDER_REC * list[base + r] + w];
    }
    for (int k = threadIdx.x; k < m; k += RND_THREADS) s_face[k] = list[base + k] - c.item;
    __syncthreads();
    if (in)
      for (int k = 0; k < m; k++) {
        double t;
        if (gpdb_render_hit(s_rec[k], d[0], d[1], &t) && (t < bt || (t == bt && s_face[k] < bf))) {
          bt = t;
          bf = s_face[k];
        }
      }
  }
  if (!in) return;
  if (!last) {
    best_t[gp] = bt;
    best_f[gp] = bf;
    return;
  }
  const long long o = c.pix + (long long)v * c.W + u;
  bool ret = false;
  const uint32_t raw = bf >= 0 ? gpdb_render_raw(bt, c.scale, format, &ret) : 0u;
  if (format == GPDB_DEPTH_F32) static_cast<uint32_t *>(depth)[o] = raw;
  else static_cast<uint16_t *>(depth)[o] = (uint16_t)raw;
  if (face_out) face_out[o] = ret ? bf : -1;
}

// One camera of a sensor group: its entry in the group's camera table, its projector's (-1: none), its index within its
// view and its view's key
struct SensorCam {
  int cam, proj, k, pad;
  unsigned long long key;
};

// rules 1-8 of every pixel of the group's n sensor cameras (spix_off[n+1]: their first pixels, N in all) from the
// running minima the resolve left, then the depth and face images (rule 8)
__global__ void k_sensor(const RndCam *cams, const SensorCam *sc, const int *spix_off, int n, int N, const double *best_t,
                         const int *best_f, const long long *pix_off, const float *vtx, const int *faces, const double *T,
                         gpdb_sensor_params sp, int format, void *depth, int *face_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int j = csr_owner(spix_off, n, i);
  const SensorCam &s = sc[j];
  const RndCam &c = cams[s.cam];
  const int p = i - spix_off[j], u = p % c.W, v = p / c.W;
  const long long o = pix_off[s.cam], po = s.proj >= 0 ? pix_off[s.proj] : o;
  double z = 0.0;
  const int f = gpdb_sensor_pixel(&sp, T, s.key, (uint32_t)s.k, u, v, c.W, c.H, c.fx, c.fy, c.cx, c.cy, c.pose,
                                  best_t + o, best_f + o, best_t + po, best_f + po, vtx + 3 * (size_t)c.vbase,
                                  faces + 3 * (size_t)c.fbase, &z);
  bool ret = false;
  const uint32_t raw = f >= 0 ? gpdb_render_raw(z, c.scale, format, &ret) : 0u;
  const long long out = c.pix + p;
  if (format == GPDB_DEPTH_F32) static_cast<uint32_t *>(depth)[out] = raw;
  else static_cast<uint16_t *>(depth)[out] = (uint16_t)raw;
  if (face_out) face_out[out] = ret ? f : -1;
}

// the cameras [first, last) of one group and their sizes
struct RndGroup {
  int first, last;
  long long verts, items, pixels, tiles, pairs_max;  // pairs_max: the most (face, tile) pairs its faces can make
};

size_t rnd_camera_bytes(long long nv, long long nf, long long px, long long tiles) {
  return nv * 3 * sizeof(double) + nf * (GPDB_RENDER_REC * sizeof(double) + sizeof(int4) + sizeof(int)) +
         px * (sizeof(double) + sizeof(int)) + tiles * 2 * sizeof(int);
}

// The scratch of one group, sized for the largest: camera table, offsets, camera-frame vertices, face records, tile
// rectangles and pair counts, the running minimum, the tile counts and positions, the pair total and the lists
struct RndScratch {
  RndCam *cams;
  int *xv_off, *item_off, *tile_off;
  long long *pix_off;
  double *q, *rec, *best_t;
  int4 *rect;
  int *count, *best_f, *tcnt, *tpos, *list;
  unsigned long long *pairs;
  // sensor views only: the table, the group's sensor cameras and their first pixels
  double *table;
  SensorCam *scam;
  int *spix_off;
};

// gpd_b200_sensor.h rule 2's table (GPDB_SENSOR_TABLE doubles, host), built on first use
const double *sensor_table() {
  static const std::vector<double> T = [] {
    std::vector<double> t(GPDB_SENSOR_TABLE);
    gpdb_sensor_table_build(t.data());
    return t;
  }();
  return T.data();
}

// The render of a call (sp null) or of a sensor call (sp given, view b with the key seed + b): camera k of the call is
// entry k * per of the camera table, and with a baseline (per = 2) entry k * per + 1 is its projector
int render_batch(gpdb_ctx *ctx, int B, const int *voff, const int *foff, const float *d_vtx, const int *d_faces,
                 const int *n_cameras, const gpdb_depth_camera *cams, int format, void *d_depth, int *d_face,
                 const gpdb_sensor_params *sp, unsigned long long seed) {
  const int per = sp && sp->baseline > 0.0 ? 2 : 1;
  // the cameras of the call, view by view
  int C = 0;
  for (int b = 0; b < B; b++) C += n_cameras[b];
  std::vector<RndCam> rc((size_t)C * per);
  std::vector<SensorCam> sc((size_t)C);
  long long pix = 0;
  for (int b = 0, k = 0; b < B; b++)
    for (int j = 0; j < n_cameras[b]; j++, k++) {
      const gpdb_depth_camera &D = cams[k];
      sc[k] = SensorCam{0, -1, j, 0, seed + (unsigned long long)b};
      RndCam &c = rc[(size_t)k * per];
      memset(&c, 0, sizeof(c));
      for (int e = 0; e < 12; e++) c.pose[e] = D.pose[e];
      c.fx = D.fx, c.fy = D.fy, c.cx = D.cx, c.cy = D.cy, c.scale = D.depth_scale;
      c.W = D.width, c.H = D.height;
      c.tx = (D.width + RND_TILE - 1) / RND_TILE, c.ty = (D.height + RND_TILE - 1) / RND_TILE;
      c.vbase = voff[b], c.nv = voff[b + 1] - voff[b], c.fbase = foff[b], c.nf = foff[b + 1] - foff[b];
      c.pix = pix;
      pix += (long long)D.width * D.height;
      if (per == 2) {
        RndCam &p = rc[(size_t)k * per + 1];
        p = c;
        gpdb_sensor_projector_pose(c.pose, sp->baseline, p.pose);
        p.pix = -1;  // never written out
      }
    }
  // consecutive cameras (with their projectors), each group's per-camera arrays within RND_GROUP_BYTES (a larger camera
  // is a group of its own)
  std::vector<RndGroup> groups;
  RndGroup cur{0, 0, 0, 0, 0, 0, 0};
  for (int k = 0; k < C * per; k += per) {
    long long nv = 0, nf = 0, px = 0, tl = 0, pm = 0;
    for (int e = k; e < k + per; e++) {
      const RndCam &c = rc[e];
      const long long ct = (long long)c.tx * c.ty;
      nv += c.nv, nf += c.nf, px += (long long)c.W * c.H, tl += ct, pm += (long long)c.nf * ct;
    }
    if (cur.last > cur.first &&
        rnd_camera_bytes(cur.verts + nv, cur.items + nf, cur.pixels + px, cur.tiles + tl) > RND_GROUP_BYTES) {
      groups.push_back(cur);
      cur = RndGroup{k, k, 0, 0, 0, 0, 0};
    }
    cur.last = k + per;
    cur.verts += nv, cur.items += nf, cur.pixels += px, cur.tiles += tl;
    cur.pairs_max += pm;
  }
  groups.push_back(cur);
  long long g_max = 0, v_max = 0, i_max = 0, p_max = 0, t_max = 0, cap = 0;
  for (const RndGroup &G : groups) {
    g_max = std::max(g_max, (long long)(G.last - G.first));
    v_max = std::max(v_max, G.verts), i_max = std::max(i_max, G.items);
    p_max = std::max(p_max, G.pixels), t_max = std::max(t_max, G.tiles);
    cap = std::max(cap, std::min(G.pairs_max, RND_LIST_CAP));
  }
  for (const RndCam &c : rc) cap = std::max(cap, (long long)c.tx * c.ty);  // one face's pairs always fit a chunk
  if (v_max * 3 >= INT_MAX || i_max >= INT_MAX / GPDB_RENDER_REC || t_max >= INT_MAX) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "gpdb_render_depth: a camera of %lld vertices, %lld faces and %lld tiles exceeds "
                   "the int32 ranges of one group", v_max, i_max, t_max);
    return GPDB_ERR_INVALID;
  }
  RndScratch s;
  if (!gpdb_carve(ctx, SCR_RENDER, [&](Carve &c) {
        s.cams = c.take<RndCam>(g_max);
        s.xv_off = c.take<int>(g_max + 1);
        s.item_off = c.take<int>(g_max + 1);
        s.tile_off = c.take<int>(g_max + 1);
        s.pix_off = c.take<long long>(g_max + 1);
        s.q = c.take<double>(3 * v_max);
        s.rec = c.take<double>(GPDB_RENDER_REC * i_max);
        s.rect = c.take<int4>(i_max);
        s.count = c.take<int>(i_max);
        s.best_t = c.take<double>(p_max);
        s.best_f = c.take<int>(p_max);
        s.tcnt = c.take<int>(t_max + 1);
        s.tpos = c.take<int>(t_max + 1);
        s.pairs = c.take<unsigned long long>(1);
        s.list = c.take<int>(cap);
        if (sp) {
          s.table = c.take<double>(GPDB_SENSOR_TABLE);
          s.scam = c.take<SensorCam>(g_max);
          s.spix_off = c.take<int>(g_max + 1);
        }
      }))
    return GPDB_ERR_CUDA;
  if (sp)
    CUDA_TRY(cudaMemcpyAsync(s.table, sensor_table(), sizeof(double) * GPDB_SENSOR_TABLE, cudaMemcpyHostToDevice,
                             ctx->stream));
  const int tb = 256;
  for (const RndGroup &G : groups) {
    const int n = G.last - G.first;
    std::vector<RndCam> gc(rc.begin() + G.first, rc.begin() + G.last);
    std::vector<int> xv((size_t)n + 1, 0), it((size_t)n + 1, 0), tl((size_t)n + 1, 0);
    std::vector<long long> px((size_t)n + 1, 0);
    for (int k = 0; k < n; k++) {
      RndCam &c = gc[k];
      c.xv = xv[k], c.item = it[k], c.tile = tl[k];
      xv[k + 1] = xv[k] + c.nv;
      it[k + 1] = it[k] + c.nf;
      tl[k + 1] = tl[k] + c.tx * c.ty;
      px[k + 1] = px[k] + (long long)c.W * c.H;
    }
    CUDA_TRY(cudaMemcpyAsync(s.cams, gc.data(), sizeof(RndCam) * n, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(s.xv_off, xv.data(), sizeof(int) * (n + 1), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(s.item_off, it.data(), sizeof(int) * (n + 1), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(s.tile_off, tl.data(), sizeof(int) * (n + 1), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(s.pix_off, px.data(), sizeof(long long) * (n + 1), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(s.pairs, 0, sizeof(*s.pairs), ctx->stream));
    const int NV = xv[n], NI = it[n], NT = tl[n];
    if (NV > 0) {
      k_rnd_xform<<<(NV + tb - 1) / tb, tb, 0, ctx->stream>>>(s.cams, s.xv_off, n, NV, d_vtx, s.q);
      LAUNCH_CHECK();
    }
    if (NI > 0) {
      k_rnd_setup<<<(NI + tb - 1) / tb, tb, 0, ctx->stream>>>(s.cams, s.item_off, n, NI, d_faces, s.q, s.rec, s.rect,
                                                             s.count, s.pairs);
      LAUNCH_CHECK();
    }
    unsigned long long pairs = 0;
    CUDA_TRY(cudaMemcpyAsync(&pairs, s.pairs, sizeof(pairs), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    // chunks of consecutive items whose pairs fit the list: one chunk unless the group makes more than `cap` pairs
    std::vector<int> cuts{0};
    if ((long long)pairs > cap) {
      std::vector<int> cnt((size_t)NI);
      CUDA_TRY(cudaMemcpyAsync(cnt.data(), s.count, sizeof(int) * (size_t)NI, cudaMemcpyDeviceToHost, ctx->stream));
      CUDA_TRY(cudaStreamSynchronize(ctx->stream));
      long long run = 0;
      for (int i = 0; i < NI; i++) {
        if (run + cnt[i] > cap) {
          cuts.push_back(i);
          run = 0;
        }
        run += cnt[i];
      }
    }
    cuts.push_back(NI);
    for (size_t ch = 0; ch + 1 < cuts.size(); ch++) {
      const int i0 = cuts[ch], i1 = cuts[ch + 1];
      CUDA_TRY(cudaMemsetAsync(s.tcnt, 0, sizeof(int) * NT, ctx->stream));
      if (i1 > i0) {
        k_rnd_bin<<<(i1 - i0 + tb - 1) / tb, tb, 0, ctx->stream>>>(s.cams, s.item_off, n, i0, i1, s.rect, s.tcnt, nullptr,
                                                                  nullptr, false);
        LAUNCH_CHECK();
      }
      const int rc2 = scan_flags(ctx, s.tcnt, s.tpos, NT);
      if (rc2 != GPDB_OK) return rc2;
      CUDA_TRY(cudaMemsetAsync(s.tcnt, 0, sizeof(int) * NT, ctx->stream));
      if (i1 > i0) {
        k_rnd_bin<<<(i1 - i0 + tb - 1) / tb, tb, 0, ctx->stream>>>(s.cams, s.item_off, n, i0, i1, s.rect, s.tcnt, s.tpos,
                                                                  s.list, true);
        LAUNCH_CHECK();
      }
      // a sensor call keeps the running minimum after the last chunk too: k_sensor reads it
      k_rnd_resolve<<<NT, RND_THREADS, 0, ctx->stream>>>(s.cams, s.tile_off, n, s.rec, s.tpos, s.list, ch == 0,
                                                         !sp && ch + 2 == cuts.size(), s.best_t, s.best_f, s.pix_off,
                                                         format, d_depth, d_face);
      LAUNCH_CHECK();
    }
    if (sp) {
      // the group's cameras (every per-th entry) and their first pixels
      const int ns = n / per;
      std::vector<SensorCam> gs((size_t)ns);
      std::vector<int> sp_off((size_t)ns + 1, 0);
      for (int j = 0; j < ns; j++) {
        gs[j] = sc[(size_t)(G.first / per + j)];
        gs[j].cam = j * per;
        gs[j].proj = per == 2 ? j * per + 1 : -1;
        sp_off[j + 1] = sp_off[j] + gc[j * per].W * gc[j * per].H;
      }
      CUDA_TRY(cudaMemcpyAsync(s.scam, gs.data(), sizeof(SensorCam) * ns, cudaMemcpyHostToDevice, ctx->stream));
      CUDA_TRY(cudaMemcpyAsync(s.spix_off, sp_off.data(), sizeof(int) * (ns + 1), cudaMemcpyHostToDevice, ctx->stream));
      const int N = sp_off[ns];
      k_sensor<<<(N + tb - 1) / tb, tb, 0, ctx->stream>>>(s.cams, s.scam, s.spix_off, ns, N, s.best_t, s.best_f, s.pix_off,
                                                          d_vtx, d_faces, s.table, *sp, format, d_depth, d_face);
      LAUNCH_CHECK();
    }
  }
  return GPDB_OK;
}

// B views (mesh b: vertices voff[b] .. voff[b+1]-1 of d_vtx, faces foff[b] .. foff[b+1]-1 of d_faces, host offsets,
// checked) rendered by their n_cameras[b] cameras cams into d_depth (format) and d_face (may be null), device arrays in the
// layout of gpdb_preprocess_depth.
int render_depth_batch(gpdb_ctx *ctx, int B, const int *voff, const int *foff, const float *d_vtx, const int *d_faces,
                       const int *n_cameras, const gpdb_depth_camera *cams, int format, void *d_depth, int *d_face) {
  return render_batch(ctx, B, voff, foff, d_vtx, d_faces, n_cameras, cams, format, d_depth, d_face, nullptr, 0);
}

// The same seen by the structured-light sensor sp (include/gpd_b200_sensor.h, checked), view b with the key seed + b.
int render_sensor_batch(gpdb_ctx *ctx, int B, const int *voff, const int *foff, const float *d_vtx, const int *d_faces,
                        const int *n_cameras, const gpdb_depth_camera *cams, int format, void *d_depth, int *d_face,
                        const gpdb_sensor_params *sp, unsigned long long seed) {
  return render_batch(ctx, B, voff, foff, d_vtx, d_faces, n_cameras, cams, format, d_depth, d_face, sp, seed);
}

// rule 6's count of every face of the call (mesh b: faces foff[b] .. foff[b+1]-1, vertices from voff[b]); cnt[f] is the
// count clamped to INT_MAX, total[b] (zeroed by the caller) the sum of mesh b's counts each clamped to 2^31, so the
// totals reach 2^31 exactly when the call would hold 2^31 or more points
__global__ void k_mesh_count(const int *voff, const int *foff, int B, int F, const float *vtx, const int *faces,
                             double density, unsigned long long seed, int *cnt, unsigned long long *total) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int b = csr_owner(foff, B, f);
  const float *a = vtx + 3 * ((size_t)voff[b] + faces[3 * (size_t)f]);
  const float *bb = vtx + 3 * ((size_t)voff[b] + faces[3 * (size_t)f + 1]);
  const float *c = vtx + 3 * ((size_t)voff[b] + faces[3 * (size_t)f + 2]);
  double n[3];
  const double L = gpdb_mesh_face(a, bb, c, n);
  const gpdb_u32x4 r = gpdb_mesh_draw(seed + (unsigned long long)b, (uint32_t)(f - foff[b]), 0u);
  const double k = fmin(gpdb_mesh_count(L, density, gpdb_mesh_unit(r.x, r.y)), 2147483648.0);
  cnt[f] = (int)fmin(k, 2147483647.0);
  if (k > 0.0) atomicAdd(total + b, (unsigned long long)k);
}

// the points of the call: point i belongs to the face f with pos[f] <= i < pos[f+1] and is its point i - pos[f]
__global__ void k_mesh_write(const int *voff, const int *foff, int B, int F, const float *vtx, const int *faces,
                             unsigned long long seed, const int *pos, int N, float *xyz, double *nrm, int *face) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int f = csr_owner(pos, F, i);
  const int b = csr_owner(foff, B, f);
  const float *a = vtx + 3 * ((size_t)voff[b] + faces[3 * (size_t)f]);
  const float *bb = vtx + 3 * ((size_t)voff[b] + faces[3 * (size_t)f + 1]);
  const float *c = vtx + 3 * ((size_t)voff[b] + faces[3 * (size_t)f + 2]);
  double n[3], p[3];
  const double L = gpdb_mesh_face(a, bb, c, n);
  const gpdb_u32x4 r = gpdb_mesh_draw(seed + (unsigned long long)b, (uint32_t)(f - foff[b]), (uint32_t)(i - pos[f] + 1));
  gpdb_mesh_point(a, bb, c, gpdb_mesh_unit(r.x, r.y), gpdb_mesh_unit(r.z, r.w), p);
  for (int k = 0; k < 3; k++) xyz[3 * (size_t)i + k] = (float)p[k];
  if (nrm)
    for (int k = 0; k < 3; k++) nrm[3 * (size_t)i + k] = n[k] / L;
  if (face) face[i] = f - foff[b];
}

// the points offsets of the meshes: poff[b] = pos[foff[b]]
__global__ void k_mesh_offsets(const int *pos, const int *foff, int B, int *poff) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b <= B) poff[b] = pos[foff[b]];
}

// SCR_RENDER of a sampling call: the offsets, the counts (scan_flags' flags), their scan and the total
struct MeshScratch {
  int *voff, *foff, *poff, *cnt, *pos;
  unsigned long long *total;
};

bool mesh_carve(gpdb_ctx *ctx, int B, int F, MeshScratch &m) {
  return gpdb_carve(ctx, SCR_RENDER, [&](Carve &c) {
    m.voff = c.take<int>((size_t)B + 1);
    m.foff = c.take<int>((size_t)B + 1);
    m.poff = c.take<int>((size_t)B + 1);
    m.cnt = c.take<int>((size_t)F + 1);
    m.pos = c.take<int>((size_t)F + 1);
    m.total = c.take<unsigned long long>(B);
  });
}

// rule 6's counts of B checked meshes: returns the total (an error when negative) and mesh_n[B] (host) each mesh's
// count (each face's count clamped to 2^31); when the total is below 2^31, poff[B+1] (host) receives the point offsets
// and SCR_RENDER keeps the per-face scan for mesh_write_batch
long long mesh_count_batch(gpdb_ctx *ctx, int B, const int *voff, const int *foff, const float *d_vtx, const int *d_faces,
                           double density, unsigned long long seed, int *poff, long long *mesh_n) {
  const int F = foff[B];
  MeshScratch m;
  if (!mesh_carve(ctx, B, F, m)) return GPDB_ERR_CUDA;
  CUDA_TRY(cudaMemcpyAsync(m.voff, voff, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(m.foff, foff, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemsetAsync(m.total, 0, sizeof(*m.total) * B, ctx->stream));
  if (F > 0) {
    k_mesh_count<<<(F + 255) / 256, 256, 0, ctx->stream>>>(m.voff, m.foff, B, F, d_vtx, d_faces, density, seed, m.cnt,
                                                          m.total);
    LAUNCH_CHECK();
  }
  CUDA_TRY(cudaMemcpyAsync(mesh_n, m.total, sizeof(long long) * B, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  long long total = 0;
  for (int b = 0; b < B; b++) total += mesh_n[b];
  if (total >= (1ll << 31)) return total;  // the caller refuses the call; nothing was scanned
  const int rc = scan_flags(ctx, m.cnt, m.pos, F);
  if (rc != GPDB_OK) return rc;
  k_mesh_offsets<<<(B + 1 + 255) / 256, 256, 0, ctx->stream>>>(m.pos, m.foff, B, m.poff);
  LAUNCH_CHECK();
  CUDA_TRY(cudaMemcpyAsync(poff, m.poff, sizeof(int) * ((size_t)B + 1), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return total;
}

// the N points mesh_count_batch counted (the same meshes and seed): xyz, normals and faces (each but xyz may be null)
int mesh_write_batch(gpdb_ctx *ctx, int B, const int *foff, const float *d_vtx, const int *d_faces, unsigned long long seed,
                     int N, float *d_xyz, double *d_nrm, int *d_face) {
  if (N == 0) return GPDB_OK;
  MeshScratch m;
  if (!mesh_carve(ctx, B, foff[B], m)) return GPDB_ERR_CUDA;  // the slot as mesh_count_batch left it
  k_mesh_write<<<(N + 255) / 256, 256, 0, ctx->stream>>>(m.voff, m.foff, B, foff[B], d_vtx, d_faces, seed, m.pos, N, d_xyz,
                                                        d_nrm, d_face);
  LAUNCH_CHECK();
  return GPDB_OK;
}

// rule 7's mesh checks: position i < V is vertex i (a non-finite coordinate), position V + f is face f (an index
// outside its view's vertices)
__global__ void k_mesh_check(const int *voff, const int *foff, int B, int V, int F, const float *vtx, const int *faces,
                             unsigned long long *first_bad) {
  const long long n = (long long)V + F;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (i < V) {
      if (!isfinite(vtx[3 * i]) || !isfinite(vtx[3 * i + 1]) || !isfinite(vtx[3 * i + 2])) atomicMin(first_bad, i);
      continue;
    }
    const int f = (int)(i - V), b = csr_owner(foff, B, f), nv = voff[b + 1] - voff[b];
    for (int k = 0; k < 3; k++) {
      const int v = faces[3 * (size_t)f + k];
      if (v < 0 || v >= nv) atomicMin(first_bad, (unsigned long long)i);
    }
  }
}

// rule 7's mesh checks (offsets d_voff / d_foff on the device): lowers *d_first_bad to the first vertex i with a
// non-finite coordinate (position i) or face f with an index outside its view's vertices (position V + f)
int mesh_check(gpdb_ctx *ctx, const int *d_voff, const int *d_foff, int B, int V, int F, const float *d_vtx,
               const int *d_faces, unsigned long long *d_first_bad) {
  const long long n = (long long)V + F;
  if (n == 0) return GPDB_OK;
  const long long blocks = std::min((n + 255) / 256, (long long)ctx->sm_count * 16);
  k_mesh_check<<<(int)blocks, 256, 0, ctx->stream>>>(d_voff, d_foff, B, V, F, d_vtx, d_faces, d_first_bad);
  LAUNCH_CHECK();
  return GPDB_OK;
}

}  // namespace

// ---- entry points: argument checks, host-twin uploads and the C-ABI calls -------------------------------------------

// the offsets of B meshes (rule 7): vertex_offsets and face_offsets start at 0 and never decrease, and the arrays they
// address are given; `unit` names a mesh in the messages
static int check_mesh_args(gpdb_ctx *ctx, const char *name, const char *unit, int32_t B, const int32_t *voff,
                           const float *vertices, const int32_t *foff, const int32_t *faces) {
  int rc = gpdb_check_offsets(ctx, name, "vertex_offsets", voff, B, unit);
  if (rc == GPDB_OK) rc = gpdb_check_offsets(ctx, name, "face_offsets", foff, B, unit);
  if (rc != GPDB_OK) return rc;
  if ((voff[B] > 0 && !vertices) || (foff[B] > 0 && !faces)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: null vertices or faces for %d vertices and %d faces", name, voff[B], foff[B]);
    return GPDB_ERR_INVALID;
  }
  return GPDB_OK;
}

// rule 7's device checks of B meshes in device memory: a non-finite vertex or a face index outside its mesh's vertices,
// the first of them named
static int check_meshes(gpdb_ctx *ctx, const char *name, const char *unit, int B, const int32_t *voff, const int32_t *foff,
                        const float *d_vtx, const int32_t *d_faces) {
  const int V = voff[B], F = foff[B];
  const size_t bytes = sizeof(int) * 2 * ((size_t)B + 1);
  unsigned long long bad;
  const int rc = first_bad(ctx, bytes, &bad, [&](unsigned long long *d_bad, void *d) -> int {
    int *d_voff = (int *)d, *d_foff = d_voff + B + 1;
    CUDA_TRY(cudaMemcpyAsync(d_voff, voff, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(d_foff, foff, sizeof(int) * ((size_t)B + 1), cudaMemcpyHostToDevice, ctx->stream));
    return mesh_check(ctx, d_voff, d_foff, B, V, F, d_vtx, d_faces, d_bad);
  });
  if (rc != GPDB_OK || bad == NO_BAD) return rc;
  int b = 0;
  if (bad < (unsigned long long)V) {
    while (voff[b + 1] <= (long long)bad) b++;
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: %s %d: vertex %d has a non-finite coordinate", name, unit, b,
                   (int)(bad - voff[b]));
    return GPDB_ERR_INVALID;
  }
  const int f = (int)(bad - V);
  while (foff[b + 1] <= f) b++;
  int32_t tri[3];
  CUDA_TRY(cudaMemcpyAsync(tri, d_faces + 3 * (size_t)f, sizeof(tri), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: %s %d: face %d = (%d, %d, %d) indexes outside its %d vertices", name, unit, b,
                 f - foff[b], tri[0], tri[1], tri[2], voff[b + 1] - voff[b]);
  return GPDB_ERR_INVALID;
}

// gpd_b200_sensor.h rule 9's parameter checks
static int check_sensor_params(gpdb_ctx *ctx, const char *name, const gpdb_sensor_params *sp) {
  if (!sp) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need sensor (gpdb_sensor_params_default for a clean render)", name);
    return GPDB_ERR_INVALID;
  }
  const struct {
    const char *name;
    double v;
  } f[] = {{"baseline", sp->baseline},
           {"lateral_sigma", sp->lateral_sigma},
           {"disparity_sigma", sp->disparity_sigma},
           {"disparity_step", sp->disparity_step},
           {"min_cos_incidence", sp->min_cos_incidence},
           {"shadow_tolerance", sp->shadow_tolerance},
           {"dropout", sp->dropout}};
  const char *bad = nullptr;
  for (const auto &e : f)
    if (!(e.v >= 0.0) || !std::isfinite(e.v)) {
      gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: sensor: %s must be finite and >= 0 (got %g)", name, e.name, e.v);
      return GPDB_ERR_INVALID;
    }
  if (sp->dropout > 1.0) bad = "dropout must lie in [0, 1]";
  else if (sp->shadow_tolerance >= 1.0) bad = "shadow_tolerance must be < 1";
  else if (sp->min_cos_incidence > 1.0) bad = "min_cos_incidence must be <= 1";
  else if ((sp->disparity_sigma > 0.0 || sp->disparity_step > 0.0) && !(sp->baseline > 0.0))
    bad = "disparity_sigma and disparity_step need a baseline > 0";
  if (bad) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: sensor: %s", name, bad);
    return GPDB_ERR_INVALID;
  }
  return GPDB_OK;
}

// gpdb_render_depth[_device] and (sensor) gpdb_render_sensor_depth[_device]: the checks, then the device render (the host
// twin uploads the meshes into SCR_UPLOAD, renders into it and copies the images back). Nothing installed changes.
static int render_entry(gpdb_ctx *ctx, const char *name, int32_t B, const int32_t *voff, const float *vertices,
                        const int32_t *foff, const int32_t *faces, const int32_t *n_cameras, const gpdb_depth_camera *cams,
                        int32_t format, void *depth_out, int32_t *face_out, bool device, bool sensor = false,
                        const gpdb_sensor_params *sp = nullptr, uint64_t seed = 0) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (B <= 0 || !n_cameras || !cams || !depth_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need n_views > 0, n_cameras, cameras, depth_out", name);
    return GPDB_ERR_INVALID;
  }
  if (check_depth_format(ctx, name, format) != GPDB_OK) return GPDB_ERR_INVALID;
  if (sensor && check_sensor_params(ctx, name, sp) != GPDB_OK) return GPDB_ERR_INVALID;
  std::vector<int> roff;
  int rc = check_mesh_args(ctx, name, "view", B, voff, vertices, foff, faces);
  if (rc == GPDB_OK) rc = check_depth_cameras(ctx, name, B, n_cameras, cams, roff);
  if (rc == GPDB_OK && device)
    rc = gpdb_check_device_ptrs(ctx, name, {{"d_vertices", vertices}, {"d_faces", faces}, {"d_depth_out", depth_out},
                                            {"d_face_out", face_out}});
  if (rc != GPDB_OK) return rc;
  CUDA_TRY(cudaSetDevice(ctx->device));
  const size_t V = (size_t)voff[B], F = (size_t)foff[B], M = (size_t)roff[B];
  const size_t elt = format == GPDB_DEPTH_U16 ? sizeof(uint16_t) : sizeof(float);
  const float *d_vtx = vertices;
  const int32_t *d_faces = faces;
  void *d_depth = depth_out;
  int32_t *d_face = face_out;
  if (!device) {
    float *v;
    int32_t *f;
    unsigned char *dd;
    if (!gpdb_carve(ctx, SCR_UPLOAD, [&](Carve &c) {
          v = c.take<float>(3 * V);
          f = c.take<int32_t>(3 * F);
          dd = c.take<unsigned char>(elt * M, 16);
          d_face = face_out ? c.take<int32_t>(M) : nullptr;
        }))
      return GPDB_ERR_CUDA;
    if (V) CUDA_TRY(cudaMemcpyAsync(v, vertices, sizeof(float) * 3 * V, cudaMemcpyHostToDevice, ctx->stream));
    if (F) CUDA_TRY(cudaMemcpyAsync(f, faces, sizeof(int32_t) * 3 * F, cudaMemcpyHostToDevice, ctx->stream));
    d_vtx = v, d_faces = f, d_depth = dd;
  }
  if ((rc = check_meshes(ctx, name, "view", B, voff, foff, d_vtx, d_faces)) != GPDB_OK) return rc;
  rc = sensor ? render_sensor_batch(ctx, B, voff, foff, d_vtx, d_faces, n_cameras, cams, format, d_depth, d_face, sp, seed)
              : render_depth_batch(ctx, B, voff, foff, d_vtx, d_faces, n_cameras, cams, format, d_depth, d_face);
  if (rc != GPDB_OK) return rc;
  if (!device) {
    CUDA_TRY(cudaMemcpyAsync(depth_out, d_depth, elt * M, cudaMemcpyDeviceToHost, ctx->stream));
    if (face_out) CUDA_TRY(cudaMemcpyAsync(face_out, d_face, sizeof(int32_t) * M, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  }
  return B;
}

// gpdb_sample_meshes[_device]: the checks, the count, then (xyz_out given) the points. The host twin uploads the meshes
// into SCR_UPLOAD, and once the count is known carves the outputs behind them there (uploading again: a grown slot
// starts empty). Nothing installed changes.
static int sample_entry(gpdb_ctx *ctx, const char *name, int32_t B, const int32_t *voff, const float *vertices,
                        const int32_t *foff, const int32_t *faces, double density, uint64_t seed, int32_t *poff_out,
                        float *xyz_out, double *normals_out, int32_t *face_out, bool device) {
  if (!ctx) return GPDB_ERR_INVALID;
  if (B <= 0 || !poff_out) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: need n_meshes > 0 and point_offsets_out", name);
    return GPDB_ERR_INVALID;
  }
  if (!(density > 0.0) || !std::isfinite(density)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: density must be finite and > 0 (got %g)", name, density);
    return GPDB_ERR_INVALID;
  }
  int rc = check_mesh_args(ctx, name, "mesh", B, voff, vertices, foff, faces);
  if (rc == GPDB_OK && device)
    rc = gpdb_check_device_ptrs(ctx, name, {{"d_vertices", vertices}, {"d_faces", faces}, {"d_xyz_out", xyz_out},
                                            {"d_normals_out", normals_out}, {"d_face_out", face_out}});
  if (rc != GPDB_OK) return rc;
  CUDA_TRY(cudaSetDevice(ctx->device));
  const size_t V = (size_t)voff[B], F = (size_t)foff[B];
  const float *d_vtx = vertices;
  const int32_t *d_faces = faces;
  float *d_xyz = xyz_out;
  double *d_nrm = normals_out;
  int32_t *d_face = face_out;
  // the host twin's buffers: the meshes, then n points of the outputs the caller asked for
  auto upload = [&](size_t n) -> int {
    float *v;
    int32_t *f;
    if (!gpdb_carve(ctx, SCR_UPLOAD, [&](Carve &c) {
          v = c.take<float>(3 * V);
          f = c.take<int32_t>(3 * F);
          d_xyz = c.take<float>(3 * n);
          d_nrm = normals_out ? c.take<double>(3 * n) : nullptr;
          d_face = face_out ? c.take<int32_t>(n) : nullptr;
        }))
      return GPDB_ERR_CUDA;
    if (V) CUDA_TRY(cudaMemcpyAsync(v, vertices, sizeof(float) * 3 * V, cudaMemcpyHostToDevice, ctx->stream));
    if (F) CUDA_TRY(cudaMemcpyAsync(f, faces, sizeof(int32_t) * 3 * F, cudaMemcpyHostToDevice, ctx->stream));
    d_vtx = v, d_faces = f;
    return GPDB_OK;
  };
  if (!device && (rc = upload(0)) != GPDB_OK) return rc;
  if ((rc = check_meshes(ctx, name, "mesh", B, voff, foff, d_vtx, d_faces)) != GPDB_OK) return rc;
  std::vector<int> poff((size_t)B + 1);
  std::vector<long long> mesh_n((size_t)B);
  const long long n = mesh_count_batch(ctx, B, voff, foff, d_vtx, d_faces, density, seed, poff.data(), mesh_n.data());
  if (n < 0) return (int)n;
  if (n >= (1ll << 31)) {
    long long run = 0;
    int b = 0;
    while ((run += mesh_n[b]) < (1ll << 31)) b++;
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s: mesh %d: the call reaches 2^31 or more sampled points (lower the density)",
                   name, b);
    return GPDB_ERR_INVALID;
  }
  if (xyz_out && n > 0) {
    if (!device && (rc = upload((size_t)n)) != GPDB_OK) return rc;
    if ((rc = mesh_write_batch(ctx, B, foff, d_vtx, d_faces, seed, (int)n, d_xyz, d_nrm, d_face)) != GPDB_OK) return rc;
    if (!device) {
      CUDA_TRY(cudaMemcpyAsync(xyz_out, d_xyz, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, ctx->stream));
      if (normals_out)
        CUDA_TRY(cudaMemcpyAsync(normals_out, d_nrm, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, ctx->stream));
      if (face_out) CUDA_TRY(cudaMemcpyAsync(face_out, d_face, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
      CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    }
  }
  memcpy(poff_out, poff.data(), sizeof(int32_t) * ((size_t)B + 1));
  return (int)n;
}

extern "C" {

int gpdb_render_depth(gpdb_ctx *ctx, int32_t n_views, const int32_t *vertex_offsets, const float *vertices,
                      const int32_t *face_offsets, const int32_t *faces, const int32_t *n_cameras,
                      const gpdb_depth_camera *cameras, int32_t depth_format, void *depth_out, int32_t *face_out) {
  return render_entry(ctx, "gpdb_render_depth", n_views, vertex_offsets, vertices, face_offsets, faces, n_cameras, cameras,
                      depth_format, depth_out, face_out, false);
}

int gpdb_render_depth_device(gpdb_ctx *ctx, int32_t n_views, const int32_t *vertex_offsets, const float *d_vertices,
                             const int32_t *face_offsets, const int32_t *d_faces, const int32_t *n_cameras,
                             const gpdb_depth_camera *cameras, int32_t depth_format, void *d_depth_out,
                             int32_t *d_face_out) {
  return render_entry(ctx, "gpdb_render_depth_device", n_views, vertex_offsets, d_vertices, face_offsets, d_faces, n_cameras,
                      cameras, depth_format, d_depth_out, d_face_out, true);
}

void gpdb_sensor_params_default(gpdb_sensor_params *p) {
  if (p) memset(p, 0, sizeof(*p));
}

int gpdb_render_sensor_depth(gpdb_ctx *ctx, int32_t n_views, const int32_t *vertex_offsets, const float *vertices,
                             const int32_t *face_offsets, const int32_t *faces, const int32_t *n_cameras,
                             const gpdb_depth_camera *cameras, int32_t depth_format, void *depth_out, int32_t *face_out,
                             const gpdb_sensor_params *sensor, uint64_t seed) {
  return render_entry(ctx, "gpdb_render_sensor_depth", n_views, vertex_offsets, vertices, face_offsets, faces, n_cameras,
                      cameras, depth_format, depth_out, face_out, false, true, sensor, seed);
}

int gpdb_render_sensor_depth_device(gpdb_ctx *ctx, int32_t n_views, const int32_t *vertex_offsets, const float *d_vertices,
                                    const int32_t *face_offsets, const int32_t *d_faces, const int32_t *n_cameras,
                                    const gpdb_depth_camera *cameras, int32_t depth_format, void *d_depth_out,
                                    int32_t *d_face_out, const gpdb_sensor_params *sensor, uint64_t seed) {
  return render_entry(ctx, "gpdb_render_sensor_depth_device", n_views, vertex_offsets, d_vertices, face_offsets, d_faces,
                      n_cameras, cameras, depth_format, d_depth_out, d_face_out, true, true, sensor, seed);
}

int gpdb_debug_sensor_table(double *table_out) {
  if (!table_out) return GPDB_ERR_INVALID;
  memcpy(table_out, sensor_table(), sizeof(double) * GPDB_SENSOR_TABLE);
  return GPDB_SENSOR_TABLE;
}

int gpdb_sample_meshes(gpdb_ctx *ctx, int32_t n_meshes, const int32_t *vertex_offsets, const float *vertices,
                       const int32_t *face_offsets, const int32_t *faces, double density, uint64_t seed,
                       int32_t *point_offsets_out, float *xyz_out, double *normals_out, int32_t *face_out) {
  return sample_entry(ctx, "gpdb_sample_meshes", n_meshes, vertex_offsets, vertices, face_offsets, faces, density, seed,
                      point_offsets_out, xyz_out, normals_out, face_out, false);
}

int gpdb_sample_meshes_device(gpdb_ctx *ctx, int32_t n_meshes, const int32_t *vertex_offsets, const float *d_vertices,
                              const int32_t *face_offsets, const int32_t *d_faces, double density, uint64_t seed,
                              int32_t *point_offsets_out, float *d_xyz_out, double *d_normals_out, int32_t *d_face_out) {
  return sample_entry(ctx, "gpdb_sample_meshes_device", n_meshes, vertex_offsets, d_vertices, face_offsets, d_faces, density,
                      seed, point_offsets_out, d_xyz_out, d_normals_out, d_face_out, true);
}

}  // extern "C"
