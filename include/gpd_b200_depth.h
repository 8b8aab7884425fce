/*
 * gpd_b200_depth.h — SPECIFICATION of the depth-image front of preprocessing (gpdb_preprocess_depth[_device]) and of
 * Cloud::subsample on the device (gpdb_subsample_clouds[_device]); the entry points are declared in gpd_b200.h.
 *
 * Sensors and simulators hand out depth images, not clouds. gpdb_preprocess_depth back-projects the K_b pinhole cameras of
 * every view, fuses them into the view's raw cloud (the reference's multi-camera Cloud constructor, cloud.cpp:120-152,
 * generalised to K cameras) and preprocesses that cloud as gpdb_preprocess_clouds does, without ever materialising the raw
 * cloud: back-projection is fused into the NaN / workspace filter, so only filtered points take memory.
 *
 *  1. Camera. gpdb_depth_camera below. Pixel (u, v) is column u, row v of a height x width row-major image, with no
 *     half-pixel offset. One depth format per call (GPDB_DEPTH_U16 or GPDB_DEPTH_F32).
 *  2. Arithmetic. Every operation is rounded on its own, with no FMA:
 *        z  = (float)raw * (float)depth_scale                         float32 (F32: raw is the stored float)
 *        valid iff the pixel has a return (U16: raw != 0; F32: raw finite and > 0) and min_depth <= (double)z <= max_depth
 *        xc = (((float)u - (float)cx) * z) / (float)fx                float32
 *        yc = (((float)v - (float)cy) * z) / (float)fy                float32
 *        zc = z
 *        x  = (float)(((R00 * (double)xc + R01 * (double)yc) + R02 * (double)zc) + t0)   float64, one final rounding;
 *        likewise y (row 1) and z (row 2) of pose = [R | t] (camera to world, row-major 3 x 4).
 *     R is not checked for orthonormality: any finite 3 x 3 matrix is applied as given.
 *  3. Raw cloud of view b (K_b = 1..8 cameras). Its raw points are the pixels of camera 0 in row-major order, then those
 *     of camera 1, and so on: raw point i of the view is pixel i of the concatenation. An invalid pixel stays in that
 *     numbering as a NaN point. cam_source is one-hot (the camera the pixel came from), view point k is t of camera k,
 *     and normals are estimated (estimate_normals must be 1). So the src_out of gpdb_get_clouds decodes to
 *     (camera, v, u), and a per-pixel mask lines up with the raw points.
 *  4. Equivalence. gpdb_preprocess_depth[_device] installs exactly what gpdb_preprocess_clouds[_device] installs from that
 *     raw cloud, bit for bit: offsets, xyz, normals, camera sources and source indices. Dropping an invalid pixel is
 *     removeNans (cloud.cpp:154-164) on its NaN point.
 *  5. Sampling (Cloud::subsample, cloud.cpp:350-370). The eligible points of installed cloud b are all of its points, or,
 *     given a mask (one byte per raw point of the last preprocessing call, concatenated by view), those whose source raw
 *     point has a nonzero mask byte. Cloud-local point j gets the 64-bit key (c.x << 32) | c.y with
 *     c = gpdb_philox4x32_10({j, 0, 2, 0}, key), key = seed + b split into (low word, high word) as in gpd_b200_sis.h;
 *     stream word 2 keeps these draws apart from the SIS streams 0 and 1. The cloud takes the min(num_samples,
 *     |eligible|) eligible points with the smallest (key, j), in ascending j (pcl::RandomSample's selection sampling
 *     also returns ascending indices, without replacement); num_samples = 0 takes every eligible point (the reference's
 *     "no subsampling", cloud.cpp:351-353). A cloud's draw depends only on (seed + b, its points, its mask).
 *
 * tests/depth_reference.py restates this file in numpy.
 */
#ifndef GPD_B200_DEPTH_H_
#define GPD_B200_DEPTH_H_

#include <stdint.h>

#include "gpd_b200.h"     /* the typedef of gpdb_depth_camera, the entry points */
#include "gpd_b200_sis.h" /* gpdb_philox4x32_10, GPDB_HD */

struct gpdb_depth_camera {
  int32_t width, height;       /* pixels; the image is height x width, row-major, contiguous                           */
  double fx, fy, cx, cy;       /* pinhole intrinsics in pixels (sensor_msgs/CameraInfo K)                              */
  double pose[12];             /* camera-to-world [R | t], row-major 3 x 4; optical frame x right, y down, z forward  */
  double depth_scale;          /* metres per stored unit: 0.001 for 16UC1 millimetres, 1.0 for 32FC1 metres          */
  double min_depth, max_depth; /* a pixel is valid iff min_depth <= z <= max_depth (metres; max may be +inf)           */
};

#define GPDB_DEPTH_U16 0 /* uint16, 0 = no return                    */
#define GPDB_DEPTH_F32 1 /* float32, non-finite or <= 0 = no return  */

/* the stream word of the subsample draws (gpd_b200_sis.h uses 0 and 1) */
#define GPDB_SUBSAMPLE_STREAM 2u

/* the 64-bit sampling key of cloud-local point j of the cloud whose key is seed + b */
GPDB_HD uint64_t gpdb_subsample_key(uint64_t key, uint32_t j) {
  const gpdb_u32x4 c = {j, 0u, GPDB_SUBSAMPLE_STREAM, 0u};
  const gpdb_u32x4 r = gpdb_philox4x32_10(c, (uint32_t)key, (uint32_t)(key >> 32));
  return ((uint64_t)r.x << 32) | r.y;
}

#endif /* GPD_B200_DEPTH_H_ */
