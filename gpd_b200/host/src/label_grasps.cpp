// label_grasps CONFIG_FILE PCD_FILE MESH_FILE — the reference's labelling program (src/label_grasps.cpp) over the GPU
// path, without its two plots: the candidates of a camera view, labelled against a ground-truth cloud (e.g. points
// sampled from the object's mesh) of the same object or scene.
//
// The view: filterWorkspace, voxelizeCloud(0.003), calculateNormals(normals_radius) in one gpdb_preprocess call; the
// normals times -1; sampleAbovePlane when the cfg's sample_above_plane is set (default 1); subsample(num_samples).
// The mesh: calculateNormals alone (gpdb_preprocess with voxelize = 0 and an unbounded workspace), the normals times -1.
// Then GraspDetector::createGraspImages on the view and GraspDetector::evalGroundTruth against the mesh, and the
// reference's `labels: N` / `(i) label: l` lines (a full antipodal hand's line twice, as upstream prints it).
//
// Departures from the reference:
//  - NaN points of either cloud are dropped by the device preprocessing; the reference keeps them in the mesh, where
//    PCL's normal estimation gives them NaN normals and no radius search finds them.
//  - num_threads is read and printed but unused: the normals are estimated on the GPU.
//  - Cloud::subsample and sampleAbovePlane draw with the shim's fixed-seed generators (util::Cloud in gpd.h), so a run
//    can be reproduced; the reference seeds from the clock.
//  - The plots (plotAntipodalHands, plotValidHands) are not drawn.
#include <cmath>
#include <cstdio>
#include <fstream>
#include <iostream>

#include "gpd/gpd.h"

using namespace gpd;

static bool checkFileExists(const std::string &file_name) {
  std::ifstream file(file_name.c_str());
  if (!file) {
    std::cout << "File " + file_name + " could not be found!\n";
    return false;
  }
  return true;
}

// gpdb_preprocess of `cloud` (raw points, one camera) on ctx with pp; the processed points, with their normals times -1,
// replace the cloud's (cloud.setNormals(cloud.getNormals() * (-1.0))). Returns false after printing the error.
static bool preprocess_flipped(gpdb_ctx *ctx, util::Cloud &cloud, const gpdb_preprocess_params &pp) {
  const int n = gpdb_preprocess(ctx, cloud.getPoints().data(), nullptr, nullptr, (int)cloud.size(), cloud.getViewPoints().data(),
                                cloud.numCameras(), &pp);
  if (n < 0) {
    printf("ERROR: %s\n", gpdb_last_error(ctx));
    return false;
  }
  double ms[6];
  gpdb_preprocess_timings(ctx, ms);
  if (pp.voxelize) printf("Voxelized cloud: %d\n", n);
  printf("Calculated %d surface normals in %3.4fs (mode: GPU).\n", n, ms[4] * 1e-3);
  std::vector<float> xyz(3 * (size_t)n);
  std::vector<double> nrm(3 * (size_t)n);
  std::vector<int> cam((size_t)n * cloud.numCameras());
  if (n > 0 && gpdb_get_cloud(ctx, xyz.data(), nrm.data(), cam.data()) < 0) {
    printf("ERROR: %s\n", gpdb_last_error(ctx));
    return false;
  }
  for (double &v : nrm) v = -v;
  cloud.setProcessed(std::move(xyz), std::move(nrm), std::move(cam));
  return true;
}

int main(int argc, char *argv[]) {
  if (argc < 4) {
    std::cout << "Error: Not enough input arguments!\n\n";
    std::cout << "Usage: label_grasps CONFIG_FILE PCD_FILE MESH_FILE\n\n";
    std::cout << "Find grasp poses for a point cloud, PCD_FILE (*.pcd), "
                 "using parameters from CONFIG_FILE (*.cfg), and check them "
                 "against a mesh, MESH_FILE (*.pcd).\n\n";
    return -1;
  }
  const std::string config_filename = argv[1], pcd_filename = argv[2], mesh_filename = argv[3];
  if (!checkFileExists(config_filename)) {
    printf("Error: CONFIG_FILE not found!\n");
    return -1;
  }
  if (!checkFileExists(pcd_filename)) {
    printf("Error: PCD_FILE not found!\n");
    return -1;
  }
  if (!checkFileExists(mesh_filename)) {
    printf("Error: MESH_FILE not found!\n");
    return -1;
  }

  const double VOXEL_SIZE = 0.003;
  util::ConfigFile config_file(config_filename);
  config_file.ExtractKeys();
  const std::vector<double> workspace = config_file.getValueOfKeyAsStdVectorDouble("workspace", "-1 1 -1 1 -1 1");
  const int num_threads = config_file.getValueOfKey<int>("num_threads", 1);
  const int num_samples = config_file.getValueOfKey<int>("num_samples", 100);
  const bool sample_above_plane = config_file.getValueOfKey<int>("sample_above_plane", 1);
  const double normals_radius = config_file.getValueOfKey<double>("normals_radius", 0.03);
  printf("num_threads: %d, num_samples: %d\n", num_threads, num_samples);
  printf("sample_above_plane: %d\n", sample_above_plane);
  printf("normals_radius: %.3f\n", normals_radius);

  const std::vector<double> view_points = {0.0, 0.0, 0.0};  // one camera at the origin
  util::Cloud cloud(pcd_filename, view_points);
  if (cloud.size() == 0) {
    std::cout << "Error: Input point cloud is empty or does not exist!\n";
    return -1;
  }
  util::Cloud mesh(mesh_filename, view_points);
  if (mesh.size() == 0) {
    std::cout << "Error: Mesh point cloud is empty or does not exist!\n";
    return -1;
  }

  gpdb_params params;
  gpdb_params_default(&params);
  gpdb_ctx *ctx = nullptr;
  if (gpdb_create(&params, &ctx) != GPDB_OK) {
    printf("ERROR: %s\n", gpdb_last_error(nullptr));
    return -1;
  }
  gpdb_preprocess_params pp;
  gpdb_preprocess_params_default(&pp);
  pp.estimate_normals = 1;
  pp.normals_radius = normals_radius;

  // Prepare the point cloud.
  pp.voxelize = 1;
  pp.voxel_size = VOXEL_SIZE;
  for (size_t i = 0; i < 6 && i < workspace.size(); i++) pp.workspace[i] = workspace[i];
  bool ok = preprocess_flipped(ctx, cloud, pp);
  if (ok && sample_above_plane && cloud.size() > 0) ok = cloud.sampleAbovePlane(ctx);  // the plane fit reads the points alone
  if (ok) cloud.subsample(num_samples);

  // Prepare the mesh.
  pp.voxelize = 0;
  for (int i = 0; i < 6; i++) pp.workspace[i] = i % 2 ? INFINITY : -INFINITY;
  ok = ok && preprocess_flipped(ctx, mesh, pp);
  gpdb_destroy(ctx);
  if (!ok) return -1;

  // Detect grasp poses.
  std::vector<std::unique_ptr<candidate::Hand>> hands;
  std::vector<std::vector<uint8_t>> images;
  GraspDetector detector(config_filename);
  detector.createGraspImages(cloud, hands, images);

  const std::vector<int> labels = detector.evalGroundTruth(mesh, hands);
  printf("labels: %zu\n", labels.size());
  for (size_t i = 0; i < hands.size(); i++) {
    printf("(%zu) label: %d\n", i, labels[i]);
    if (hands[i]->isFullAntipodal()) printf("(%zu) label: %d\n", i, labels[i]);
  }
  return 0;
}
