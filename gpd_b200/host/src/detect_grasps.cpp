// detect_grasps CONFIG_FILE PCD_FILE [NORMALS_FILE] — the reference's command line (src/detect_grasps.cpp:20-94) over
// the GPU path. A cloud without normals is preprocessed on the device (workspace filter, voxelisation, normal
// estimation: GraspDetector::preprocessPointCloud -> gpdb_preprocess); normals given as PCD fields or as a
// NORMALS_FILE are kept.
// --dump-config prints the parsed parameters as JSON and exits (used by the CPU tests).
// --sis [SEED]  runs the reference's other entry point over the same path, cem_detect_grasps
//               (src/cem_detect_grasps.cpp:14-66 -> SequentialImportanceSampling::detectGrasps), and prints the evaluated
//               sample positions (SIS_SAMPLE lines) so that a test can recompute the result independently.
// --gpus N      shards the samples over N GPUs inside libgpd_b200 (GraspDetector::detectGraspsMultiGpu).
// --batch PCD_FILE...  runs every PCD file as one cloud of a batch (one device pass per step for all of them, with or
//               without --sis; cloud b seeds its sampler with SEED + b) and prints, per file, a line `CLOUD b PCD_FILE`
//               followed by the result lines a run on that file alone prints.
#include <cstdio>
#include <cstdlib>
#include <cstring>
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

static void print_grasps(const std::vector<std::unique_ptr<candidate::Hand>> &grasps) {
  for (size_t i = 0; i < grasps.size() && i < 5; i++) {
    printf("--- grasp %zu ---\n", i);
    grasps[i]->print();
  }
  printf("RESULT n_grasps=%zu best_score=%.6f\n", grasps.size(), grasps.empty() ? 0.0 : grasps[0]->getScore());
}

static void print_sis(const std::vector<std::unique_ptr<candidate::Hand>> &grasps, const std::vector<double> &kept,
                      const std::vector<double> &evaluated) {
  for (size_t i = 0; i + 2 < kept.size(); i += 3) printf("SIS_SAMPLE %.17g %.17g %.17g\n", kept[i], kept[i + 1], kept[i + 2]);
  for (size_t i = 0; i < grasps.size(); i++)
    printf("SIS_GRASP %.9g %.17g %.17g %.17g\n", grasps[i]->getScore(), grasps[i]->getPosition()[0], grasps[i]->getPosition()[1],
           grasps[i]->getPosition()[2]);
  printf("RESULT n_grasps=%zu evaluated=%zu hand_sets=%zu\n", grasps.size(), evaluated.size() / 3, kept.size() / 3);
}

// --batch: every PCD file one cloud of a batch
static int run_batch(const std::string &config_filename, const std::vector<std::string> &files, bool sis, unsigned sis_seed) {
  for (const std::string &f : files)
    if (!checkFileExists(f)) return -1;
  util::ConfigFile config_file(config_filename);
  config_file.ExtractKeys();
  if (config_file.getValueOfKey<bool>("centered_at_origin", false)) {
    std::cout << "Error: --batch does not support centered_at_origin\n";
    return -1;
  }
  std::vector<double> camera_position = config_file.getValueOfKeyAsStdVectorDouble("camera_position", "0.0 0.0 0.0");
  std::vector<util::Cloud> clouds;
  for (const std::string &f : files) {
    clouds.emplace_back(f, camera_position);
    if (clouds.back().size() == 0) {
      std::cout << "Error: Input point cloud " << f << " is empty or does not exist!\n";
      return -1;
    }
  }
  std::vector<std::vector<std::unique_ptr<candidate::Hand>>> grasps;
  std::unique_ptr<SequentialImportanceSampling> sampler;
  std::unique_ptr<GraspDetector> detector;
  if (sis) {
    sampler = std::make_unique<SequentialImportanceSampling>(config_filename);
    sampler->setSeed(sis_seed);
    if (!sampler->detector().preprocessPointClouds(clouds)) return -1;
    grasps = sampler->detectGrasps(clouds);
  } else {
    detector = std::make_unique<GraspDetector>(config_filename);
    if (!detector->preprocessPointClouds(clouds)) return -1;
    grasps = detector->detectGrasps(clouds);
  }
  for (size_t b = 0; b < files.size(); b++) {
    printf("CLOUD %zu %s\n", b, files[b].c_str());
    if (sis) print_sis(grasps[b], sampler->batchHandSetPositions()[b], sampler->batchEvaluatedPositions()[b]);
    else print_grasps(grasps[b]);
  }
  return 0;
}

int main(int argc, char *argv[]) {
  bool dump = false, sis = false, batch = false;
  unsigned sis_seed = 1;
  int gpus = 1;
  std::vector<std::string> args;
  for (int i = 1; i < argc; i++) {
    if (std::strcmp(argv[i], "--dump-config") == 0) dump = true;
    else if (std::strcmp(argv[i], "--batch") == 0) batch = true;
    else if (std::strcmp(argv[i], "--sis") == 0) {
      sis = true;
      if (i + 1 < argc && argv[i + 1][0] >= '0' && argv[i + 1][0] <= '9') sis_seed = (unsigned)std::atoi(argv[++i]);
    } else if (std::strcmp(argv[i], "--gpus") == 0 && i + 1 < argc) gpus = std::atoi(argv[++i]);
    else args.push_back(argv[i]);
  }
  if (args.size() < (dump ? 1u : 2u)) {
    std::cout << "Error: Not enough input arguments!\n\nUsage: detect_grasps CONFIG_FILE PCD_FILE [NORMALS_FILE]\n\n"
                 "Detect grasp poses for a processed point cloud, PCD_FILE (*.pcd), using parameters from CONFIG_FILE (*.cfg).\n\n"
                 "[NORMALS_FILE] (optional) contains a surface normal for each point in the cloud (*.csv).\n";
    return -1;
  }
  const std::string config_filename = args[0];
  if (!checkFileExists(config_filename)) return -1;
  if (dump) {
    gpdb_params p;
    std::string weights;
    int num_selected, num_samples, min_inliers;
    if (!paramsFromConfig(config_filename, p, weights, num_selected, num_samples, min_inliers)) return -1;
    util::Cloud cloud;
    if (args.size() >= 2) cloud = util::Cloud(args[1], {0.0, 0.0, 0.0});
    gpdb_preprocess_params pp;
    preprocessParamsFromConfig(config_filename, pp);
    printf("{\"voxelize\": %d, \"voxel_size\": %.17g, \"normals_radius\": %.17g, \"workspace\": [%.17g, %.17g, %.17g, %.17g, %.17g, %.17g], ",
           pp.voxelize, pp.voxel_size, pp.normals_radius, pp.workspace[0], pp.workspace[1], pp.workspace[2], pp.workspace[3],
           pp.workspace[4], pp.workspace[5]);
    printf("\"finger_width\": %.17g, \"hand_outer_diameter\": %.17g, \"hand_depth\": %.17g, \"hand_height\": %.17g, "
           "\"init_bite\": %.17g, \"volume_width\": %.17g, \"volume_depth\": %.17g, \"volume_height\": %.17g, "
           "\"image_size\": %d, \"image_num_channels\": %d, \"nn_radius\": %.17g, \"num_orientations\": %d, "
           "\"num_finger_placements\": %d, \"num_hand_axes\": %d, \"hand_axes0\": %d, \"deepen_hand\": %d, "
           "\"friction_coeff\": %.17g, \"min_viable\": %d, \"min_aperture\": %.17g, \"max_aperture\": %.17g, "
           "\"workspace_grasps\": [%.17g, %.17g, %.17g, %.17g, %.17g, %.17g], \"filter_approach_direction\": %d, "
           "\"direction\": [%.17g, %.17g, %.17g], \"thresh_rad\": %.17g, \"weights_file\": \"%s\", \"num_selected\": %d, "
           "\"num_samples\": %d, \"min_inliers\": %d",
           p.finger_width, p.hand_outer_diameter, p.hand_depth, p.hand_height, p.init_bite, p.volume_width, p.volume_depth,
           p.volume_height, p.image_size, p.image_num_channels, p.nn_radius, p.num_orientations, p.num_finger_placements,
           p.num_hand_axes, p.hand_axes[0], p.deepen_hand, p.friction_coeff, p.min_viable, p.min_aperture, p.max_aperture,
           p.workspace_grasps[0], p.workspace_grasps[1], p.workspace_grasps[2], p.workspace_grasps[3], p.workspace_grasps[4],
           p.workspace_grasps[5], p.filter_approach_direction, p.direction[0], p.direction[1], p.direction[2], p.thresh_rad,
           weights.c_str(), num_selected, num_samples, min_inliers);
    if (args.size() >= 2) {
      printf(", \"cloud_points\": %zu, \"cloud_has_normals\": %d", cloud.size(), (int)(cloud.getNormals().size() == 3 * cloud.size()));
      if (cloud.size()) printf(", \"first_point\": [%.9g, %.9g, %.9g]", cloud.getPoints()[0], cloud.getPoints()[1], cloud.getPoints()[2]);
    }
    printf("}\n");
    return 0;
  }
  if (batch) return run_batch(config_filename, std::vector<std::string>(args.begin() + 1, args.end()), sis, sis_seed);
  const std::string pcd_filename = args[1];
  if (!checkFileExists(pcd_filename)) return -1;
  util::ConfigFile config_file(config_filename);
  config_file.ExtractKeys();
  std::vector<double> camera_position = config_file.getValueOfKeyAsStdVectorDouble("camera_position", "0.0 0.0 0.0");
  util::Cloud cloud(pcd_filename, camera_position);
  if (cloud.size() == 0) {
    std::cout << "Error: Input point cloud is empty or does not exist!\n";
    return -1;
  }
  if (args.size() > 2) {
    cloud.setNormalsFromFile(args[2]);
    std::cout << "Loaded surface normals from file: " << args[2] << "\n";
  }
  if (sis) {  // cem_detect_grasps.cpp:52-64
    SequentialImportanceSampling sampler(config_filename);
    sampler.setSeed(sis_seed);
    sampler.detector().preprocessPointCloud(cloud);
    std::vector<std::unique_ptr<candidate::Hand>> grasps = sampler.detectGrasps(cloud);
    print_sis(grasps, sampler.handSetPositions(), sampler.evaluatedPositions());
    return 0;
  }
  GraspDetector detector(config_filename);
  detector.preprocessPointCloud(cloud);
  bool centered_at_origin = config_file.getValueOfKey<bool>("centered_at_origin", false);
  if (centered_at_origin) {  // detect_grasps.cpp:75-80
    std::vector<double> n = cloud.getNormals();
    for (double &v : n) v *= -1.0;
    cloud.setNormals(n);
    printf("Reversing normal directions ...\n");
  }
  std::vector<std::unique_ptr<candidate::Hand>> grasps = gpus > 1 ? detector.detectGraspsMultiGpu(cloud, gpus) : detector.detectGrasps(cloud);
  print_grasps(grasps);
  return 0;
}
