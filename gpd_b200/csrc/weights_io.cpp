// weights_io.cpp — host-side import of the reference's OTHER weight formats into the layout of the .bin parameter
// directory (SURVEY.md 8(f).2): the Caffe backend's `.caffemodel` (net::Classifier::create(model_file, weights_file),
// classifier.cpp:33-61, caffe_classifier.cpp) and the OpenVINO backend's IR `.xml` + `.bin`
// (openvino_classifier.cpp:20-57). No protobuf / XML library: the two containers are read at the wire level.
//
//   .bin directory layout (eigen_classifier.cpp:24-47, SURVEY.md A14): conv = OIHW row-major; ip = column-major
//   (out, in); ip1's input index is k = c + 50 j (j = 12 x 12 spatial) because the Eigen classifier flattens the
//   pooled map column-major, whereas Caffe / the IR flatten CHW: in = c * 144 + j and store (out, in) row-major.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"

namespace {

struct Blob {
  std::vector<float> data;
};
struct LayerBlobs {
  std::string name;
  std::vector<Blob> blobs;
};

// ---- protobuf wire format (https://protobuf.dev/programming-guides/encoding/) --------------------------------
struct Reader {
  const uint8_t *p, *end;
  bool ok = true;
  bool more() const { return ok && p < end; }
  uint64_t varint() {
    uint64_t v = 0;
    for (int shift = 0; shift < 64; shift += 7) {
      if (p >= end) { ok = false; return 0; }
      uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return v;
    }
    ok = false;
    return 0;
  }
  Reader sub() {  // length-delimited payload
    uint64_t n = varint();
    if (!ok || n > (uint64_t)(end - p)) { ok = false; return Reader{p, p}; }
    Reader r{p, p + n};
    p += n;
    return r;
  }
  void skip(int wire) {
    switch (wire) {
      case 0: varint(); break;
      case 1: if (end - p < 8) ok = false; else p += 8; break;
      case 2: sub(); break;
      case 5: if (end - p < 4) ok = false; else p += 4; break;
      default: ok = false;
    }
  }
};

// caffe.BlobProto: data = 5 (repeated float, packed or one per tag)
void parse_blob(Reader r, Blob &b) {
  while (r.more()) {
    uint64_t key = r.varint();
    const int field = (int)(key >> 3), wire = (int)(key & 7);
    if (field == 5 && wire == 2) {
      Reader d = r.sub();
      const size_t n = (size_t)(d.end - d.p) / 4;
      const size_t old = b.data.size();
      b.data.resize(old + n);
      memcpy(b.data.data() + old, d.p, n * 4);
    } else if (field == 5 && wire == 5) {
      float f;
      if (r.end - r.p < 4) { r.ok = false; break; }
      memcpy(&f, r.p, 4);
      r.p += 4;
      b.data.push_back(f);
    } else {
      r.skip(wire);
    }
  }
}
// caffe.LayerParameter: name = 1, blobs = 7; caffe.V1LayerParameter: name = 4, blobs = 6
void parse_layer(Reader r, int f_name, int f_blobs, LayerBlobs &l) {
  while (r.more()) {
    uint64_t key = r.varint();
    const int field = (int)(key >> 3), wire = (int)(key & 7);
    if (field == f_name && wire == 2) {
      Reader s = r.sub();
      l.name.assign((const char *)s.p, (size_t)(s.end - s.p));
    } else if (field == f_blobs && wire == 2) {
      l.blobs.emplace_back();
      parse_blob(r.sub(), l.blobs.back());
    } else {
      r.skip(wire);
    }
  }
}
// caffe.NetParameter: layer = 100 (LayerParameter), layers = 2 (V1LayerParameter)
bool parse_caffemodel(const std::vector<uint8_t> &buf, std::vector<LayerBlobs> &layers) {
  Reader r{buf.data(), buf.data() + buf.size()};
  while (r.more()) {
    uint64_t key = r.varint();
    const int field = (int)(key >> 3), wire = (int)(key & 7);
    if (field == 100 && wire == 2) {
      layers.emplace_back();
      parse_layer(r.sub(), 1, 7, layers.back());
    } else if (field == 2 && wire == 2) {
      layers.emplace_back();
      parse_layer(r.sub(), 4, 6, layers.back());
    } else {
      r.skip(wire);
    }
  }
  return r.ok;
}

bool read_file(const std::string &path, std::vector<uint8_t> &out) {
  FILE *f = fopen(path.c_str(), "rb");
  if (!f) return false;
  fseek(f, 0, SEEK_END);
  long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  out.resize(n > 0 ? (size_t)n : 0);
  bool ok = n >= 0 && fread(out.data(), 1, out.size(), f) == out.size();
  fclose(f);
  return ok;
}

bool ends_with(const std::string &s, const char *suf) {
  const size_t n = strlen(suf);
  return s.size() >= n && s.compare(s.size() - n, n, suf) == 0;
}

// (out, in = c * 144 + j) row-major -> .bin ip1 layout [o + 500 * (c + 50 j)]; (out, in) row-major -> [o + 2 k]
void fc_to_bin_layout(const std::vector<float> &f1, const std::vector<float> &f2, std::vector<float> &ip1, std::vector<float> &ip2) {
  ip1.resize((size_t)500 * 7200);
  for (int o = 0; o < 500; o++)
    for (int c = 0; c < 50; c++)
      for (int j = 0; j < 144; j++) ip1[(size_t)o + 500 * ((size_t)c + 50 * (size_t)j)] = f1[(size_t)o * 7200 + (size_t)c * 144 + j];
  ip2.resize(1000);
  for (int o = 0; o < 2; o++)
    for (int k = 0; k < 500; k++) ip2[o + 2 * k] = f2[(size_t)o * 500 + k];
}

}  // namespace

#define FAIL(code, ...)                          \
  do {                                           \
    snprintf(err, 480, __VA_ARGS__);             \
    return code;                                 \
  } while (0)

// reads a .caffemodel / OpenVINO IR into the .bin layout; relu_layers receives the number of ReLU layers of an IR
// (-1 for a caffemodel: the prototxt decides, the reference's nets have none after the convolutions)
static int read_weights(const char *model_file, const std::string &wf, int C, std::vector<float> a[8], int *relu_layers, char *err) {
  const size_t sizes[8] = {(size_t)20 * C * 25, 20, 50 * 20 * 25, 50, (size_t)500 * 7200, 500, 1000, 2};
  *relu_layers = -1;
  if (ends_with(wf, ".caffemodel")) {
    std::vector<uint8_t> buf;
    if (!read_file(wf, buf)) {
      FAIL(GPDB_ERR_IO, "Cannot open file: %s", wf.c_str());
    }
    std::vector<LayerBlobs> layers;
    if (!parse_caffemodel(buf, layers)) {
      FAIL(GPDB_ERR_IO, "%s: not a caffe NetParameter", wf.c_str());
    }
    const char *names[4] = {"conv1", "conv2", "ip1", "ip2"};
    std::vector<float> raw[8];
    for (int l = 0; l < 4; l++) {
      const LayerBlobs *found = nullptr;
      for (const LayerBlobs &lb : layers)
        if (lb.name == names[l] && lb.blobs.size() >= 2) found = &lb;
      if (!found) {
        FAIL(GPDB_ERR_IO, "%s: layer '%s' with weight and bias blobs not found", wf.c_str(), names[l]);
      }
      raw[2 * l] = found->blobs[0].data;
      raw[2 * l + 1] = found->blobs[1].data;
    }
    for (int i = 0; i < 8; i++)
      if (raw[i].size() != sizes[i]) {
        FAIL(GPDB_ERR_IO, "%s: blob %d has %zu values, expected %zu for %d channels", wf.c_str(), i, raw[i].size(), sizes[i], C);
      }
    a[0] = raw[0]; a[1] = raw[1]; a[2] = raw[2]; a[3] = raw[3]; a[5] = raw[5]; a[7] = raw[7];
    fc_to_bin_layout(raw[4], raw[6], a[4], a[6]);
  } else if (ends_with(wf, ".bin") || ends_with(wf, ".xml")) {
    // OpenVINO IR v4: <weights offset= size=/> <biases offset= size=/> per Convolution / FullyConnected layer, in order
    std::string xml_path = (model_file && *model_file) ? model_file : wf.substr(0, wf.size() - 4) + ".xml";
    std::string bin_path = ends_with(wf, ".bin") ? wf : wf.substr(0, wf.size() - 4) + ".bin";
    if (ends_with(wf, ".xml")) xml_path = wf;
    std::vector<uint8_t> xml, bin;
    if (!read_file(xml_path, xml) || !read_file(bin_path, bin)) {
      FAIL(GPDB_ERR_IO, "Cannot open file: %s / %s", xml_path.c_str(), bin_path.c_str());
    }
    const std::string x((const char *)xml.data(), xml.size());
    std::vector<std::pair<size_t, size_t>> blobs;
    for (size_t pos = 0;;) {
      size_t w = x.find("<weights ", pos), b = x.find("<biases ", pos);
      size_t at = std::min(w, b);
      if (at == std::string::npos) break;
      unsigned long long off = 0, sz = 0;
      size_t o = x.find("offset=\"", at), s = x.find("size=\"", at);
      if (o == std::string::npos || s == std::string::npos) break;
      off = strtoull(x.c_str() + o + 8, nullptr, 10);
      sz = strtoull(x.c_str() + s + 6, nullptr, 10);
      blobs.push_back({(size_t)off, (size_t)sz});
      pos = at + 8;
    }
    int n_relu = 0;
    for (size_t pos = 0; (pos = x.find("type=\"ReLU\"", pos)) != std::string::npos; pos += 10) n_relu++;
    if (blobs.size() != 8) {
      FAIL(GPDB_ERR_IO, "%s: expected 8 weight / bias blobs (conv1, conv2, fc1, fc2), found %zu", xml_path.c_str(), blobs.size());
    }
    *relu_layers = n_relu;
    std::vector<float> raw[8];
    for (int i = 0; i < 8; i++) {
      if (blobs[i].second != sizes[i] * 4 || blobs[i].first > bin.size() || blobs[i].second > bin.size() - blobs[i].first) {  // no wrap-around
        FAIL(GPDB_ERR_IO, "%s: blob %d has %zu bytes, expected %zu for %d channels", xml_path.c_str(), i, blobs[i].second, sizes[i] * 4, C);
      }
      raw[i].resize(sizes[i]);
      memcpy(raw[i].data(), bin.data() + blobs[i].first, blobs[i].second);
    }
    a[0] = raw[0]; a[1] = raw[1]; a[2] = raw[2]; a[3] = raw[3]; a[5] = raw[5]; a[7] = raw[7];
    fc_to_bin_layout(raw[4], raw[6], a[4], a[6]);
  } else {
    FAIL(GPDB_ERR_INVALID, "weights_file '%s': expected a parameter directory (trailing '/'), a .caffemodel or an OpenVINO IR .bin / .xml",
         wf.c_str());
  }
  return GPDB_OK;
}

extern "C" {

// Host-only conversion (no device needed): fills the eight caller-allocated arrays in the .bin layout.
int gpdb_read_weights_file(const char *model_file, const char *weights_file, int32_t channels, float *const out[8],
                           int32_t *relu_layers_out, char *err_out, int32_t err_len) {
  char err[512] = "";
  std::vector<float> a[8];
  int relu = -1;
  if (!weights_file || !out) return GPDB_ERR_INVALID;
  int rc = read_weights(model_file, weights_file, channels, a, &relu, err);
  if (err_out && err_len > 0) snprintf(err_out, (size_t)err_len, "%s", err);
  if (rc != GPDB_OK) return rc;
  for (int i = 0; i < 8; i++) memcpy(out[i], a[i].data(), a[i].size() * sizeof(float));
  if (relu_layers_out) *relu_layers_out = relu;
  return GPDB_OK;
}

int gpdb_load_weights_file(gpdb_ctx *ctx, const char *model_file, const char *weights_file) {
  if (!ctx || !weights_file) return GPDB_ERR_INVALID;
  const std::string wf = weights_file;
  if (wf.empty() || wf.back() == '/') return gpdb_load_weights_dir(ctx, weights_file);
  char err[512] = "";
  std::vector<float> a[8];
  int relu = -1;
  int rc = read_weights(model_file, wf, ctx->prm.image_num_channels, a, &relu, err);
  if (rc != GPDB_OK) {
    gpdb_set_error(ctx, rc, "%s", err);
    return rc;
  }
  if (relu >= 0 && (relu >= 3) != (ctx->prm.relu_after_conv != 0)) {
    gpdb_set_error(ctx, GPDB_ERR_INVALID, "%s has %d ReLU layers: create the context with relu_after_conv = %d", weights_file, relu,
                   relu >= 3 ? 1 : 0);
    return GPDB_ERR_INVALID;
  }
  return gpdb_set_weights(ctx, a[0].data(), a[1].data(), a[2].data(), a[3].data(), a[4].data(), a[5].data(), a[6].data(), a[7].data());
}

// The .bin parameter directory, written: each array as raw little-endian float32, the layout gpdb_load_weights_dir and
// readBinaryFileIntoVector (eigen_classifier.cpp:185-205) read.
int gpdb_write_weights_dir(const char *dir, int32_t channels, const float *const w[8]) {
  if (!dir || !*dir || !w || !(channels == 1 || channels == 3 || channels == 12 || channels == 15)) return GPDB_ERR_INVALID;
  for (int i = 0; i < 8; i++)
    if (!w[i]) return GPDB_ERR_INVALID;
  const char *names[8] = {"conv1_weights", "conv1_biases", "conv2_weights", "conv2_biases",
                          "ip1_weights",   "ip1_biases",   "ip2_weights",   "ip2_biases"};
  const size_t sizes[8] = {(size_t)20 * channels * 25, 20, 50 * 20 * 25, 50, (size_t)500 * 7200, 500, 1000, 2};
  std::string d = dir;
  if (d.back() != '/') d += '/';
  for (int i = 0; i < 8; i++) {
    FILE *f = fopen((d + names[i] + ".bin").c_str(), "wb");
    if (!f) return GPDB_ERR_IO;
    const bool ok = fwrite(w[i], sizeof(float), sizes[i], f) == sizes[i];
    if ((fclose(f) != 0) || !ok) return GPDB_ERR_IO;
  }
  return GPDB_OK;
}

}  // extern "C"
