// train_chains.cpp — a sequential host restatement of include/gpd_b200_train.h rules 1, 2 and 5 (test infrastructure
// only): every float32 chain of a training step, in the header's order, so the device's pooling choices, per-image
// stages and gradients can be held against it bit for bit (tests/train_chains.py loads it).
//
// Built with -ffp-contract=off and without -mfma or -ffast-math: a product outside fmaf is rounded on its own, and fmaf
// is libm's, correctly rounded. With OpenMP the loops spread outputs (or whole images) over threads; every output's chain
// stays in one thread and in its order.
//
// Arrays are those of gpdb_train_debug and the .bin layouts: images HWC uint8 [n][60][60][C]; pool1 / choice1 / d pool1
// [n][20][28][28]; pool2 / choice2 / d pool2 [n][7200] with k = c + 50 j; ip1 / d ip1 [n][500]; d logits [n][2]; dense
// d conv2 [n][50][24][24]. `variant` = 0 is the header's rule everywhere; the other values are deliberate departures that
// tests/test_train_chains.py uses to show what a bit-exact comparison catches and an error bound lets through.
#include <math.h>
#include <stdint.h>

#include <vector>

namespace {

constexpr int NF1 = 20, NF2 = 50, NH = 500, S = 60, P1 = 28, O2 = 24, P2 = 12, K = 7200;

// rule 2: the first strict maximum in row-major window order (variant 1: the last maximum)
int choose(const float v[4], int variant) {
  int a = 0;
  for (int q = 1; q < 4; q++)
    if (variant ? v[q] >= v[a] : v[q] > v[a]) a = q;
  return a;
}

// rule 1: ReLU of a pooled value when relu_after_conv
float relu_of(float v, int relu) { return (relu && !(v > 0.0f)) ? 0.0f : v; }

// rule 2: the gradient a pooled value passes to its chosen position, none under a ReLU that output 0
float pooled_grad(float d, float pooled, int relu) { return (!relu || pooled > 0.0f) ? d : 0.0f; }

}  // namespace

// Rules 1 and 2, conv1: per (image, filter o, pooled pixel) four accumulators from +0, fmaf(w1[o][c][kh][kw], pixel,
// acc) in (c, kh, kw) order over the true HWC -> CHW transpose; v_q = acc_q + b1[o]; the choice and v_choice (then ReLU).
extern "C" void tc_pool1(int n, int C, int relu, const uint8_t *img, const float *w1, const float *b1, int variant,
                         uint8_t *choice, float *pooled) {
#pragma omp parallel for schedule(dynamic)
  for (long t = 0; t < (long)n * NF1; t++) {
    const long i = t / NF1;
    const int o = (int)(t % NF1);
    const uint8_t *g = img + i * S * S * C;
    for (int py = 0; py < P1; py++)
      for (int px = 0; px < P1; px++) {
        float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        for (int c = 0; c < C; c++)
          for (int kh = 0; kh < 5; kh++)
            for (int kw = 0; kw < 5; kw++) {
              const float wv = w1[((o * C + c) * 5 + kh) * 5 + kw];
              for (int q = 0; q < 4; q++) {
                const int y = 2 * py + kh + (q >> 1), x = 2 * px + kw + (q & 1);
                acc[q] = fmaf(wv, (float)g[(y * S + x) * C + c], acc[q]);
              }
            }
        float v[4];
        for (int q = 0; q < 4; q++) v[q] = acc[q] + b1[o];
        const int a = choose(v, variant);
        const long at = t * P1 * P1 + py * P1 + px;
        choice[at] = (uint8_t)a;
        pooled[at] = relu_of(v[a], relu);
      }
  }
}

// Rules 1 and 2, conv2 over a given pool1: the same with c over 20, out in the k = c + 50 j order.
extern "C" void tc_pool2(int n, int relu, const float *p1, const float *w2, const float *b2, int variant, uint8_t *choice,
                         float *pooled) {
#pragma omp parallel for schedule(dynamic)
  for (long t = 0; t < (long)n * NF2; t++) {
    const long i = t / NF2;
    const int o = (int)(t % NF2);
    const float *in = p1 + i * NF1 * P1 * P1;
    for (int py = 0; py < P2; py++)
      for (int px = 0; px < P2; px++) {
        float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        for (int c = 0; c < NF1; c++)
          for (int kh = 0; kh < 5; kh++)
            for (int kw = 0; kw < 5; kw++) {
              const float wv = w2[((o * NF1 + c) * 5 + kh) * 5 + kw];
              for (int q = 0; q < 4; q++) {
                const int y = 2 * py + kh + (q >> 1), x = 2 * px + kw + (q & 1);
                acc[q] = fmaf(wv, in[(c * P1 + y) * P1 + x], acc[q]);
              }
            }
        float v[4];
        for (int q = 0; q < 4; q++) v[q] = acc[q] + b2[o];
        const int a = choose(v, variant);
        const long at = i * K + (py * P2 + px) * NF2 + o;
        choice[at] = (uint8_t)a;
        pooled[at] = relu_of(v[a], relu);
      }
  }
}

// Rule 5, d ip1: h > 0 ? fmaf(W2[2k+1], dz1, W2[2k] dz0) : +0, the product W2[2k] dz0 rounded on its own.
extern "C" void tc_dip1(int n, const float *h, const float *dz, const float *W2, float *dh) {
#pragma omp parallel for
  for (long e = 0; e < (long)n * NH; e++) {
    const long i = e / NH;
    const int k = (int)(e % NH);
    const float p0 = W2[2 * k] * dz[2 * i];
    dh[e] = h[e] > 0.0f ? fmaf(W2[2 * k + 1], dz[2 * i + 1], p0) : 0.0f;
  }
}

// Rule 5, d pool2[i][k]: one FMA chain over o = 0..499 of dh[i][o] W1[o + 500 k], from +0.
extern "C" void tc_dpool2(int n, const float *dh, const float *W1, float *dx) {
#pragma omp parallel for schedule(static)
  for (long e = 0; e < (long)n * K; e++) {
    const long i = e / K, k = e % K;
    float acc = 0.0f;
    for (int o = 0; o < NH; o++) acc = fmaf(dh[i * NH + o], W1[o + NH * k], acc);
    dx[e] = acc;
  }
}

// Rules 2 and 5, dense d conv2: the masked d pool2 at the chosen window position, +0 elsewhere.
extern "C" void tc_dconv2(int n, int relu, const float *dx, const float *p2, const uint8_t *ch2, float *dc2) {
#pragma omp parallel for
  for (long e = 0; e < (long)n * NF2 * O2 * O2; e++) {
    const long i = e / (NF2 * O2 * O2);
    const int o = (int)((e / (O2 * O2)) % NF2), Y = (int)((e / O2) % O2), X = (int)(e % O2);
    const long k = i * K + ((Y >> 1) * P2 + (X >> 1)) * NF2 + o;
    dc2[e] = ch2[k] == (Y & 1) * 2 + (X & 1) ? pooled_grad(dx[k], p2[k], relu) : 0.0f;
  }
}

// Rule 5, d pool1[i][c][y][x]: one chain over o, then kh in [max(0, y-23), min(4, y)], then kw in [max(0, x-23),
// min(4, x)], of dc2[o][y-kh][x-kw] w2[o][c][kh][kw], from +0. Variant 1 chains over (kh, kw, o) instead.
extern "C" void tc_dpool1(int n, const float *dc2, const float *w2, int variant, float *dp1) {
#pragma omp parallel for schedule(dynamic)
  for (long t = 0; t < (long)n * NF1; t++) {
    const long i = t / NF1;
    const int c = (int)(t % NF1);
    const float *d = dc2 + i * NF2 * O2 * O2;
    for (int y = 0; y < P1; y++)
      for (int x = 0; x < P1; x++) {
        const int kh0 = y > O2 - 1 ? y - (O2 - 1) : 0, kh1 = y < 4 ? y : 4;
        const int kw0 = x > O2 - 1 ? x - (O2 - 1) : 0, kw1 = x < 4 ? x : 4;
        auto term = [&](int o, int kh, int kw, float acc) {
          return fmaf(d[(o * O2 + y - kh) * O2 + x - kw], w2[((o * NF1 + c) * 5 + kh) * 5 + kw], acc);
        };
        float acc = 0.0f;
        if (variant == 0) {
          for (int o = 0; o < NF2; o++)
            for (int kh = kh0; kh <= kh1; kh++)
              for (int kw = kw0; kw <= kw1; kw++) acc = term(o, kh, kw, acc);
        } else {
          for (int kh = kh0; kh <= kh1; kh++)
            for (int kw = kw0; kw <= kw1; kw++)
              for (int o = 0; o < NF2; o++) acc = term(o, kh, kw, acc);
        }
        dp1[t * P1 * P1 + y * P1 + x] = acc;
      }
  }
}

namespace {

// Rule 5, the sum over images of per-image partials part[i][e]: one float-add chain over the images in order from +0.
// restart > 0: a second chain starts at image `restart` and the two totals are added (a departure).
void image_chain(int n, int ne, const float *part, int restart, float *out) {
#pragma omp parallel for schedule(static)
  for (int e = 0; e < ne; e++) {
    float s = 0.0f, head = 0.0f;
    for (int i = 0; i < n; i++) {
      if (restart > 0 && i == restart) head = s, s = 0.0f;
      s += part[(long)i * ne + e];
    }
    out[e] = (restart > 0 && n > restart) ? head + s : s;
  }
}

}  // namespace

// Rule 5, conv2 weight and bias gradients. Per image: each weight one FMA chain over the 144 pooled positions in
// row-major order of g[o][j] p1[c][window + (kh, kw)] at the chosen window, each bias a float-add chain of g[o][j]
// (g the masked d pool2); then image_chain. gw [25000] (.bin order), gb [50].
extern "C" void tc_conv2_grad(int n, int relu, const float *p1, const float *dx, const float *p2, const uint8_t *ch2,
                              int restart, float *gw, float *gb) {
  constexpr int NW = NF2 * NF1 * 25 + NF2;
  std::vector<float> part((size_t)n * NW);
#pragma omp parallel for schedule(dynamic)
  for (long t = 0; t < (long)n * NF2; t++) {
    const long i = t / NF2;
    const int o = (int)(t % NF2);
    float g[P2 * P2];
    int pos[P2 * P2];
    for (int j = 0; j < P2 * P2; j++) {
      const long k = i * K + j * NF2 + o;
      const int a = ch2[k];
      g[j] = pooled_grad(dx[k], p2[k], relu);
      pos[j] = (2 * (j / P2) + (a >> 1)) * P1 + 2 * (j % P2) + (a & 1);
    }
    float *pt = part.data() + i * NW;
    for (int c = 0; c < NF1; c++)
      for (int kh = 0; kh < 5; kh++)
        for (int kw = 0; kw < 5; kw++) {
          const float *x = p1 + (i * NF1 + c) * P1 * P1 + kh * P1 + kw;
          float acc = 0.0f;
          for (int j = 0; j < P2 * P2; j++) acc = fmaf(g[j], x[pos[j]], acc);
          pt[((o * NF1 + c) * 5 + kh) * 5 + kw] = acc;
        }
    float acc = 0.0f;
    for (int j = 0; j < P2 * P2; j++) acc += g[j];
    pt[NF2 * NF1 * 25 + o] = acc;
  }
  std::vector<float> tot(NW);
  image_chain(n, NW, part.data(), restart, tot.data());
  for (int e = 0; e < NW; e++) (e < NF2 * NF1 * 25 ? gw[e] : gb[e - NF2 * NF1 * 25]) = tot[e];
}

// Rule 5, conv1 weight and bias gradients: as conv2 over the 784 pooled positions of the masked d pool1, against the
// image's pixels (true HWC -> CHW transpose). gw [20 C 25] (.bin order), gb [20].
extern "C" void tc_conv1_grad(int n, int C, int relu, const uint8_t *img, const float *dp1, const float *p1,
                              const uint8_t *ch1, int restart, float *gw, float *gb) {
  const int nw = NF1 * C * 25, NW = nw + NF1;
  std::vector<float> part((size_t)n * NW);
#pragma omp parallel for schedule(dynamic)
  for (long t = 0; t < (long)n * NF1; t++) {
    const long i = t / NF1;
    const int o = (int)(t % NF1);
    const uint8_t *im = img + i * S * S * C;
    std::vector<float> g(P1 * P1);
    std::vector<int> pos(P1 * P1);
    for (int p = 0; p < P1 * P1; p++) {
      const long at = t * P1 * P1 + p;
      const int a = ch1[at];
      g[p] = pooled_grad(dp1[at], p1[at], relu);
      pos[p] = (2 * (p / P1) + (a >> 1)) * S + 2 * (p % P1) + (a & 1);
    }
    float *pt = part.data() + i * NW;
    for (int c = 0; c < C; c++)
      for (int kh = 0; kh < 5; kh++)
        for (int kw = 0; kw < 5; kw++) {
          float acc = 0.0f;
          for (int p = 0; p < P1 * P1; p++) acc = fmaf(g[p], (float)im[(pos[p] + kh * S + kw) * C + c], acc);
          pt[((o * C + c) * 5 + kh) * 5 + kw] = acc;
        }
    float acc = 0.0f;
    for (int p = 0; p < P1 * P1; p++) acc += g[p];
    pt[nw + o] = acc;
  }
  std::vector<float> tot(NW);
  image_chain(n, NW, part.data(), restart, tot.data());
  for (int e = 0; e < NW; e++) (e < nw ? gw[e] : gb[e - nw]) = tot[e];
}

// Rule 5, ip1 and ip2 gradients, chained directly over the images from +0: dW1[k][o] (index 500 k + o) an FMA chain of
// pool2[i][k] dh[i][o]; dW2[o + 2k] of ip1[i][k] dz[i][o]; db1, db2 float-add chains of dh and dz. reverse = 1 chains
// dW1 over the images in reverse order (a departure).
extern "C" void tc_ip_grads(int n, const float *p2, const float *dh, const float *h, const float *dz, int reverse,
                            float *dW1, float *db1, float *dW2, float *db2) {
#pragma omp parallel for schedule(static)
  for (int k = 0; k < K; k++) {
    float acc[NH];
    for (int o = 0; o < NH; o++) acc[o] = 0.0f;
    for (int r = 0; r < n; r++) {
      const long i = reverse ? n - 1 - r : r;
      const float a = p2[i * K + k];
      for (int o = 0; o < NH; o++) acc[o] = fmaf(a, dh[i * NH + o], acc[o]);
    }
    for (int o = 0; o < NH; o++) dW1[(long)k * NH + o] = acc[o];
  }
#pragma omp parallel for schedule(static)
  for (int k = 0; k < NH; k++) {
    float a0 = 0.0f, a1 = 0.0f, s = 0.0f;
    for (long i = 0; i < n; i++) {
      a0 = fmaf(h[i * NH + k], dz[2 * i], a0);
      a1 = fmaf(h[i * NH + k], dz[2 * i + 1], a1);
      s += dh[i * NH + k];
    }
    dW2[2 * k] = a0, dW2[2 * k + 1] = a1, db1[k] = s;
  }
  for (int o = 0; o < 2; o++) {
    float s = 0.0f;
    for (long i = 0; i < n; i++) s += dz[2 * i + o];
    db2[o] = s;
  }
}
