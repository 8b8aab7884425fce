/*
 * gpd_b200_train.h — SPECIFICATION of LeNet training on the device (gpdb_train_begin, gpdb_train_step[_device],
 * gpdb_train_weights, gpdb_debug_train_step); the entry points are declared in gpd_b200.h.
 *
 * Network. The context's classifier: C = image_num_channels input channels, 60 x 60 images (image_size 60 only, as
 * gpdb_classify), raw 0..255 inputs without scaling. conv1 (C -> 20, 5 x 5), 2 x 2 max-pool, conv2 (20 -> 50, 5 x 5),
 * 2 x 2 max-pool, with a ReLU before each pool when relu_after_conv = 1; ip1 (7 200 -> 500) + ReLU; ip2 (500 -> 2
 * logits). relu_after_conv = 1 is the reference's pytorch/network.py Net, 0 the Caffe LeNet. Parameters are the eight
 * arrays of the .bin layout (gpdb_set_weights): conv OIHW row-major, ip1 / ip2 column-major (out, in), ip1's input
 * k = c + 50 j (pool2 channel c, pixel j = 12 y + x): torch's fc1.weight[o][144 c + j] is ip1_w[o + 500 (c + 50 j)].
 * Pixel (y, x) of channel c of an HWC image is byte (60 y + x) C + c: the true HWC -> CHW transpose of the inference
 * kernels. DEPARTURE: the reference's train_net.py, train_net2.py and train_net4.py `reshape` HWC arrays to CHW, so those
 * networks see scrambled pixels compared with what EigenClassifier gives them at inference.
 *
 *  1. Forward. Bit for bit the float32 FMA chains of gpdb_classify with lenet_impl = 1 (lenet_simt.cu): the same kernels
 *     run. The pooled value of a window is max(acc) + bias (then ReLU), max first: fl(. + b) is monotone, so it equals the
 *     max over the window of fl(acc + b).
 *  2. Pooling choice. The window position that receives the gradient is the FIRST maximum, in row-major order
 *     ((0,0), (0,1), (1,0), (1,1)), of v_a = fl(acc_a + b), acc_a the same FMA chains as 1 — torch's max_pool2d rule on the
 *     pre-ReLU values (ReLU is monotone, so it picks the same position after it). With ReLU before the pool, a pooled value
 *     of 0 passes no gradient (ReLU'(0) = 0, as torch): the mask is pooled > 0. ip1's ReLU likewise passes h > 0.
 *  3. Loss. Image i with logits z0, z1 and label y in {0, 1}: d = |z1 - z0|, e = expf(-d), l = log1pf(e);
 *     loss_i = l when z_y is the larger logit (z_y >= z_other), else d + l (gpdb_train_loss). The step's loss is
 *     (sum_i loss_i) / n, the sum one float32 chain in image order. Mean of torch.nn.CrossEntropyLoss.
 *  4. d logits. With s = 1 + e, the larger logit (z1 on a tie) has probability 1 / s and the other e / s;
 *     dz_k = (p_k - [k == y]) / n (gpdb_train_dlogits). When expf underflows, p = (1, 0) exactly.
 *     The device's expf and log1pf (2 and 1 ulp) may differ from the host's libm by a few ulp; these two helpers are
 *     bit-exact between host builds only. The device's loss is checked against them within 8 ulp, and each d logit
 *     within 8 ulp of the larger of |dz_k| and p_k / n: for the labelled, larger logit, p_k - 1 cancels the leading
 *     bits of p_k, so a 1-ulp difference in p_k can be many ulp of dz_k itself (63 measured on an H100 at a logit gap
 *     of 4.1, n = 65). Everything after the d logits is defined on the device's own d logits.
 *  5. Backward, every reduction one FMA chain in a fixed order (no atomics; two identical call sequences give identical
 *     bits). For each parameter the sum over images is: per-image partial sums, then one chain over the images in order,
 *     continuing from the previous chunk's total (a step of more than GPDB_TRAIN_CHUNK images is processed in chunks),
 *     so the result does not depend on the chunk size. ip1 / ip2 weight gradients chain directly over the images.
 *       ip2:   dW2[o + 2k] = sum_i dz[i][o] h[i][k];  db2[o] = sum_i dz[i][o]
 *       dh[i][k] = fmaf(W2[2k+1], dz1, W2[2k] dz0), 0 where h = 0
 *       ip1:   dW1[k][o] = sum_i x[i][k] dh[i][o];  db1[o] = sum_i dh[i][o];  dx[i][k] = sum_o dh[i][o] W1[k][o] (o in order)
 *       pool2: g2 = dx masked by rule 2; conv2 weight / bias gradients per image over the 144 pooled positions in
 *              row-major order, each at its chosen input window; d conv2 (dense 24 x 24, zero off the choices)
 *       pool1: dp1[c][y][x] = sum over (o, kh, kw) in order of dconv2[o][y-kh][x-kw] W2[o][c][kh][kw];
 *              g1 = dp1 masked; conv1 gradients per image over the 784 pooled positions. conv1 has no data gradient.
 *  6. Optimisers, float32, one rounding per written operation (no FMA):
 *       SGD (torch.optim.SGD, dampening 0, no Nesterov): g' = g + wd p (skipped when wd = 0);
 *         with momentum mu != 0: b = g' at the first step, else b = mu b + g'; g' = b.  p = p - lr g'.
 *       Adam (torch.optim.Adam, L2 weight decay, amsgrad off), step t = 1, 2, ..: g' = g + wd p (skipped when wd = 0);
 *         m = b1 m + (1 - b1) g';  v = b2 v + (1 - b2) (g' g');  with bc1 = 1 - b1^t, bc2 = 1 - b2^t in float64 (as
 *         torch's Python arithmetic), step = (float)(lr / bc1), r = (float)sqrt(bc2):
 *         p = p - step (m / (sqrtf(v) / r + eps)).  (1 - b1) and (1 - b2) are rounded to float32 once.
 *       torch writes m with lerp and fuses some of these operations on some devices, so its float32 update can differ
 *       from this one in the last bit; the rules here are what the tests pin.
 *
 * tests/train_reference.py restates this file in numpy.
 */
#ifndef GPD_B200_TRAIN_H_
#define GPD_B200_TRAIN_H_

#include <math.h>
#include <stdint.h>

#include "gpd_b200_shadow.h" /* GPDB_HD */

/* images per chunk of a training step; a larger step runs in chunks (rule 5) */
#define GPDB_TRAIN_CHUNK 256

/* rule 3: the loss of one image */
GPDB_HD float gpdb_train_loss(float z0, float z1, int32_t y) {
  const float d = fabsf(z1 - z0);
  const float l = log1pf(expf(-d));
  const bool top = y ? (z1 >= z0) : (z0 >= z1);
  return top ? l : d + l;
}

/* rule 4: d logits of one image in a step of n images */
GPDB_HD void gpdb_train_dlogits(float z0, float z1, int32_t y, float n, float *dz) {
  const float e = expf(-fabsf(z1 - z0));
  const float s = 1.0f + e;
  const float pb = 1.0f / s, ps = e / s;
  const float p1 = (z1 >= z0) ? pb : ps, p0 = (z1 >= z0) ? ps : pb;
  dz[0] = (p0 - (y == 0 ? 1.0f : 0.0f)) / n;
  dz[1] = (p1 - (y == 1 ? 1.0f : 0.0f)) / n;
}

/* rule 6, SGD: one parameter; first = the optimiser's first step since gpdb_train_begin */
GPDB_HD void gpdb_train_sgd(float *p, float g, float *buf, float lr, float mu, float wd, bool first) {
  if (wd != 0.0f) g = g + wd * *p;
  if (mu != 0.0f) {
    *buf = first ? g : mu * *buf + g;
    g = *buf;
  }
  *p = *p - lr * g;
}

/* rule 6, Adam: one parameter; omb1 = (float)(1 - b1), omb2 = (float)(1 - b2), step and r from gpdb_train_adam_scalars */
GPDB_HD void gpdb_train_adam(float *p, float g, float *m, float *v, float b1, float omb1, float b2, float omb2, float eps,
                             float wd, float step, float r) {
  if (wd != 0.0f) g = g + wd * *p;
  *m = b1 * *m + omb1 * g;
  *v = b2 * *v + omb2 * (g * g);
  const float denom = sqrtf(*v) / r + eps;
  *p = *p - step * (*m / denom);
}

/* rule 6, Adam: the bias corrections of step t >= 1 (float64, as torch's Python scalars) */
GPDB_HD void gpdb_train_adam_scalars(float lr, float b1, float b2, int64_t t, float *step, float *r) {
  const double bc1 = 1.0 - pow((double)b1, (double)t), bc2 = 1.0 - pow((double)b2, (double)t);
  *step = (float)((double)lr / bc1);
  *r = (float)sqrt(bc2);
}

#endif /* GPD_B200_TRAIN_H_ */
