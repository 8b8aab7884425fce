"""Independent pin of the oracle's grasp-image stage (A8, A10-A12): a line-by-line numpy restatement of
ImageStrategy::transformToUnitImage / findCellIndices / createNormalsImage / createDepthImage and
Image12ChannelsStrategy::calculateImage (image_strategy.cpp:32-191, image_12_channels_strategy.cpp:35-86) that calls the
REAL OpenCV (cv2.dilate / cv2.normalize / convertScaleAbs = the code the reference links against) for every image
operation, against oracle.images() on the same poses. The neighbourhood comes from the oracle's radius search (pinned
separately against brute force). Shadow channels are not covered here: they follow the deterministic variant of
include/gpd_b200_shadow.h, for which no upstream behaviour exists to pin against."""
import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import abi, scenes
from image_reference import shadow_points
from oracle import oracle

cv2 = pytest.importorskip("cv2")
S = 60
EL = None


def _post(img):
    """cv::dilate(3x3 rect) -> cv::normalize(NORM_MINMAX, 0..1) -> convertTo(CV_8U, 255)."""
    d = cv2.dilate(img, cv2.getStructuringElement(cv2.MORPH_RECT, (3, 3)))
    n = cv2.normalize(d, None, 0.0, 1.0, cv2.NORM_MINMAX, cv2.CV_32F)
    return cv2.convertScaleAbs(n, alpha=255.0).reshape(S, S, -1)


def _normals_image(normals, cells):
    img = np.zeros((S, S, 3), np.float32)
    for i, idx in enumerate(cells):
        row, col = S - 1 - idx // S, idx % S
        v = img[row, col]
        a = np.abs(normals[:, i]).astype(np.float32)          # cv::Vec3f(fabs(n))
        if v[0] == 0 and v[1] == 0 and v[2] == 0:
            img[row, col] = a
        else:                                                  # v += (a - v) * (1.0 / sqrt(v.v)): double factor, Vec3f result
            f = 1.0 / np.sqrt(float(v[0]) * float(v[0]) + float(v[1]) * float(v[1]) + float(v[2]) * float(v[2]))
            img[row, col] = (v + ((a - v).astype(np.float64) * f).astype(np.float32)).astype(np.float32)
    return _post(img)


def _depth_image(points, cells):
    img = np.zeros((S, S), np.float32)
    avgs, counts = np.zeros(S * S, np.float32), np.zeros(S * S, np.float32)
    for i, idx in enumerate(cells):
        counts[idx] = np.float32(counts[idx] + np.float32(1.0))
        avgs[idx] = np.float32(float(avgs[idx]) + (points[2, i] - float(avgs[idx])) * (1.0 / float(counts[idx])))
        img[S - 1 - idx // S, idx % S] = np.float32(1.0 - float(avgs[idx]))
    return _post(img)[:, :, 0]


def _shadow_image(points, cells):
    """createShadowImage (image_strategy.cpp:193-233): float32 running mean per cell, max over occupied - mean."""
    img = np.zeros((S, S), np.float32)
    nonzero = np.zeros((S, S), bool)
    counts = np.zeros(S * S, np.float32)
    for i, idx in enumerate(cells):
        row, col = S - 1 - idx // S, idx % S
        counts[idx] = np.float32(counts[idx] + np.float32(1.0))
        img[row, col] = np.float32(float(img[row, col]) + (points[2, i] - float(img[row, col])) * (1.0 / float(counts[idx])))
        nonzero[row, col] = True
    mx = np.float32(img[nonzero].max()) if nonzero.any() else np.float32(0.0)     # cv::minMaxLoc with mask
    out = np.where(nonzero, mx - img, np.float32(0.0)).astype(np.float32)          # max_img - image
    return _post(out)[:, :, 0]


def reference_image(pose, pts, nrm, channels, w=0.10, d=0.06, h=0.02, shadow=None):
    F = np.array(pose["frame"]).reshape(3, 3).T                                   # column-major Hand::getFrame
    sample = np.array(pose["sample"])
    P = F.T @ (pts.T - sample[:, None])                                           # rotation * (points - sample)
    N = F.T @ nrm.T
    bottom, center = float(pose["bottom"]), float(pose["center"])
    m = ((P[0] > bottom) & (P[0] < bottom + d) & (P[1] > center - w / 2.0) & (P[1] < center + w / 2.0) & (P[2] > -1.0 * h) & (P[2] < h))
    P, N = P[:, m], N[:, m]
    U = np.stack([(P[0] - bottom) / d, (P[1] - (center - w / 2.0)) / w, (P[2] + h) / (2.0 * h)])
    cellsize = 1.0 / float(S)
    out = []
    proj = U.copy()
    sproj = None
    if shadow is not None:                                   # Image15ChannelsStrategy::createImage step 2
        Sf = F.T @ (shadow.T - sample[:, None])
        ms = ((Sf[0] > bottom) & (Sf[0] < bottom + d) & (Sf[1] > center - w / 2.0) & (Sf[1] < center + w / 2.0) & (Sf[2] > -1.0 * h) & (Sf[2] < h))
        Sf = Sf[:, ms]
        sproj = np.stack([(Sf[0] - bottom) / d, (Sf[1] - (center - w / 2.0)) / w, (Sf[2] + h) / (2.0 * h)])
    for i, swap in enumerate([None, (0, 2), (1, 2)]):
        if swap:
            proj[[swap[0], swap[1]]] = proj[[swap[1], swap[0]]]
            if sproj is not None:
                sproj[[swap[0], swap[1]]] = sproj[[swap[1], swap[0]]]
        vert = np.minimum(np.floor(proj[0] / cellsize).astype(np.int64), S - 1)
        horiz = np.minimum(np.floor(proj[1] / cellsize).astype(np.int64), S - 1)
        cells = horiz + vert * S
        if channels == 1:
            return _depth_image(proj, cells)[:, :, None]
        out.append(_normals_image(N, cells))
        if channels == 3:
            return out[0]
        out.append(_depth_image(proj, cells)[:, :, None])
        if sproj is not None:
            sv = np.minimum(np.floor(sproj[0] / cellsize).astype(np.int64), S - 1)
            sh = np.minimum(np.floor(sproj[1] / cellsize).astype(np.int64), S - 1)
            out.append(_shadow_image(sproj, sh + sv * S)[:, :, None])
    return np.concatenate(out, axis=2)


@pytest.mark.parametrize("scene,channels", [("krylon", 12), ("krylon", 3), ("krylon", 1), ("table", 12)])
def test_oracle_images_match_a_cv2_restatement(scene, channels):
    c = scenes.krylon_cloud() if scene == "krylon" else scenes.synthetic_table_scene(7, n_points=60000, two_cameras=True)
    oc = oracle.OracleCloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    p = abi.default_params(channels)
    sidx = scenes.sample_indices(2 if scene == "krylon" else 3, len(c["xyz"]), 60 if scene == "krylon" else 150)
    frames, valid = oc.frames(p, sidx)
    poses, flags = oc.hand_search(p, sidx, frames, valid)
    cand = poses.reshape(-1)[(flags.reshape(-1) & 3) == 3][:25]
    assert len(cand) >= 10
    imgs = oc.images(p, cand)
    bad_pixels = total = 0
    for pose, got in zip(cand, imgs):
        q = np.array(pose["sample"], np.float32)
        idx, _ = oc.radius_search(q, 0.10)                                        # image_generator.cpp:43-46,61
        want = reference_image(pose, c["xyz"][idx].astype(np.float64), c["normals"][idx], channels)
        d = np.abs(want.astype(np.int32) - got.astype(np.int32))
        assert d.max() <= 1
        bad_pixels += int(np.count_nonzero(d))
        total += d.size
    assert bad_pixels <= 1e-4 * total, (bad_pixels, total)


@pytest.mark.parametrize("two_cameras", [False, True])
def test_oracle_15_channel_images_match_the_spec_restatement(two_cameras):
    """All 15 channels: the point channels as above plus the occlusion channels, whose point set follows the
    deterministic variant SPECIFIED in include/gpd_b200_shadow.h — restated here in numpy from that header (LCG draws,
    float64 voxel arithmetic, per-camera sets and their intersection, hashed Gaussian jitter) and rasterised by a
    line-by-line createShadowImage with real OpenCV calls. (The reference's own shadow is irreproducible, DESIGN.md 2.)"""
    c = scenes.synthetic_table_scene(5 if two_cameras else 7, n_points=60000, two_cameras=two_cameras)
    oc = oracle.OracleCloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
    p = abi.default_params(15)
    sidx = scenes.sample_indices(3, 60000, 150)
    frames, valid = oc.frames(p, sidx)
    poses, flags = oc.hand_search(p, sidx, frames, valid)
    cand = poses.reshape(-1)[(flags.reshape(-1) & 3) == 3][:10]
    assert len(cand) >= 6
    imgs = oc.images(p, cand)
    bad = total = 0
    for pose, got in zip(cand, imgs):
        idx, _ = oc.radius_search(np.array(pose["sample"], np.float32), 0.10)
        sh = shadow_points(c, idx, int(pose["sample_index"]))
        want = reference_image(pose, c["xyz"][idx].astype(np.float64), c["normals"][idx], 15, shadow=sh)
        assert want.shape == got.shape == (60, 60, 15)
        d = np.abs(want.astype(np.int32) - got.astype(np.int32))
        assert d.max() <= 1
        assert (got[:, :, 4::5] > 0).any()                    # the occlusion channels are not trivially empty
        bad += int(np.count_nonzero(d))
        total += d.size
    assert bad <= 1e-4 * total, (bad, total)
