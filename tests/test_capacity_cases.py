"""CPU proofs of the capacity-edge inputs (tests/capacity_cases.py): each case puts exactly its target number of points
into the list whose size decides the tier, counted independently of the kernels — the float32 ball with numpy and with
the oracle's radius search, the hand-height slab in float64 with the oracle's frame, the image box in float64."""
import numpy as np
import pytest

import capacity_cases as cc
from gpd_b200 import abi
from oracle import oracle

FRAME_EDGES = [cc.FRAMES_CAP0, cc.FRAMES_CAP0 + 1, cc.FRAMES_CAP1, cc.FRAMES_CAP1 + 1, cc.FRAMES_CAP2, cc.FRAMES_CAP2 + 1]
HAND_EDGES = [cc.HANDS_CAP1, cc.HANDS_CAP1 + 1, cc.HANDS_CAP2, cc.HANDS_CAP2 + 1]
BOX_EDGES = [cc.BOX_CAP2, cc.BOX_CAP2 + 1, cc.BOX_CAP, cc.BOX_CAP + 1]


def test_caps_mirror_the_kernels():
    assert cc.BALL_CAP2 == 3600 and cc.WL_CAP2 == 1440 and cc.WL_CAP == 2880 and cc.DL_CAP == 7200
    # k_images2's voxel stash: the default 15-channel bitmap (48^2 x 2 words) at one camera, and 46^2 at two
    # (volume_depth 0.05); shared memory first (ST_SM), then 1 800 entries in the image's HBM slot (ST_CAP)
    assert cc.st_sm2(48, 1) == 2304 and cc.st_cap2(48, 1) == 4104
    assert cc.st_sm2(46, 2) == 376 and cc.st_cap2(46, 2) == 2176
    # k_images' voxel list behind bitmap 0 (BL_CAP): 13 824 at the default geometry, 12 600 at volume_height 0.04
    assert cc.bl_cap(cc.bm_dim(), 1) == 13824 and cc.bl_cap(cc.bm_dim(volume_height=0.04), 1) == 12600
    # k_images2 takes two cameras up to bm_dim 46 (volume_depth 0.05); 47 (volume_depth 0.055) goes to k_images
    assert cc.fast_path_15(cc.bm_dim(volume_depth=0.05), 2) and not cc.fast_path_15(cc.bm_dim(volume_depth=0.055), 2)
    assert cc.bm_dim(volume_depth=0.05) == 46 and cc.bm_dim(volume_depth=0.055) == 47


@pytest.mark.parametrize("n,at_position", [(n, False) for n in FRAME_EDGES] +
                         [(cc.FRAMES_CAP1, True), (cc.FRAMES_CAP1 + 1, True)])
def test_frames_ball_counts(n, at_position):
    cloud, si, pos, plane = cc.frames_ball(n, at_position)
    q = pos.astype(np.float32) if at_position else cloud["xyz"][si]
    assert cc.ball_count(cloud["xyz"], q, cc.R_LRF) == n
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"])
    assert len(oc.radius_search(q, cc.R_LRF)[0]) == n
    for i in plane[:5]:  # the plane samples stay in tier 0
        assert cc.ball_count(cloud["xyz"], cloud["xyz"][i], cc.R_LRF) <= cc.FRAMES_CAP0


@pytest.mark.parametrize("n", HAND_EDGES)
def test_hand_cylinder_counts(n):
    cloud, si = cc.hand_cylinder(n)
    q = cloud["xyz"][si]
    assert cc.ball_count(cloud["xyz"], q, cc.R_HS) == n
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    assert len(oc.radius_search(q, cc.R_HS)[0]) == n
    for axes in ([2], [0, 1, 2]):
        p = abi.default_params(15, hand_axes=axes)
        fr, fv = oc.frames(p, [si])
        assert fv[0] == 1
        if axes == [2]:
            assert cc.slab_count(cloud, si, fr[0]) == n
        poses, flags = oc.hand_search(p, [si], fr, fv)
        assert ((flags & 3) == 3).any(), "no VALID | FILTERED pose: the case would not exercise the hand search"


@pytest.mark.parametrize("n", [cc.SURV_CAP, cc.SURV_CAP + 1])
def test_hand_cylinder_closing_region_counts(n):
    """The whole cylinder lies in the closing region of every valid pose: n members, the count SURV_CAP decides on."""
    cloud, si = cc.hand_cylinder(n)
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    p = abi.default_params(15)
    fr, fv = oc.frames(p, [si])
    poses, flags = oc.hand_search(p, [si], fr, fv)
    assert ((flags & 3) == 3).any()
    c = cc.closing_counts(cloud, si, poses[0], flags[0])
    assert (c[(flags[0] & 1) == 1] == n).all(), c


@pytest.mark.parametrize("n", BOX_EDGES + [cc.BOX_CAP_GL, cc.BOX_CAP_GL + 1])
def test_image_box_counts(n):
    cloud, pose = cc.image_box(n, n_outside=100)
    assert cc.box_count(cloud, pose) == n
    q = pose["sample"][0].astype(np.float32)
    assert cc.ball_count(cloud["xyz"], q, cc.R_IMG) == n + 100
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"])
    assert len(oc.radius_search(q, cc.R_IMG)[0]) == n + 100


@pytest.mark.parametrize("n_ball", [cc.BALL_CAP2, cc.BALL_CAP2 + 1])
def test_image_in_ball_counts(n_ball):
    cloud, pose = cc.image_box(1000, n_outside=n_ball - 1000)
    assert cc.box_count(cloud, pose) == 1000
    assert cc.ball_count(cloud["xyz"], pose["sample"][0].astype(np.float32), cc.R_IMG) == n_ball
