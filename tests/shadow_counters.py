"""The shadow counters one gpdb_images call must show, from the restatement of tests/shadow_cast_reference.py: event slots
9 / 10 / 11 / 14 of gpdb_debug_phase_cycles and the shadow path counters of gpdb_debug_path_counts, per image, for the
kernel that makes it (k_images2 or k_images)."""
import capacity_cases as cc
import shadow_cast_reference as scr

IMAGES2_EVENTS = ["images2_cast_in_place", "images2_draw_in_place", "images2_stash_full"]
IMAGES_EVENTS = ["images_cast_in_place", "images_draw_in_place", "images_voxel_list_full", "images_ball_record_full"]


def counted_images(ctx, poses, forced, monkeypatch):
    """(images, path counters, event slots) of one gpdb_images call, k_images alone when forced."""
    if forced:
        monkeypatch.setenv("GPD_B200_IMAGES_KERNEL", "1")
    try:
        ctx.phase_cycles(1)
        img = ctx.images(poses)
        paths = ctx.path_counts()
        slots = ctx.phase_cycles(0)
    finally:
        monkeypatch.delenv("GPD_B200_IMAGES_KERNEL", raising=False)
    return img, paths, slots


def expected(r, g, box_n, forced, maxk=None):
    """The counters one image adds, from its restatement r: which kernel makes it (k_images2 unless forced, outside the
    fast path's geometry or with more than BOX_CAP2 box points), the capped sums of slots 9 / 10 / 11 and the excess
    of every list. Slot 10 is a (least, most) pair: exact unless a work list overflows with unequal windows. maxk: the
    largest camera count of the call (a batch), which sizes the launch: the fast-path choice and k_images' voxel list
    follow it, k_images2's stash follows the image's own camera count."""
    K, P = r["K"], scr.Params(g)
    maxk = K if maxk is None else maxk
    fast = not forced and cc.fast_path_15(P.bm_dim, maxk) and box_n <= cc.BOX_CAP2
    wl_cap = cc.WL_CAP2 if fast else cc.WL_CAP
    ev = {e: 0 for e in IMAGES2_EVENTS + IMAGES_EVENTS}
    pre = "images2_" if fast else "images_"
    s9, lo10, hi10 = 0, 0, 0
    for k in range(K):
        if r["cams"][k] is None:
            continue
        s9 += min(r["wl_n"][k], wl_cap)
        ev[pre + "cast_in_place"] += max(r["wl_n"][k] - wl_cap, 0)
        lo, hi = scr.listed_draws_bounds(r, k, wl_cap)
        lo10, hi10 = lo10 + lo, hi10 + hi
        ev[pre + "draw_in_place"] += max(lo - cc.DL_CAP, 0) if lo == hi else 0
    if fast:
        ev["images2_stash_full"] = int(r["nset_all"] > cc.st_cap2(P.bm_dim, K))
        walks = sum(c is not None for c in r["cams"]) if r["n_ball"] > cc.BALL_CAP2 else 0
    else:
        ev["images_voxel_list_full"] = int(r["nset_all"] > cc.bl_cap(P.bm_dim, maxk))
        ev["images_ball_record_full"] = int(r["n_ball"] > 2 * g.S * g.S)
        walks = 0
    return {"fast": fast, "s9": s9, "s10": (lo10, hi10), "s11": r["nset_all"], "events": ev, "walks": walks}


def assert_counters(exp, paths, slots):
    assert int(slots[9]) == exp["s9"], (int(slots[9]), exp["s9"])
    lo, hi = exp["s10"]
    assert lo <= int(slots[10]) <= hi, (int(slots[10]), exp["s10"])
    assert int(slots[11]) == exp["s11"], (int(slots[11]), exp["s11"])
    for e, v in exp["events"].items():
        if e.endswith("draw_in_place") and lo != hi:
            continue
        assert paths[e] == v, (e, paths[e], v)
    assert paths["images2_box"] == 0 and paths["images2_nonunit"] == 0
    assert int(slots[14]) == exp["walks"], (int(slots[14]), exp["walks"])
