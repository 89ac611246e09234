"""The detection front end's configuration matrix (front_scenes) covers what test_front_matrix_gpu claims it covers: every two stream
configurations in one tick, every tick-wide switch in both states, the frame budget, every edge case, and a launch rule that names a
kernel for each switch.  Guards the matrix against shrinking when layouts or schedules are edited."""
import itertools

import front_scenes as fs


def test_twelve_configurations():
    """3 tables x own values x deskew; separate rigs of 2 or 3 sensors, merging rigs of 2 to 4"""
    assert len(fs.CONFIGS) == 12
    for name, c in fs.CONFIGS.items():
        assert fs.config_name(c["table"], c["own"], c["dsk"]) == name
        assert {"none": (0, 0), "sep": (2, 3), "merge": (2, 4)}[c["table"]][0] <= c["n_sensors"] <= \
            {"none": (0, 0), "sep": (2, 3), "merge": (2, 4)}[c["table"]][1], name
    # the own values move the fields whose loss changes boxes
    assert {"sensor_height", "t_hmin", "t_hmax", "h_sensor", "min_cluster_points"} <= set(fs.OWN)


def test_every_pair_shares_a_tick():
    """a pair that never shares a tick would leave a wrong OR over the groups unseen for it"""
    want = {tuple(sorted(p)) for p in itertools.combinations(fs.CONFIGS, 2)}
    assert want - fs.pairs_covered() == set()


def test_frame_budget_and_layouts():
    """every layout fits lmot_seq_set_sensors' budget of 8 frames and names each configuration at most once"""
    for lay in fs.LAYOUTS:
        assert sum(fs.frames_of(n) for n in lay) <= fs.MAX_FRAMES, lay
        assert len(set(lay)) == len(lay) and all(n in fs.CONFIGS for n in lay), lay
    assert fs.OVER_MAX["sensors"] + 1 <= fs.MAX_FRAMES
    for tk in fs.OVER_MAX["ticks"]:
        assert len(tk) == len(fs.OVER_MAX["layout"])
    for _, _, lay, tk in fs.all_ticks():
        assert len(tk) == len(lay) and set(tk) <= set("FReEL-") and any(c != "-" for c in tk), (lay, tk)


def test_every_switch_in_both_states():
    """rigged, own_det, merging, deskew, rig_fit and gf each seen on and off across the matrix's FRAMES ticks"""
    states = {}
    for (sw, _), _ in fs.switch_states().items():
        for k, v in sw:
            states.setdefault(k, set()).add(v)
    assert set(states) == {"rigged", "own_det", "merging", "deskew", "rig_fit", "gf"}
    for k, v in states.items():
        assert v == {False, True}, k
    # the launch change of the front-end rewrite: merging without a separate rig, and merging next to one
    seen = {tuple(sorted(sw)) for sw, _ in fs.switch_states()}
    assert any(dict(s)["merging"] and not dict(s)["rig_fit"] and not dict(s)["own_det"] for s in seen)
    assert any(dict(s)["merging"] and dict(s)["rig_fit"] and not dict(s)["own_det"] for s in seen)


def test_edge_cases_present():
    """an empty frame inside a merging rig and inside a separate rig, a tick whose frames are all empty, LISTS entries and a restart
    in mixed ticks, and a merged cloud above max_points"""
    found = dict(empty_in_merge=False, empty_in_sep=False, all_empty=False, lists_mixed=False, restart_mixed=False)
    for _, _, lay, tk in fs.all_ticks():
        cf, empty, lists = fs.tick_cfgs(lay, tk)
        for n, c in zip(lay, tk):
            if c == "e" and fs.CONFIGS[n]["table"] == "merge":
                found["empty_in_merge"] = True
            if c == "e" and fs.CONFIGS[n]["table"] == "sep":
                found["empty_in_sep"] = True
        found["all_empty"] |= fs.all_empty(cf, empty) and len(cf) > 1
        found["lists_mixed"] |= lists and len(cf) > 1
        found["restart_mixed"] |= "R" in tk and len(cf) > 1
    assert all(found.values()), found
    assert fs.OVER_MAX["sensors"] >= 7 and fs.OVER_MAX["layout"][1] == "none"


def test_launch_rule():
    """the rule names one ground kernel and one box-fit kernel per FRAMES tick, with the documented precedence"""
    r = fs.launch_rule(["merge"], 0)
    assert "box_fit_kernel<false>" in r and "ccl_dense_kernel" in r and "rig_merge_kernel" in r and "concat_boxes_seq_kernel" in r
    assert "box_fit_kernel<true>" in fs.launch_rule(["merge", "sep"], 0)
    assert "box_fit_frame_kernel" in fs.launch_rule(["sep", "none+own"], 0)
    assert fs.launch_rule(["none"], 0) == sorted(["ground_fused_kernel", "tile_hist_kernel", "scatter_kernel", "box_fit_kernel<false>"])
    assert "seg_offsets_kernel" in fs.launch_rule(["none", "sep"], 1, empty=["none", "sep"])
    # deskew runs on the points it has: none when the deskewing streams' frames are all empty
    assert "deskew_points_kernel" not in fs.launch_rule(["none+dsk", "sep"], 0, empty=["none+dsk"])
    assert "deskew_points_kernel" in fs.launch_rule(["none+dsk", "sep"], 0, empty=["sep"])
    assert fs.launch_rule([], 1, lists=True) == ["boxes_to_global_seq_kernel", "pack_lists_seq_kernel"]
    for (sw, empty), (i, t, gf) in fs.switch_states().items():
        cf, e, lists = fs.tick_cfgs(fs.LAYOUTS[i], fs.schedule(fs.LAYOUTS[i])[t])
        r = fs.launch_rule(cf, gf, e, lists)
        assert sum(x.startswith("ground_fused") for x in r) == 1 and sum(x.startswith("box_fit") for x in r) == 1, r
    assert fs.kernel_key("void lmot::box_fit_kernel<256, false>(lmot::FitBatch, lmot::BoxParams)") == "box_fit_kernel<false>"
    assert fs.kernel_key("void lmot::(anonymous namespace)::ground_fused_rig_kernel(lmot::GroundBatch)") == "ground_fused_rig_kernel"
    assert fs.kernel_key("void lmot::publish_seq_kernel(lmot::PubSeq)") is None
