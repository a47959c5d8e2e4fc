"""Calibration and parameter sets of the reference's shipped datasets (values only).

Sources (all under /root/reference/esvo_core/):
  calib/hkust/{left,right}.yaml, calib/dsec/zurich_city_04_a/{left,right}.yaml, calib/rpg/{left,right}.yaml,
  cfg/mapping/mapping_{hkust,dsec}.yaml, cfg/tracking/tracking_{hkust,dsec}.yaml, cfg/mvstereo/mvstereo_{rpg,upenn}.yaml,
  ../esvo_time_surface/cfg/parameters.yaml.
"A" = 346x260 (hkust DAVIS346), "B" = 640x480 (DSEC-shaped), rpg = 240x180 (DAVIS240C).
"""
from __future__ import annotations

import numpy as np

from . import capi

RIGS = {
    "hkust": dict(
        width=346, height=260, model="plumb_bob",
        left=dict(
            K=[263.796, 0, 176.994, 0, 263.738, 124.373, 0, 0, 1],
            D=[-0.386589, 0.157241, 0.000322143, 6.13759e-06],
            R=[0.999809, 0.0161928, 0.0109163, -0.0162088, 0.999868, 0.0013701, -0.0108927, -0.00154678, 0.999939],
            P=[189.705, 0, 165.382, 0, 0, 189.705, 121.295, 0, 0, 0, 1, 0]),
        right=dict(
            # the third row of K really is like this in calib/hkust/right.yaml:7
            K=[263.485, 0, 162.942, 0, 263.276, 118.029, -0.0151344, 0.00133093, 0.999885],
            D=[-0.383425, 0.152823, -0.000257745, 0.000268432],
            R=[0.9993960957463914, 0.0034732142808621717, -0.03457427641222047,
               -0.0035085878889783376, 0.9999933816804096, -0.0009625000798637905,
               0.03457070461958685, 0.0010832257094615543, 0.9994016675011942],
            P=[189.705, 0, 165.382, -13.8634, 0, 189.705, 121.295, 0, 0, 0, 1, 0])),
    "dsec": dict(
        width=640, height=480, model="plumb_bob",
        left=dict(
            K=[553.469, 0, 346.653, 0, 553.399, 216.521, 0, 0, 1],
            D=[-0.0935648, 0.194458, 7.64243e-05, 0.00195639],
            R=[0.999866, -0.00319364, 0.0160517, 0.00322964, 0.999992, -0.00221712, -0.0160445, 0.00226867, 0.999869],
            P=[534.094, 0, 335.446, 0, 0, 534.094, 223.233, 0, 0, 0, 1, 0]),
        right=dict(
            K=[552.182, 0, 336.874, 0, 551.445, 226.326, 0, 0, 1],
            D=[-0.0949368, 0.202115, 0.000582129, 0.00145529],
            R=[0.999963, 0.00818053, -0.00267849, -0.0081745, 0.999964, 0.00225394, 0.00269683, -0.00223196, 0.999994],
            P=[534.094, 0, 335.446, -319.94, 0, 534.094, 223.233, 0, 0, 0, 1, 0])),
    # calib/upenn/{left,right}.yaml -- the reference's equidistant (fisheye) rig
    "upenn": dict(
        width=346, height=260, model="equidistant",
        left=dict(
            K=[226.38018519795807, 0.0, 173.6470807871759, 0.0, 226.15002947047415, 133.73271487507847, 0, 0, 1],
            D=[-0.048031442223833355, 0.011330957517194437, -0.055378166304281135, 0.021500973881459395],
            R=[0.999877311526236, 0.015019439766575743, -0.004447282784398257,
               -0.014996983873604017, 0.9998748347535599, 0.005040367172759556,
               0.004522429630305261, -0.004973052949604937, 0.9999774079320989],
            P=[199.6530123165822, 0.0, 177.43276376280926, 0.0, 0.0, 199.6530123165822, 126.81215684365904, 0.0, 0.0, 0.0, 1.0, 0.0]),
        right=dict(
            K=[226.0181418548734, 0, 174.5433576736815, 0, 225.7869434267677, 124.21627572590607, 0, 0, 1],
            D=[-0.04846669832871334, 0.010092844338123635, -0.04293073765014637, 0.005194706897326005],
            R=[0.9999922706537476, 0.003931701344419404, -1.890238450965101e-05,
               -0.003931746704476347, 0.9999797362744968, -0.005006836150689904,
               -7.83382948021244e-07, 0.0050068717705076754, 0.9999874655386736],
            P=[199.6530123165822, 0.0, 177.43276376280926, -19.941771812941038, 0.0, 199.6530123165822, 126.81215684365904, 0.0,
               0.0, 0.0, 1.0, 0.0])),
    # calib/rpg/{left,right}.yaml -- the stereo DAVIS240C rig of the rpg datasets (esvo_MVStereo's mvstereo_rpg.launch)
    "rpg": dict(
        width=240, height=180, model="plumb_bob",
        left=dict(
            K=[196.639, 0, 105.064, 0, 196.733, 72.4717, 0.0, 0.0, 1.0],
            D=[-0.336733, 0.111789, -0.00140053, -0.000459594],
            R=[0.999791, -0.018779, -0.00802416, 0.0187767, 0.999824, -0.000360707, 0.00802952, 0.000209964, 0.999968],
            P=[156.925, 0, 108.167, 0, 0, 156.925, 78.4205, 0, 0, 0, 1, 0]),
        right=dict(
            K=[196.426, 0, 110.745, 0, 196.564, 88.1131, 0.0, 0.0, 1.0],
            D=[-0.346294, 0.12772, -0.000272051, -0.000195801],
            R=[0.999589, 0.0222217, -0.0181009, -0.0222166, 0.999753, 0.000486491, 0.0181073, -8.41512e-05, 0.999836],
            P=[156.925, 0, 108.167, -23.2327, 0, 156.925, 78.4205, 0, 0, 0, 1, 0])),
}

# cfg/mvstereo/mvstereo_{rpg,upenn}.yaml: the keys of the esvo_MVStereo node (the loop's own keys first, then the
# mapping back-end's).  Values only.  MVStereoMode: 0 PURE_EVENT_MATCHING, 1 PURE_BLOCK_MATCHING, 2 EM_PLUS_ESTIMATION,
# 3 BM_PLUS_ESTIMATION (ESVO's mapper), 4 PURE_SEMI_GLOBAL_MATCHING.  dvs_frame_id comes from the launch file: the rpg
# ground truth is the marker's pose ("marker"), the upenn one the left camera's ("dvs").
MVSTEREO = {k: dict(rpg=a, upenn=b) for k, a, b in [
    #  key                           rpg         upenn
        ("MVStereoMode",              3,          3),
        ("EM_Slice_Thickness",        0.001,      0.001),
        ("EM_Time_THRESHOLD",         0.0005,     0.0005),
        ("EM_EPIPOLAR_THRESHOLD",     1.0,        1.0),
        ("EM_TS_NCC_THRESHOLD",       0.1,        0.1),
        ("EM_NUM_EVENT_MATCHING",     3000,       3000),
        ("BM_half_slice_thickness",   0.001,      0.001),
        ("PROCESS_EVENT_NUM",         1000,       1000),
        ("TS_HISTORY_LENGTH",         100,        100),
        ("mapping_rate_hz",           20,         20),
        ("Denoising",                 True,       False),
        ("dvs_frame_id",              "marker",   "dvs"),
        ("invDepth_min_range",        0.2,        0.16),
        ("invDepth_max_range",        2.0,        1.0),
        ("residual_vis_threshold",    20,         20),
        ("stdVar_vis_threshold",      0.015,      0.15),
        ("age_vis_threshold",         1,          1),
        ("fusion_radius",             0,          0),
        ("FUSION_STRATEGY",           "CONST_FRAMES", "CONST_POINTS"),
        ("maxNumFusionFrames",        40,         40),
        ("maxNumFusionPoints",        5000,       3000),
        ("SmoothTimeSurface",         False,      False),
        ("Regularization",            True,       False),
        ("patch_size_X",              15,         15),
        ("patch_size_Y",              7,          7),
        ("Tdist_nu",                  2.1897,     2.182),
        ("Tdist_scale",               16.6397,    17.277),
        ("BM_min_disparity",          1,          1),
        ("BM_max_disparity",          40,         40),
        ("BM_step",                   1,          1),
        ("BM_ZNCC_Threshold",         0.1,        0.1),
        ("BM_bUpDownConfiguration",   False,      False),
]}


def mvstereo_config(name):
    """The MVSTEREO column of one dataset as a dict."""
    return {k: v[name] for k, v in MVSTEREO.items()}


def mvstereo_params_for(name, lib) -> capi.Params:
    """esvo_params of the esvo_MVStereo node with cfg/mvstereo/mvstereo_<name>.yaml (time surfaces: the ts parameters; the
    node's ITERATION_OPTIMIZATION and regularisation radius / neighbours keep their constructor defaults 10 / 5 / 8 / 8)."""
    c = mvstereo_config(name)
    p = capi.default_params(lib)
    p.decay_ms = 30.0; p.ignore_polarity = 1; p.median_blur_kernel_size = 1
    p.max_event_queue_len = 20; p.time_surface_mode = 0
    p.patch_size_x, p.patch_size_y = c["patch_size_X"], c["patch_size_Y"]
    p.bm_step = c["BM_step"]; p.bm_zncc_threshold = c["BM_ZNCC_Threshold"]; p.bm_updown = int(c["BM_bUpDownConfiguration"])
    p.bm_min_disparity, p.bm_max_disparity = c["BM_min_disparity"], c["BM_max_disparity"]
    p.lsnorm = capi.LSNORM_TDIST; p.max_iteration = 10
    p.td_nu, p.td_scale = c["Tdist_nu"], c["Tdist_scale"]
    p.invdepth_min_range, p.invdepth_max_range = c["invDepth_min_range"], c["invDepth_max_range"]
    p.residual_vis_threshold = c["residual_vis_threshold"]; p.stdvar_vis_threshold = c["stdVar_vis_threshold"]
    p.age_vis_threshold = c["age_vis_threshold"]; p.fusion_radius = c["fusion_radius"]
    p.fusion_strategy = capi.FUSION_CONST_FRAMES if c["FUSION_STRATEGY"] == "CONST_FRAMES" else capi.FUSION_CONST_POINTS
    p.max_num_fusion_frames = c["maxNumFusionFrames"]; p.max_num_fusion_points = c["maxNumFusionPoints"]
    p.smooth_time_surface = int(c["SmoothTimeSurface"]); p.regularization = int(c["Regularization"])
    p.reg_radius, p.reg_min_neighbours, p.reg_min_close_neighbours = 5, 8, 8
    p.num_thread_mapping = 4
    return p


def rig_calibs(name):
    r = RIGS[name]
    mk = lambda c: capi.make_calib(r["width"], r["height"], r["model"], c["K"], c["D"], c["R"], c["P"])
    return mk(r["left"]), mk(r["right"])


def rig_arrays(name):
    r = RIGS[name]
    out = {"width": r["width"], "height": r["height"]}
    for side in ("left", "right"):
        c = r[side]
        out[side] = dict(K=np.array(c["K"], float).reshape(3, 3), D=np.array(c["D"], float),
                         R=np.array(c["R"], float).reshape(3, 3), P=np.array(c["P"], float).reshape(3, 4))
    return out


def params_for(name, lib) -> capi.Params:
    """cfg/mapping/mapping_<name>.yaml + cfg/tracking/tracking_<name>.yaml + ts parameters."""
    p = capi.default_params(lib)
    # esvo_time_surface/cfg/parameters.yaml
    p.decay_ms = 30.0; p.ignore_polarity = 1; p.median_blur_kernel_size = 1
    p.max_event_queue_len = 20; p.time_surface_mode = 0
    p.patch_size_x, p.patch_size_y = 15, 7
    p.bm_step = 1; p.bm_zncc_threshold = 0.1; p.bm_updown = 0
    p.lsnorm = capi.LSNORM_TDIST; p.max_iteration = 10  # ITERATION_OPTIMIZATION is never set -> 10
    p.age_vis_threshold = 1
    p.fusion_strategy = capi.FUSION_CONST_FRAMES
    p.num_thread_mapping = 4
    # tracking (identical in hkust/dsec except batch size and ranges)
    p.trk_patch_size_x = p.trk_patch_size_y = 1; p.trk_kernel_size = 5
    p.trk_lsnorm = capi.TRK_HUBER; p.trk_huber_threshold = 50.0
    p.trk_max_registration_points = 2000; p.trk_max_iteration = 10; p.trk_min_num_events = 1000
    if name == "hkust":
        p.invdepth_min_range, p.invdepth_max_range = 0.25, 2.0
        p.residual_vis_threshold = 20; p.stdvar_vis_threshold = 0.15
        p.fusion_radius = 0; p.max_num_fusion_frames = 20; p.max_num_fusion_points = 4000
        p.smooth_time_surface = 0
        p.regularization = 1  # Regularization: True; radius/min-neighbours keep the ctor defaults 5/8/8
        p.reg_radius, p.reg_min_neighbours, p.reg_min_close_neighbours = 5, 8, 8
        p.td_nu, p.td_scale = 2.1897, 16.6397
        p.bm_min_disparity, p.bm_max_disparity = 1, 40
        p.trk_batch_size = 500
    elif name == "dsec":
        p.invdepth_min_range, p.invdepth_max_range = 0.001, 0.25
        p.residual_vis_threshold = 30; p.stdvar_vis_threshold = 1.0
        p.fusion_radius = 1; p.max_num_fusion_frames = 5; p.max_num_fusion_points = 20000
        p.smooth_time_surface = 1
        p.regularization = 1
        p.reg_radius, p.reg_min_neighbours, p.reg_min_close_neighbours = 20, 32, 32
        p.td_nu, p.td_scale = 2.182, 17.277
        p.bm_min_disparity, p.bm_max_disparity = 0, 150
        p.trk_batch_size = 300
    elif name == "upenn":   # cfg/mapping/mapping_upenn.yaml, cfg/tracking/tracking_upenn.yaml
        p.invdepth_min_range, p.invdepth_max_range = 0.16, 1.0
        p.residual_vis_threshold = 20; p.stdvar_vis_threshold = 0.15
        p.fusion_radius = 0; p.max_num_fusion_frames = 40; p.max_num_fusion_points = 3000
        p.smooth_time_surface = 0; p.regularization = 0
        p.td_nu, p.td_scale = 2.182, 17.277
        p.bm_min_disparity, p.bm_max_disparity = 1, 40
        p.trk_batch_size = 300
    else:
        raise KeyError(name)
    return p
