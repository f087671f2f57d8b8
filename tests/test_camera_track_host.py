"""Host-side pieces of CameraMotion that need no GPU: the structs as capi mirrors them, the output tables and the status bits."""
import ctypes as C

from vdo_slam_b200 import capi


def test_structs_match_the_library():
    L = capi.load()
    for name, cls in (("vdo_stat_feat_set", capi.StatFeatSet), ("vdo_stat_opts", capi.StatOpts), ("vdo_cam_track_opts", capi.CamTrackOpts),
                      ("vdo_cam_track_out", capi.CamTrackOut)):
        assert L.vdo_abi_struct_size(name.encode()) == C.sizeof(cls), name
    assert [k for k, _ in capi.StatFeatSet._fields_] == [k + "_dev" for k in capi._SS_SET]
    assert [k for k, _ in capi.CamTrackOut._fields_] == [k + "_dev" for k in capi._CT_OUT]
    assert list(capi._SS_SET) == ["x", "y", "depth", "cx", "cy", "flow", "inlier_id", "point", "count", "status", "Tcw", "velocity", "has_velocity"]
    assert list(capi._CT_OUT) == ["T", "T_init", "velocity", "info", "stats", "status", "flags", "key", "flow_ref"]


def test_status_bits_are_distinct():
    bits = [capi.CAM_FEW_POINTS, capi.CAM_NO_MODEL, capi.CAM_USED_MM, capi.CAM_SET_COUNT, capi.CAM_KEY_COUNT]
    assert bits == [1, 2, 4, 8, 16]


def test_entries_are_exported():
    L = capi.load()
    for name in ("vdo_cam_motion_create", "vdo_cam_motion_destroy", "vdo_cam_motion_info", "vdo_stat_build_batch_dev", "vdo_cam_track_batch_dev",
                 "vdo_stat_renew_batch_dev", "vdo_sample_keys_dev"):
        assert hasattr(L, name), name
