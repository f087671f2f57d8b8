"""Host-side pieces of ObjectMotion.renew that need no GPU: the feature set's layout as capi mirrors it, and its status bits."""
import ctypes as C

from vdo_slam_b200 import capi


def test_feature_set_struct_matches_the_library():
    L = capi.load()
    assert L.vdo_abi_struct_size(b"vdo_obj_feat_set") == C.sizeof(capi.ObjFeatSet)
    assert [k for k, _ in capi.ObjFeatSet._fields_] == [k + "_dev" for k in capi._OS_SET]
    assert list(capi._OS_SET) == ["x", "y", "label", "depth", "cx", "cy", "flow", "inlier_id", "obj_label", "point", "count", "status"]


def test_pair_status_bits_are_distinct():
    bits = [capi.OM_PAIR_OBJECT_CAP, capi.OM_PAIR_LABEL_RANGE, capi.OM_PAIR_FEATURE_CAP, capi.OM_PAIR_SET_COUNT]
    assert bits == [1, 2, 4, 8]
