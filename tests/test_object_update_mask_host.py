"""Host-side pieces of ObjectMotion.update_mask that need no GPU: the output struct's layout as capi mirrors it."""
import ctypes as C

from vdo_slam_b200 import capi


def test_update_mask_struct_matches_the_library():
    L = capi.load()
    assert L.vdo_abi_struct_size(b"vdo_obj_mask_out") == C.sizeof(capi.ObjMaskOut)
    assert [k for k, _ in capi.ObjMaskOut._fields_] == [k + "_dev" for k in capi._OU_OUT]
    assert list(capi._OU_OUT) == ["label", "n_vote", "vote", "recovered", "n_samples", "pair_status"]
