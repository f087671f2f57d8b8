"""Host-side pieces of ObjectMotion.track that need no GPU: the C structs' layout as capi mirrors it, and synth's parked objects."""
import ctypes as C

import numpy as np

from vdo_slam_b200 import capi
from vdo_slam_b200.synth import make_sequence_frame


def test_track_structs_match_the_library():
    L = capi.load()
    assert L.vdo_abi_struct_size(b"vdo_obj_track_opts") == C.sizeof(capi.ObjTrackOpts)
    assert L.vdo_abi_struct_size(b"vdo_obj_track_out") == C.sizeof(capi.ObjTrackOut)
    # the track outputs are the motion outputs (first, as one struct) and then the table's own entries, in table order
    assert [k for k, _ in capi.ObjTrackOut._fields_] == ["motion"] + [k + "_dev" for k in capi._OT_OUT if k not in capi._OM_OUT]


def test_parked_objects_draw_the_same_random_numbers():
    kw = dict(seed=3, width=320, height=120, n_obj=4)
    a, b = make_sequence_frame(2, **kw), make_sequence_frame(2, parked=(), **kw)
    for k in ("gray", "depth_raw", "flow", "mask"):
        assert np.array_equal(a[k], b[k]), k
    p0 = make_sequence_frame(0, parked=(2,), **kw)
    q0 = make_sequence_frame(0, **kw)
    assert np.array_equal(p0["mask"], q0["mask"])                    # at t = 0 nothing has moved yet
    assert np.array_equal(p0["depth_raw"] == -1, q0["depth_raw"] == -1)  # the same noise draws
    assert np.allclose(p0["obj_vel"][2], 0) and not np.allclose(q0["obj_vel"][2], 0)
