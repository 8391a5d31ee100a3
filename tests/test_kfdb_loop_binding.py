"""The loop query's entry point is typed from the header and refuses a call without a handle on the host, before any device work (no GPU)."""
import ctypes as C

from pysgs import binding as B


def test_loop_entry_point_is_typed_and_refuses_on_the_host():
    P, I = C.c_void_p, C.c_int32
    L = B.lib()
    assert L.sgs_kfdb_loop_candidates_device.argtypes == [P, I, P, P, P, P, I, P, P, P, P, P, P, P, P, I, P, P, P, P]
    assert L.sgs_kfdb_loop_candidates_device.restype == C.c_int
    assert L.sgs_kfdb_loop_candidates_device(None, 1, None, None, None, None, 1, None, None, None, None, None, None, None, None, 1, None, None, None,
                                             None) == B.SGS_ERR_INVALID
