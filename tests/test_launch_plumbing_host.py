"""The diagnostic forward entry points (pilco_mm_forward_profile, pilco_mm_forward_taped_profile) make the argument
checks of pilco_mm_forward / pilco_mm_forward_taped, checked WITHOUT a GPU: a call with R < 1, or with a workspace or
tape that the TMA bulk copies could not read (not 16-byte aligned), is rejected before anything is enqueued.  Pointers
are fake non-null addresses, as in test_abi_errors.py; only rejecting calls are made."""
import ctypes as C

from pilco_b200._lib import lib
from abi_fakes import ERR_ALIGN, ERR_DIM, ERR_NULL, FAKE, _gp

BIG = 1 << 30
MS = (C.c_float * 3)()          # the timings (host memory); a rejected call never writes them


def _profile(R=1, ws=FAKE, ms_out=MS):
    g = _gp()
    return lib.pilco_mm_forward_profile(C.byref(g), R, FAKE, FAKE, FAKE, FAKE, FAKE, None, ws, BIG, ms_out, None)


def _taped_profile(R=1, ws=FAKE, tape=FAKE, ms_out=MS):
    g = _gp()
    return lib.pilco_mm_forward_taped_profile(C.byref(g), R, FAKE, FAKE, FAKE, FAKE, FAKE, None, ws, BIG, tape, BIG,
                                              ms_out, None)


def test_profile_entry_points_reject_empty_batches():
    assert _profile(R=0) == ERR_DIM
    assert _taped_profile(R=0) == ERR_DIM


def test_profile_entry_points_reject_misaligned_buffers():
    assert _profile(ws=FAKE + 8) == ERR_ALIGN
    assert _taped_profile(ws=FAKE + 8) == ERR_ALIGN
    assert _taped_profile(tape=FAKE + 8) == ERR_ALIGN


def test_profile_entry_points_still_need_their_timing_output():
    assert _profile(ms_out=None) == ERR_NULL
    assert _taped_profile(ms_out=None) == ERR_NULL
