"""CPU checks of the independently advancing channels' interface: the C++ program that drives them through the drop-in header
compiles, and the library's ctypes binding declares the new symbols with the argument types of the header."""
import ctypes as C
import os
import re
import subprocess

from maximilian_b200 import capi

ROOT = os.path.dirname(os.path.abspath(__file__))


def test_ragged_streams_program_compiles_against_the_dropin_header(tmp_path):
    from test_cpp_dropin import compile_patch
    exe = compile_patch(tmp_path, os.path.join(ROOT, "cpp", "ragged_streams.cpp"))
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


def test_ragged_symbols_are_exported_and_declared():
    hdr = open(os.path.join(os.path.dirname(ROOT), "include", "maxib200.h")).read()
    for name in ("mxb_stft_process_ragged", "mxb_stft_get_pos", "mxb_istft_process_ragged"):
        assert name in capi.EXPORTS
        assert re.search(r"\b%s\s*\(" % name, hdr), name


def test_ragged_prototypes_take_per_channel_host_arrays():
    L = capi.lib()
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    # (handle, in, stride_c, stride_t, n_samples[C], max_frames, outputs, post, mfcc, n_frames[C], mem, stream)
    f = L.mxb_stft_process_ragged
    assert f.restype is i32
    assert f.argtypes == [vp, vp, i64, i64, vp, i32, C.POINTER(capi.StftOutputs), vp, vp, vp, i32, vp]
    assert L.mxb_stft_get_pos.argtypes == [vp, vp] and L.mxb_stft_get_pos.restype is i32
    # (handle, mags, phases, frames[C], max_frames, out, mem, stream)
    f = L.mxb_istft_process_ragged
    assert f.restype is i32 and f.argtypes == [vp, vp, vp, vp, i32, vp, i32, vp]
