"""Control events (MXB_IN_EVENTS) without a device: the generated source of a patch with events streams compiles for sm_90a with NVRTC,
the stream kind is part of that source (and so of the cubin cache key), a patch without events streams gets the source it always got,
and the host-side helpers restate the definition of include/maxib200.h."""
import numpy as np
import pytest

import events_checks as EV
from maximilian_b200 import capi
from maximilian_b200 import workloads as W
from maximilian_b200.patchdef import PatchDef, R


@pytest.mark.parametrize("case", EV.CASES, ids=lambda c: c[0])
def test_events_patch_compiles_for_sm90a(case):
    name, build, values, taps = case
    src = capi.patch_codegen(build("events"), compile=True)
    head, loop = src.split("for (int t = 0", 1)
    assert "ev_start(a.ev[0], vv, live, ec0, en0);" in head
    assert "ev_advance(a.ev[0], vv, t, h0, ec0, en0);" in loop and "const double i0 = h0;" in loop
    assert "a.held[(size_t)0 * V + (size_t)v] = h0;" in loop.rsplit("if (live) {", 1)[1]


def test_stream_kind_is_part_of_the_program():
    srcs = {ty: capi.patch_codegen(EV._frequency(ty)) for ty in ("f64", "u8", "bits", "events")}
    assert len(set(srcs.values())) == 4
    for ty in ("f64", "u8", "bits"):
        assert "ev_" not in srcs[ty] and "a.held" not in srcs[ty]


def test_unused_events_streams_still_move_their_held_values():
    """an events stream no stage reads is advanced all the same (its held value is state), numbered among the events streams only"""
    d = PatchDef()
    d.IN("dense")
    d.IN("unused", "events")
    d.stage("osc", d.IN("used", "events"), kind="saw", dst=R(0))
    d.stage("out", R(0))
    src = capi.patch_codegen(d, compile=True)
    assert "ev_advance(a.ev[0], vv, t, h1, ec1, en1);" in src and "const double i1" not in src
    assert "ev_advance(a.ev[1], vv, t, h2, ec2, en2);" in src and "const double i2 = h2;" in src


def test_source_of_patches_without_events_is_unchanged():
    """the generator's text for patches without events streams, pinned by a digest of the parent's output for the bench's patches"""
    import hashlib
    digests = {ty: hashlib.sha256(capi.patch_codegen(W.polysynth_patch(ty)).encode()).hexdigest()[:16] for ty in ("f64", "u8", "bits")}
    assert digests == GOLDEN_DIGESTS


def test_events_type_is_accepted_and_the_next_one_refused():
    import ctypes as C
    desc, keep = capi._patch_desc(EV._frequency("events"), 1, 1, 1)
    need = C.c_int64(0)
    assert desc.input_types[0] == 3 and capi.lib().mxb_patch_codegen(C.byref(desc), None, 0, C.byref(need), 0) == 0
    desc.input_types[0] = 4
    assert capi.lib().mxb_patch_codegen(C.byref(desc), None, 0, C.byref(need), 0) == -1


def test_held_accessors_refuse_a_null_patch():
    a = np.zeros(4)
    assert capi.lib().mxb_patch_get_held(None, 0, capi._np_ptr(a), capi.MEM_HOST) == -1
    assert capi.lib().mxb_patch_set_held(None, 0, capi._np_ptr(a), capi.MEM_HOST) == -1


def test_pack_events_keeps_each_voices_order():
    first, frame, value = capi.pack_events([[(5, 1.0), (2, 2.0)], [], [(0, 3.0)]])
    assert first.tolist() == [0, 2, 2, 3] and frame.tolist() == [5, 2, 0] and value.tolist() == [1.0, 2.0, 3.0]
    assert first.dtype == np.int32 and frame.dtype == np.int32 and value.dtype == np.float64


def test_dense_equivalent_follows_the_definition():
    """events_to_dense, which the GPU tests hold both kernels to, against a direct reading of the definition on random lists"""
    rng = np.random.default_rng(2)
    for _ in range(200):
        V, n = int(rng.integers(1, 30)), int(rng.integers(1, 25))
        lists = EV.random_events(rng, V, n)
        held = rng.normal(size=V)
        dense, h = EV.events_to_dense(*capi.pack_events(lists), n, held)
        for v, evs in enumerate(lists):
            cur, at, col = held[v], 0, np.empty(n)
            when = []
            for f, x in evs:                                   # event i at max(frame_i, frame of event i-1), frame < 0 -> 0
                at = max(at, f, 0)
                when.append((at, x))
            for t in range(n):
                for w, x in when:
                    if w == t:
                        cur = x
                col[t] = cur
            assert np.array_equal(dense[:, v], col) and h[v] == col[-1]


# sha256 prefixes of the source the parent commit generated for W.polysynth_patch(ty)
GOLDEN_DIGESTS = {"f64": "757ea5f1e5a35ecd", "u8": "f181c6a3c46c0a72", "bits": "7824448d7667389a"}
