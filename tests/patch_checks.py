"""What the voice-patch tests share: the reference's oscillator tables on both sides, the comparison bars, which state words are
integral, which stages own delay lines, and stage kinds a patch refuses."""
import numpy as np

import golden_checks as G
from maximilian_b200 import capi
from maximilian_b200.patchdef import OP, PatchDef, R

# state words that hold integral members (envelope flags and hold counts, maxiEnvGen segment / play state / counter, delay ring indices):
# exact whatever the patch
INT_SLOTS = {OP["env_adsr"]: (2, 3), OP["env_ar"]: (2, 3), OP["envgen"]: (1, 2, 4), OP["delay"]: (0,), OP["flanger"]: (0,), OP["chorus"]: (0, 1)}


def set_tables(port, library=True):
    """sineBuffer / transition of the golden fixture, to the C port and (library=True, needs a GPU) to the library"""
    g = G.load("tables")
    port.set_tables(g["sine"], g["transition"], float(g["sine_before"]), "port")
    if library:
        capi.set_tables(g["sine"], g["transition"], float(g["sine_before"]))


def cmp(got, ref, exact, what):
    """bit for bit, or 1e-9 relative + 1e-12"""
    if exact:
        assert np.array_equal(got, ref, equal_nan=True), f"{what}: not bit-identical, max abs err {np.nanmax(np.abs(got - ref))}"
    else:
        np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-12, err_msg=what)


def ring_stages(d):
    """(stage, delay lines it owns) of every delay, flanger and chorus stage"""
    return [(si, 2 if op == OP["chorus"] else 1) for si, (op, *_) in enumerate(d.stages) if op in (OP["delay"], OP["flanger"], OP["chorus"])]


# stage kinds mxb_patch_create refuses (ENVGEN: kind 4 of a patch with one shape; mxb_patch_codegen accepts shapes 0..3)
BAD_KINDS = [("osc", -1), ("osc", 12), ("osc", 42), ("filter", 0), ("filter", 3), ("filter", 4), ("filter", 8), ("biquad", -1), ("biquad", 7),
             ("nonlin", -1), ("nonlin", 6), ("envgen", -1), ("envgen", 4)]


def bad_kind_patch(op, kind):
    """one stage of `op` with a kind mxb_patch_create refuses, into the output"""
    d = PatchDef()
    if op == "envgen":
        d.envgen([0.0, 1.0], [1.0], [1.0])
    d.stage(op, d.K(1.0), d.K(2.0), d.K(3.0), kind=kind, dst=R(0))
    d.stage("out", R(0))
    return d
