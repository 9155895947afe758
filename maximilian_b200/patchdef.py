"""Stage lists of voice patches (include/maxib200.h: mxb_stage / mxb_patch_desc), host side, numpy-free.

A PatchDef is what a reference play() body looks like once it is written down as data: stages over 16 per-voice registers,
operands that are registers, per-voice parameters, scalar constants or per-sample input streams. The same PatchDef drives
the GPU (capi.Patch) and, in the tests, both CPU oracles (oracle_py.Patch): one description, three executors.
"""
OP = dict(osc=1, env_adsr=2, env_ar=3, envgen=4, filter=5, svf=6, biquad=7, dcblock=8, nonlin=9, delay=10, flanger=11,
          add=12, sub=13, mul=14, div=15, mix_stereo=16, out=17, chorus=18)
OSC = dict(sinewave=0, coswave=1, phasor=2, saw=3, square=4, pulse=5, impulse=6, triangle=7, phasorbetween=8, sinebuf=9, sinebuf4=10, sawn=11)
FILT = dict(lores=1, hires=2, lopass=5, hipass=6, bandpass=7)
BIQUAD = dict(lowpass=0, highpass=1, bandpass=2, notch=3, peak=4, lowshelf=5, highshelf=6)
NONLIN = dict(atandist=0, fastatandist=1, softclip=2, hardclip=3, asymclip=4, fastatan=5)
DELAY = dict(dl=0, position=1)
KINDS = dict(osc=OSC, filter=FILT, biquad=BIQUAD, nonlin=NONLIN, delay=DELAY)
# state words of a stage, by op (the layouts include/maxib200.h documents with the ops); ops not listed have none
STATE_SLOTS = {OP["osc"]: 2, OP["env_adsr"]: 4, OP["env_ar"]: 4, OP["envgen"]: 12, OP["filter"]: 2, OP["svf"]: 3, OP["biquad"]: 2,
               OP["dcblock"]: 2, OP["delay"]: 1, OP["flanger"]: 3, OP["chorus"]: 4}
ENVGEN_HOLD = -46692.0
NONE = -1
NSRC = 8


def R(i):
    assert 0 <= i < 16
    return i


class PatchDef:
    def __init__(self):
        self.stages = []          # (op, kind, dst, [src...])
        self.consts = []
        self.params = []          # names, index = parameter slot
        self.inputs = []          # names, index = input stream
        self.input_types = {}     # name -> "u8" | "bits" for byte / packed-bit streams (triggers, gates), "events" for control events; doubles otherwise
        self.eg = None            # maxiEnvGen shape 0: (levels, times, curves, loop, retrigger)

    def K(self, value):
        """scalar constant operand (deduplicated by bit pattern)"""
        import struct
        key = struct.pack("<d", float(value))
        for i, c in enumerate(self.consts):
            if struct.pack("<d", c) == key:
                return 0x200 + i
        self.consts.append(float(value))
        assert len(self.consts) <= 64
        return 0x200 + len(self.consts) - 1

    def P(self, name):
        """per-voice parameter operand"""
        if name not in self.params:
            self.params.append(name)
            assert len(self.params) <= 32
        return 0x100 + self.params.index(name)

    def IN(self, name, dtype="f64"):
        """per-sample input stream operand; dtype "u8": the caller passes unsigned bytes, "bits": one bit per voice-sample packed into
        uint32 words (both read as doubles by the stages), "events": per-voice values set at any frame and held (MXB_IN_EVENTS)"""
        if name not in self.inputs:
            self.inputs.append(name)
            assert len(self.inputs) <= 8
            if dtype in ("u8", "bits", "events"):
                self.input_types[name] = dtype
        return 0x300 + self.inputs.index(name)

    def stage(self, op, *src, kind=0, dst=NONE):
        k = KINDS[op][kind] if isinstance(kind, str) else int(kind)
        s = list(src) + [NONE] * (NSRC - len(src))
        assert len(s) == NSRC
        self.stages.append((OP[op], k, dst, s))
        return len(self.stages) - 1

    # shapes 1, 2, ... of a patch with several maxiEnvGen shapes; an instance attribute from the second shape on, so that a PatchDef
    # with one shape has exactly the attributes it always had (the oracle's recorded reference calls digest a PatchDef by them)
    eg_more = ()

    def envgen(self, levels, times, curves, loop=False, retrigger=False):
        """A maxiEnvGen shape: the arguments of maxiEnvGen::setup(levels, times, curves, looping, allowRetrigger). Returns its index, the
        `kind` of the envgen stages that play it (stage("envgen", trigger, kind=i)). One level and no times / curves: a maxiEnvGen whose
        setup() was never called (it plays 0)."""
        assert len(levels) == len(times) + 1 == len(curves) + 1
        shape = (list(map(float, levels)), list(map(float, times)), list(map(float, curves)), bool(loop), bool(retrigger))
        if self.eg is None:
            self.eg = shape
            return 0
        self.eg_more = list(self.eg_more) + [shape]
        assert len(self.shapes) <= 4
        return len(self.eg_more)

    @property
    def shapes(self):
        """every maxiEnvGen shape, in index order"""
        return ([self.eg] if self.eg is not None else []) + list(self.eg_more)
