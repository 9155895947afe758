"""Voice patches with several maxiEnvGen shapes on the CPU oracles, which take one shape per patch (oracle/oracle_api.h: the eg_* of
mxo_patch_desc; the C port oracle/maxi_oracle.c, or the reference's own maxiEnvGen objects through oracle/ref_shim.cpp).

A maxiEnvGen stage's output depends only on its trigger and its own state, and the stages of a sample run in list order. So a patch with
envelope stages e1 < e2 < ... runs as one oracle patch per envelope stage plus one for the rest, in lock step, block by block:
  * the patch of envelope stage e is the stage list up to e, plus an output stage for e's register. Stage e plays its own shape, which is
    the oracle patch's one shape. Every earlier envelope stage j is replaced by `input(eg<j>) * 1.0`, where the input carries j's output
    for this block, already computed. Multiplying by 1.0 is exact;
  * the last patch is the whole list with every envelope stage replaced that way. It gives the outputs, the bus and the state of every
    other stage.
Each envelope stage's state is read from its own patch. A patch with one shape gives the same bits as the oracle running it directly
(tests/test_oracle_envgen_shapes.py checks that).
"""
import copy

from maximilian_b200.patchdef import NONE, NSRC

ENVGEN, MUL, OUT = 4, 14, 17


def _variant(defn, upto, keep):
    """stages[:upto] of `defn` with envelope stage `keep` (or none) kept and every other envelope stage fed from an input stream"""
    d = copy.deepcopy(defn)
    d.__dict__.pop("eg_more", None)
    d.eg = defn.shapes[defn.stages[keep][1]] if keep is not None else None
    stages = []
    for i, (op, kind, dst, src) in enumerate(defn.stages[:upto]):
        if op != ENVGEN:
            stages.append((op, kind, dst, list(src)))
        elif i == keep:
            stages.append((op, 0, dst, list(src)))
        else:
            stages.append((MUL, 0, dst, [d.IN(f"eg{i}"), d.K(1.0)] + [NONE] * (NSRC - 2)))
    if keep is not None and defn.stages[keep][2] >= 0:
        stages.append((OUT, 0, NONE, [defn.stages[keep][2]] + [NONE] * (NSRC - 1)))
    d.stages = stages
    return d


class ShapesPatch:
    """oracle_py.Patch's interface (set, process, get_state) for a PatchDef with any number of maxiEnvGen shapes."""

    def __init__(self, oracle, defn, voices, sample_rate=48000, delay_taps=0, kind="port"):
        self.V = int(voices)
        self.eg = [i for i, s in enumerate(defn.stages) if s[0] == ENVGEN]
        mk = lambda d: oracle.Patch(d, self.V, sample_rate=sample_rate, delay_taps=delay_taps, kind=kind)      # noqa: E731
        self.sub = {e: mk(_variant(defn, e + 1, e)) for e in self.eg}
        self.full = mk(_variant(defn, len(defn.stages), None))

    def set(self, name, values):
        for p in list(self.sub.values()) + [self.full]:
            if name in p.defn.params:
                p.set(name, values)

    def process(self, nframes, inputs=None, want_out=True, want_mix=False):
        ins = dict(inputs or {})
        for e in self.eg:
            o, _ = self.sub[e].process(nframes, {k: ins[k] for k in self.sub[e].defn.inputs})
            ins[f"eg{e}"] = o
        return self.full.process(nframes, {k: ins[k] for k in self.full.defn.inputs}, want_out=want_out, want_mix=want_mix)

    def get_state(self, stage, slot):
        return (self.sub[stage] if stage in self.sub else self.full).get_state(stage, slot)
