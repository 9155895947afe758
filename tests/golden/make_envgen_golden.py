"""Generates tests/golden/envgen_shapes.npz from the UNMODIFIED reference (oracle/_ref/libmaxiref.so, built by oracle/Makefile): the
voice patches of tests/envgen_cases.py, which hold several maxiEnvGen shapes, run by the reference's own objects -- one maxiEnvGen per
envelope stage and voice, set up with that stage's shape. Inputs are stored beside the outputs. Run where the reference is built:

    python tests/golden/make_envgen_golden.py [output.npz]

(default: tests/golden/envgen_shapes.npz)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import oracle_py as O          # noqa: E402
import envgen_cases as EC                  # noqa: E402
from maximilian_b200.patchdef import OP    # noqa: E402

V, B, NB = 12, 300, 3


def main(path=os.path.join(HERE, "envgen_shapes.npz")):
    O.build("reference")
    out = {"V": V, "B": B, "NB": NB}
    for name, d, params, inputs in EC.cases():
        ins = inputs(V, NB * B, 5)
        p = O.Patch(d, V, kind="reference")
        for k, v in params(V, 3).items():
            p.set(k, v)
            out[f"{name}/param/{k}"] = np.asarray(v, dtype=np.float64)
        for k, a in ins.items():
            out[f"{name}/in/{k}"] = a
        outs, mixes = [], []
        for blk in range(NB):
            o, m = p.process(B, {k: a[blk * B:(blk + 1) * B] for k, a in ins.items()}, want_mix=True)
            outs.append(o); mixes.append(m)
        out[name + "/out"] = np.stack(outs)
        out[name + "/mix"] = np.stack(mixes)
        for si, st in enumerate(d.stages):
            if st[0] == OP["envgen"]:
                out[f"{name}/state/{si}"] = np.stack([p.get_state(si, sl) for sl in range(EC.SLOTS)])
    np.savez_compressed(path, **out)


if __name__ == "__main__":
    main(*sys.argv[1:])
