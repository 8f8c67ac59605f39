#!/usr/bin/env python
"""Generate tests/golden/lineart.pt by running the REFERENCE ITSELF: `LineArt` of the upstream ControlAR repository's
condition/lineart.py (read-only import from $CONTROLAR_REFERENCE, default ../reference next to this repository), in fp32 on the
CPU, on procedural weights (tests/lineart_oracle.py:make_lineart_state_dict) and seeded inputs (lineart_inputs).  The module
imports `controlnet_aux` at the top without using it; a stand-in module is put in sys.modules for it.  Run from the repo root:

    python tests/golden/make_lineart_golden.py

Stored: header, seed, the reference's state-dict keys and shapes, the pre-sigmoid range and, per input, the output shape and the
fp32 output map.  For the 512 x 512 input only windows of the map are kept (tests/lineart_oracle.py:GOLDEN_WINDOWS_512: the corners
with the reflection borders, the edge middles and the centre), which keeps the fixture small.  For the 70 x 90 and 5 x 7 inputs the
reference evaluated in fp64 is stored too.  Weights and inputs are regenerated from the seeds by the tests.
"""
from __future__ import annotations

import os
import sys
import types

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = os.environ.get("CONTROLAR_REFERENCE", os.path.join(os.path.dirname(REPO), "reference"))
OUT = os.path.join(REPO, "tests", "golden")
sys.path.insert(0, REPO)
sys.path.insert(0, REF)

import torch

from tests.lineart_oracle import make_lineart_state_dict, lineart_inputs, GOLDEN_WINDOWS_512

SEED = 8


def main():
    torch.set_grad_enabled(False)
    sys.modules["controlnet_aux"] = types.SimpleNamespace(LineartDetector=None)
    from condition.lineart import LineArt
    net = LineArt().float().eval()
    sd = make_lineart_state_dict(SEED)
    ref_sd = net.state_dict()
    assert list(ref_sd) == list(sd), (list(ref_sd), list(sd))
    for k in sd:
        assert tuple(ref_sd[k].shape) == tuple(sd[k].shape), k
    net.load_state_dict(sd, strict=True)
    out = {"header": {"torch": str(torch.__version__), "device": "cpu", "dtype": "float32", "generator": "tests/golden/make_lineart_golden.py",
                      "reference": "condition/lineart.py LineArt()"},
           "seed": SEED, "keys": list(ref_sd), "shapes": {k: tuple(v.shape) for k, v in ref_sd.items()},
           "n_params": sum(v.numel() for v in ref_sd.values())}
    for name, x in lineart_inputs().items():
        y = net(x)
        pre = net.model4[:2](net.model3(net.model2(net.model1(net.model0(x)))))
        out[name + "_shape"] = tuple(y.shape)
        if x.shape[-1] == 512:
            out[name + "_windows"] = [(box, y[..., box[0]:box[0] + box[2], box[1]:box[1] + box[3]].clone()) for box in GOLDEN_WINDOWS_512]
        else:
            out[name] = y.clone()
        out[name + "_preact_range"] = (float(pre.min()), float(pre.max()), float(pre.std()))
        if name in ("b1_70x90", "b1_5x7"):  # the reference itself in fp64: the exact value its fp32 output approximates
            out[name + "_fp64"] = net.double()(x.double()).clone()
            net.float()
        print(name, tuple(x.shape), "->", tuple(y.shape), "pre-sigmoid min/max/std %.2f %.2f %.2f" % out[name + "_preact_range"], flush=True)
    torch.save(out, os.path.join(OUT, "lineart.pt"))


if __name__ == "__main__":
    main()
