"""Write tests/golden/live_reference_deconv.json from the unmodified reference DeConvBnRelu (seg_oprs.py:49-73).

    TSB_REFERENCE_DIR=<TorchSeg checkout> python tools/make_deconv_golden.py

Stores what tests/test_cpu_deconv.py compares against, so that it runs without the reference: the constructor's
parameter names and defaults, and the state_dict keys and shapes of a few configurations.
"""
import inspect
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import reference_live as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference_deconv.json")

# (in_planes, out_planes, ksize, stride, pad, output_pad, kwargs)
CONFIGS = [
    (64, 32, 4, 2, 1, 0, {}),
    (64, 64, 2, 2, 0, 0, {"has_relu": False}),
    (19, 19, 4, 2, 1, 0, {"has_bn": False, "has_bias": True}),
    (128, 64, 3, 2, 1, 1, {"has_bn": True, "has_relu": True}),
]


def main():
    assert rl.available(), "the reference checkout is needed (TSB_REFERENCE_DIR)"
    so = rl.load_seg_oprs()
    sig = inspect.signature(so.DeConvBnRelu.__init__)
    params = [[n, None if p.default is inspect.Parameter.empty else repr(p.default)]
              for n, p in sig.parameters.items() if n != "self"]
    cases = []
    for ci, co, k, s, p, op, kw in CONFIGS:
        m = so.DeConvBnRelu(ci, co, k, s, p, op, **kw)
        cases.append({"args": [ci, co, k, s, p, op], "kwargs": kw,
                      "children": [n for n, _ in m.named_children()],
                      "state_dict": [[key, list(v.shape)] for key, v in m.state_dict().items()]})
    with open(OUT, "w") as f:
        json.dump({"params": params, "cases": cases}, f, indent=1)
        f.write("\n")
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
