#!/usr/bin/env python
"""Regenerates tests/golden/solver_bits.json: the embedding and statistics digests of the cases of
tests/test_gpu_solver_bits.py, computed on cuda:0 by the library as built.

    python tests/golden/make_solver_bits_golden.py [OUT.json]

The committed fixture was recorded from the build that precedes the reorganised head-kernel history loads, so only
regenerate it for a change that is meant to alter the bits."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import torch  # noqa: E402
from tests import test_gpu_solver_bits as T  # noqa: E402


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else T.GOLDEN
    assert torch.cuda.is_available(), "the fixture is recorded on a GPU"
    doc = {"gpu": torch.cuda.get_device_name(0), "cases": {c: T.evaluate(c) for c in T.CASES}}
    with open(out, "w") as fh:
        json.dump(doc, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print("wrote", out, len(doc["cases"]), "cases")


if __name__ == "__main__":
    main()
