#!/usr/bin/env python
"""Generates tests/golden/launches.json.gz, the learner's launch traces (tests/launch_trace_util.py) of every case in
launch_trace_util.CASES, on a CUDA device:

    python tests/golden/make_golden_launches.py <commit>

<commit> is the commit whose code made the traces; it is stored beside them.  The fixture pins which kernels the learner launches,
with which shapes, pointers, epilogue flags and streams, so that a change meant to leave the learner's work as it is can show that it
did: tests/test_learner_launches_gpu.py replays the cases against it.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import launch_trace_util as lt  # noqa: E402


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    traces = {}
    for name in lt.CASES:
        traces[name] = lt.trace(name, lt._Patch())
        print(name, len(traces[name]), "launches")
    lt.write(sys.argv[1], traces)
    print("wrote", lt.FIXTURE)


if __name__ == "__main__":
    main()
