"""Child process of test_gpu_bench_workloads.test_results_do_not_depend_on_connection_count (not a test module).

    python tests/bench_workloads_child.py OUT.json

Runs the benchmark's device workloads (test_gpu_bench_workloads.CHILD_WORKLOADS) with the environment it was started
with -- the test sets CUDA_DEVICE_MAX_CONNECTIONS=32 there, before CUDA starts, as bench.py does -- and writes that
variable and each call's plan, frame count and SHA-256 of its output rows to OUT.json.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]


def main(path):
    import dsp_b200
    from test_gpu_bench_workloads import CHILD_WORKLOADS, record_of
    if dsp_b200.device_count() < 1:
        raise SystemExit("no CUDA device")
    out = {"CUDA_DEVICE_MAX_CONNECTIONS": os.environ.get("CUDA_DEVICE_MAX_CONNECTIONS"),
           "workloads": {name: record_of(dsp_b200, name) for name in CHILD_WORKLOADS}}
    with open(path, "w") as f:
        json.dump(out, f)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1]))
