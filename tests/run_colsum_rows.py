"""The exact K6 / K6b cases of test_gpu_colsum_paths.py at one rows-in-flight setting.

``FRL_B200_COLSUM_ROWS`` (1, 2 or 4; unset: the default) is read once per process, so each setting
runs in a process of its own.  The cases cover both kernels, every dtype pair and the vector and
scalar paths; the script prints the ``colsum_kernel`` instantiations torch.profiler saw launch as
one JSON line (``INSTANTIATIONS [...]``), then COLSUM_ROWS_OK.

    FRL_B200_COLSUM_ROWS=1 python tests/run_colsum_rows.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import test_gpu_colsum_paths as T  # noqa: E402


def main():
    rif = os.environ.get("FRL_B200_COLSUM_ROWS", "default")
    assert rif in ("default", "1", "2", "4"), "FRL_B200_COLSUM_ROWS must be 1, 2, 4 or unset"
    cases = T.exact_cases(T.RIF_SHAPES)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case in cases:
            T.check_exact(*case.values)
        torch.cuda.synchronize()
    seen = sorted({T._template_args(e.name) for e in prof.events() if "colsum_kernel<" in e.name})
    print("rows in flight %s: %d exact cases passed" % (rif, len(cases)), flush=True)
    print("INSTANTIATIONS " + json.dumps(seen), flush=True)
    print("COLSUM_ROWS_OK", flush=True)


if __name__ == "__main__":
    main()
