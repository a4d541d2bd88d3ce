"""One K2-lw update per instantiation (LARS and LAMB, with and without the bf16 shadow), each checked
against float64 as in test_gpu_layerwise_paths.py, under torch.profiler in a process of its own:
a profiling session ended in a process hides later sessions' kernels there, so the test process
never starts one.  Prints the ``lw_stats_kernel`` / ``lw_apply_kernel`` instantiations the profiler
saw launch as one JSON line (``INSTANTIATIONS [...]``), then LAYERWISE_INSTANTIATIONS_OK.

    python tests/run_layerwise_instantiations.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import test_gpu_layerwise_paths as T  # noqa: E402
from test_gpu_optim_paths import _template_args  # noqa: E402


def main():
    layout = [(4099, True), (5, True)]
    cases = [T._LwCase(v, layout, [T.ADAPTED, 0], ["f32", "bf16"], lp, seed=3)
             for v in ("lars_momentum", "lamb") for lp in (False, True)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in cases:
            c.new_grads()
            c.step_and_check(lr=T.LR[c.mode], step=1, wd=1e-2, what="%s shadow %s" % (c.mode, c.shadow is not None))
        torch.cuda.synchronize()
    seen = set()
    for e in prof.events():
        for kernel in ("lw_stats_kernel", "lw_apply_kernel"):
            if "frl::%s<" % kernel in e.name:
                seen.add("%s:%s" % (kernel, _template_args(e.name, "frl::" + kernel)))
    print("INSTANTIATIONS " + json.dumps(sorted(seen)), flush=True)
    print("LAYERWISE_INSTANTIATIONS_OK", flush=True)


if __name__ == "__main__":
    main()
