"""One AdamW update per new instantiation (K2: amsgrad x gradient dtype x shadow; K2-mt: amsgrad x
shadow; K2-q8: shadow), the K2 and K2-mt updates checked against float64 ``torch.optim.AdamW`` as in
test_gpu_adamw.py, under torch.profiler in a process of its own: a profiling session ended in a
process hides later sessions' kernels there, so the test process never starts one.  Prints the
instantiations the profiler saw launch as one JSON line (``INSTANTIATIONS {...}``), then
ADAMW_INSTANTIATIONS_OK.

    python tests/run_adamw_instantiations.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import test_gpu_adamw as T  # noqa: E402
from test_gpu_optim_paths import _template_args  # noqa: E402


def main():
    n = 4099
    gen = torch.Generator(device=T.DEV).manual_seed(3)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for ams in (False, True):
            for gdt in (torch.float32, torch.bfloat16):
                for lp in (False, True):
                    p = T._weights(n, gen)
                    g = T._grad(n, gen).to(gdt)
                    states = [torch.zeros(n, device=T.DEV) for _ in T.STATES[ams]]
                    shadow = torch.zeros(n, dtype=torch.bfloat16, device=T.DEV) if lp else None
                    p0, s0 = p.clone(), [s.clone() for s in states]
                    T.launch_flat(ams, p, g, states, shadow, n, lr=0.01, wd=T.WD, step=1)
                    T.check_step(ams, p, states, p0, g.double() * T.SCALE, s0, lr=0.01, wd=T.WD, step=1,
                                 what="flat amsgrad %s %s shadow %s" % (ams, gdt, lp))
            for lp in (False, True):
                c = T._MtCase("adam_amsgrad" if ams else "adam", lp, seed=3)
                g = c.new_grads()
                p0, s0 = c.p[c.idx].clone(), [s[c.idx].clone() for s in c.states]
                T.launch_mt(ams, c.p, c.states, c.shadow, c.table, lr=0.01, wd=T.WD, step=1)
                T.check_step(ams, c.p[c.idx], [s[c.idx] for s in c.states], p0, g, s0, lr=0.01, wd=T.WD, step=1,
                             what="mt amsgrad %s shadow %s" % (ams, lp))
        for lp in (False, True):
            case = T.a8._Case(torch.float32, lp, seed=5)
            p0 = case.p.clone()
            T._native.adamw8_mt(case.p, case.codes["m"], case.codes["v"], case.absmax["m"], case.absmax["v"],
                                case.shadow, case.table, case.qbase, case.flags, lr=0.01, wd=T.WD, step=1, **T.HP)
            assert torch.isfinite(case.p).all() and not torch.equal(case.p, p0), "q8 shadow %s" % lp
        torch.cuda.synchronize()
    seen = {"flat": set(), "mt": set(), "q8": set()}
    for e in prof.events():
        for key, kernel in (("flat", "frl::update_kernel"), ("mt", "frl::update_mt_kernel"),
                            ("q8", "frl::adam8_mt_kernel")):
            if kernel + "<frl::AdamWRule" in e.name:
                seen[key].add(_template_args(e.name, kernel))
    print("INSTANTIATIONS " + json.dumps({k: sorted(v) for k, v in seen.items()}), flush=True)
    print("ADAMW_INSTANTIATIONS_OK", flush=True)


if __name__ == "__main__":
    main()
