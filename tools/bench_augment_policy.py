"""Time K5p (``frl_augment_policy_images``) against K5a (``frl_augment_images``) on the ImageNet
training shape: batch 256, uint8 3x256x256 -> bf16 3x224x224 channels_last, RRC + flip.  Each arm
is captured in a CUDA graph together with a 64 MiB L2 flush; the arms alternate inside one process,
and the flush's own time (a graph of the flush alone) is subtracted.  Prints one JSON line with
median / min / max µs per batch and the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frl_b200  # noqa: E402,F401
from frl_b200 import _native, synthetic  # noqa: E402
from frl_b200.transform import RandAugment, TrivialAugmentWide  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(0)
    B = a.batch
    x = torch.randint(0, 256, (B, 3, 256, 256), generator=g, dtype=torch.uint8).to(dev)
    idx = torch.randperm(1 << 20, generator=g)[:B].to(dev)
    sc, bi = (torch.tensor(v, device=dev) for v in synthetic.U8_CHANNEL_AFFINE)
    out = torch.empty((B, 3, 224, 224), dtype=torch.bfloat16, device=dev, memory_format=torch.channels_last)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device=dev)
    common = dict(seed=1, epoch=1, mode=_native.AUG_RRC, flip=True, scale=sc, bias=bi)

    def k5p(pol, erase):
        mags = None if pol is None else pol.magnitudes(224, 224).to(dev)
        return lambda: _native.augment_policy_images(
            x, idx, out, policy=_native.POLICY_NONE if pol is None else pol.native,
            num_ops=1 if pol is None else pol.num_ops, magnitude=0 if pol is None else pol.magnitude, mags=mags,
            erase_p=0.25 if erase else 0.0, **common)

    arms = {
        "k5a": lambda: _native.augment_images(x, idx, out, **common),
        "ta_wide": k5p(TrivialAugmentWide(), False),
        "ta_wide+erasing": k5p(TrivialAugmentWide(), True),
        "ra(2,9)": k5p(RandAugment(), False),
        "ra(2,9)+erasing": k5p(RandAugment(), True),
        "erasing_only": k5p(None, True),
        "flush": lambda: None,
    }
    graphs = {}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for name, fn in arms.items():
            for _ in range(2):
                flush.zero_()
                fn()
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=s):
                flush.zero_()
                fn()
            graphs[name] = gr
    torch.cuda.current_stream().wait_stream(s)
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for name, gr in graphs.items():
            st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            gr.replay()
            st.record()
            for _ in range(a.reps):
                gr.replay()
            en.record()
            torch.cuda.synchronize()
            times[name].append(st.elapsed_time(en) * 1000.0 / a.reps)
    base = sorted(times["flush"])[len(times["flush"]) // 2]
    res = {}
    for name, ts in times.items():
        if name == "flush":
            continue
        ts = sorted(t - base for t in ts)
        res[name] = {"median_us": round(ts[len(ts) // 2], 1), "min_us": round(ts[0], 1), "max_us": round(ts[-1], 1)}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"bench": "augment_policy", "batch": B, "shape": "3x256x256 u8 -> 3x224x224 bf16 NHWC",
                      "gpu": gpu, "flush_us": round(base, 1), "arms": res}))


if __name__ == "__main__":
    main()
