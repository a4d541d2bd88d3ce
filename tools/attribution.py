#!/usr/bin/env python
"""Kernel-by-kernel attribution of the step-time difference between this repo's arm and the
stock-PyTorch arm, from the per-kernel profiles `bench.py --profile` writes.

    python tools/attribution.py mlp.json mlp_torch.json      # bench.py --profile mlp.json / --impl torch-gpu --profile mlp_torch.json
    python tools/attribution.py mlp.json mlp_e2e.json        # resident vs e2e epoch
"""
import json
import sys

GROUPS = [
    ("library GEMM / conv (cuBLAS, cuDNN)", ("nvjet", "gemm", "cutlass", "xmma", "cudnn", "sm80_", "sm90_", "sm100_", "implicit", "wgrad", "dgrad", "fprop")),
    ("gradient exchange (NCCL / K7 / K1)", ("nccl", "nvls_update", "nvls_barrier", "flatten_kernel")),
    ("input rows over PCIe (K8 / K8w, copy stream)", ("gather_rows", "gather_small_rows", "gather_window_rows")),
    ("optimizer update (K2 / multi_tensor_apply)", ("update_kernel", "update_mt_kernel", "multi_tensor_apply", "FusedSgd", "fused_adam", "FusedAdam")),
    ("criterion (K4 / loss kernels)", ("criteria_", "nll_loss", "log_softmax", "softmax", "mse_", "MseLoss")),
    ("ReLU / bias-gradient / reductions (K6, K6b)", ("colsum", "reduce_kernel", "threshold", "relu", "clamp")),
    ("normalisation / pooling (Problem's own layers)", ("batch_norm", "max_pool", "avg_pool", "adaptive")),
    ("casts / transform / copies (K5, copy kernels)", ("affine_kernel", "copy_kernel", "Memcpy", "memcpy", "direct_copy", "bfloat16_copy", "aten::copy_", "Memset", "FillFunctor")),
    ("other elementwise", ("elementwise", "CUDAFunctor", "vectorized")),
]


def grouped(path):
    d = json.load(open(path))
    out = {g: [0.0, 0.0] for g, _ in GROUPS}
    out["unclassified"] = [0.0, 0.0]
    for k in d["kernels_us_per_step"]:
        if k["name"].startswith(("Optimizer.", "ProfilerStep", "aten::", "autograd::", "nccl:", "DistributedDataParallel")):
            continue                      # profiler annotations, not kernels
        for g, pats in GROUPS:
            if any(p in k["name"] for p in pats):
                out[g][0] += k["us"]
                out[g][1] += k["launches"]
                break
        else:
            out["unclassified"][0] += k["us"]
            out["unclassified"][1] += k["launches"]
    return d, out


def main():
    a, ga = grouped(sys.argv[1])
    b, gb = grouped(sys.argv[2])
    print("| group | %s: µs/step (launches) | %s: µs/step (launches) | delta µs |" % (a["impl"], b["impl"]))
    print("|---|---|---|---|")
    for g in list(ga):
        if ga[g][0] or gb[g][0]:
            print("| %s | %.0f (%.0f) | %.0f (%.0f) | %+.0f |" % (g, ga[g][0], ga[g][1], gb[g][0], gb[g][1], gb[g][0] - ga[g][0]))
    print("| **device time, sum** | %.0f | %.0f | %+.0f |" % (sum(v[0] for v in ga.values()), sum(v[0] for v in gb.values()),
                                                            sum(v[0] for v in gb.values()) - sum(v[0] for v in ga.values())))
    if "ms_per_step" in a and "ms_per_step" in b:
        print("| **step (CUDA events)** | %.0f | %.0f | %+.0f |" % (1e3 * a["ms_per_step"], 1e3 * b["ms_per_step"],
                                                                  1e3 * (b["ms_per_step"] - a["ms_per_step"])))


if __name__ == "__main__":
    main()
