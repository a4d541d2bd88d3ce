"""``Solver.solve`` — entry point and per-rank bootstrap (reference solver.py:101-837).

Kept from the reference: the ``solve()`` signature and generator protocol, one OS process per
GPU with a one-way pipe back to the parent, per-epoch aggregation (sample-weighted means,
MSE -> RMSE renaming), checkpoint file names and contents, resume from ``.checkpoint.pth``.

Replaced: the per-rank bootstrap no longer wraps the model in ``DistributedDataParallel`` and
``torch.optim``; it builds the flat arena, the fused optimizer and the bucket pipeline
(``arena.py``, ``fused_optim.py``, ``grad_sync.py``).  There is no CPU path: without a CUDA device
(or with ``cpuonly=True``) ``solve`` raises.
"""
import io
import json
import logging
import math
import multiprocessing
import os
import pickle
import traceback
from collections import defaultdict
from contextlib import ExitStack
from multiprocessing.connection import Connection, wait as wait_pipes
from typing import IO, Any, DefaultDict, Dict, Iterator, List, NamedTuple, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from .arena import ParamArena
from .criteria import BaseParallelCriterion
from .ema import EMA_STATE_KEY
from .fused_optim import check_layer_adaptation, create_fused_optimizer, is_adapted
from .grad_sync import BufferBroadcaster, GradBucketPipeline
from .lr_scheduler import DropEpochsScheduler, WarmupMultiStepLR
from .problem import Problem
from .solver_worker import (FractionalPerformanceSummary, SerializableSampleSummary,
                            SolverWorker)
from .types import (Device, LayerAdaptation, LRSchedulerAlgorithm, Mode, Precision, RunOpts,
                    SampleSummary, Split)

logging.basicConfig(level=logging.INFO, format="%(levelname)s (%(process)d) %(message)s")
logger = logging.getLogger(__name__)

CHECKPOINT_NAME = ".checkpoint.pth"
LAYER_ADAPTATION_ENV = "FRL_B200_LAYER_ADAPTATION"   # "none" (default) | "lars" | "lamb"
PRECISION_ENV = "FRL_B200_PRECISION"      # "fp32" (default, reference parity) | "bf16"
GRAD_ACCUM_ENV = "FRL_B200_GRAD_ACCUM"     # microbatches per optimizer update, default 1
EMA_DECAY_ENV = "FRL_B200_EMA_DECAY"       # weight EMA decay in [0, 1), default 0 (off)
EMA_SUFFIX = ".ema"                        # <checkpoint>.ema: the weight EMA next to a checkpoint


class SingleSampleSummary(NamedTuple):
    plot: Any
    source: str


class SplitSampleSummaryGroup(NamedTuple):
    image: Optional[bytes]
    text: Optional[str]
    summaries: List[SingleSampleSummary]


class SplitSampleSummary(NamedTuple):
    random: SplitSampleSummaryGroup
    worst: SplitSampleSummaryGroup


class EpochSplitPerformanceSummary(NamedTuple):
    losses: Dict[str, float]
    metrics: Dict[str, float]
    sample_summary: SplitSampleSummary


class PerformanceSummary(NamedTuple):
    epoch: int
    performance: Dict[Split, EpochSplitPerformanceSummary]
    save_dir: str


class Checkpoint(NamedTuple):
    epoch: int
    modelState: Dict[Any, Any]
    optimizerState: Dict[Any, Any]


class SolverWorkerArgs(NamedTuple):
    run_opts: RunOpts
    problem: Problem
    save_dir: str
    run_device: Device
    node_idx: int
    node_count: int
    rank: int
    local_rank: int
    world_size: int
    group_name: Optional[str]
    init_method: str
    cache: Any = None
    precision: Precision = Precision.FP32
    save_every: int = 1
    graph_step: Optional[bool] = None      # None: FRL_B200_CUDA_GRAPH (default off)
    layer_adaptation: LayerAdaptation = LayerAdaptation.NONE
    # weight EMA decay, 0 = off; placed before grad_accumulation, which stays the last field
    ema_decay: float = 0.0
    grad_accumulation: int = 1


def _torch_load(f, **kw):
    # checkpoints hold whole pickled modules / optimizer dicts (reference solver.py:604-611)
    return torch.load(f, weights_only=False, **kw)


def _load_model_state(model: nn.Module, model_path: str, strict: bool = True) -> None:
    with open(model_path, "rb") as f:
        new_state = _torch_load(f, map_location="cpu")["state_dict"]
    if strict:
        model.load_state_dict(new_state)
        return
    # partial initialisation: copy what matches in name and shape, report the rest
    own = model.state_dict()
    for name, value in new_state.items():
        if name not in own:
            print("Warning: Parameter named {} is not used by this model.".format(name))
            continue
        value = value.data if isinstance(value, nn.Parameter) else value
        if own[name].size() == value.size():
            own[name].copy_(value)
        else:
            print("Warning: While copying the parameter named {}, whose dimensions in the model "
                  "are {} and whose dimensions in the checkpoint are {}.".format(
                      name, own[name].size(), value.size()))
    for name in own:
        if name not in new_state:
            print("Warning: Parameter named {} in the model is not initialized.".format(name))


def create_lr_scheduler(run_opts: RunOpts, optimizer, checkpoint_epoch=-1):
    """Epoch-granular schedule factory (reference solver.py:191-218)."""
    algo = run_opts.optim.lr_scheduler.algo
    n = run_opts.nEpochs
    if algo == LRSchedulerAlgorithm.DropEpochs:
        drops = [np.floor(n * 0.66667), np.floor(n * 0.9)] if n > 10 else []
        return DropEpochsScheduler(optimizer, drops, last_epoch=checkpoint_epoch)
    if algo == LRSchedulerAlgorithm.WarmupMultiStepLR:
        steps = [np.floor(n * r) for r in (0.33333, 0.66667, 0.9)]
        return WarmupMultiStepLR(optimizer, steps, gamma=0.1, warmup_factor=1.0 / 1000,
                                 warmup_iters=5, warmup_method="linear",
                                 last_epoch=checkpoint_epoch)
    raise ValueError("Unknown optimization algorithm type")


def _save_img(img: Optional[np.ndarray]) -> Optional[bytes]:
    if img is None:
        return None
    import cv2
    ok, png = cv2.imencode(".png", np.flip(img, axis=2))     # RGB -> BGR for OpenCV
    return png.tobytes()


def _aggregate_sample_summaries(results: List[SampleSummary]) -> SplitSampleSummaryGroup:
    images = [s.image for s in results if s.image is not None]
    texts = [s.text for s in results if s.text is not None]
    plots = [SingleSampleSummary(plot=s.plot, source=s.source) for s in results
             if s.plot is not None and s.source is not None]
    return SplitSampleSummaryGroup(
        image=_save_img(np.concatenate(images)) if images else None,
        text="\n".join(texts) if texts else None, summaries=plots)


def _cuda_device_count_without_poisoning_fork() -> int:
    """Device count for the parent process.

    ``torch.cuda.is_available()`` normally goes through ``cudaGetDeviceCount`` which arms torch's
    fork guard: children forked afterwards cannot initialise CUDA ("Cannot re-initialize CUDA in
    forked subprocess") — the stock reference trips over exactly this on current torch
    (reference solver.py:740-747).  The NVML-based check leaves the process fork-safe."""
    os.environ.setdefault("PYTORCH_NVML_BASED_CUDA_CHECK", "1")
    if not torch.cuda.is_available():
        return 0
    return torch.cuda.device_count()


def _fork_is_safe() -> bool:
    """True if a forked child of this process can still initialise CUDA (probed in a throwaway
    child, because the guard's state is only observable after the fork)."""
    if torch.cuda.is_initialized():
        return False
    pid = os.fork()
    if pid == 0:
        code = 1
        try:
            code = 1 if torch._C._cuda_isInBadFork() else 0
        finally:
            os._exit(code)
    _, status = os.waitpid(pid, 0)
    return os.WIFEXITED(status) and os.WEXITSTATUS(status) == 0


def bind_to_gpu_numa_node(local_rank: int) -> bool:
    """Pin this rank's threads to the CPUs nearest its GPU (NVML's ideal affinity), so pinned
    staging buffers are first-touched on the local NUMA node and H2D copies do not cross sockets.
    Best effort: returns False if NVML is unavailable."""
    try:
        import pynvml
        pynvml.nvmlInit()
        handle = pynvml.nvmlDeviceGetHandleByIndex(local_rank)
        pynvml.nvmlDeviceSetCpuAffinity(handle)
        return True
    except Exception as e:                           # noqa: BLE001
        logger.info("NUMA binding skipped: %s", e)
        return False


_NORM_FP32_STATS = {}


def _norm_accepts_fp32_stats(device: torch.device) -> bool:
    """Probe once per device: batch_norm with bf16 input and affine parameters but fp32 running
    statistics (training and eval mode)."""
    key = str(device)
    if key not in _NORM_FP32_STATS:
        try:
            x = torch.randn(4, 3, 2, 2, device=device).to(torch.bfloat16).requires_grad_(True)
            w = torch.ones(3, device=device, dtype=torch.bfloat16, requires_grad=True)
            b = torch.zeros(3, device=device, dtype=torch.bfloat16, requires_grad=True)
            rm, rv = torch.zeros(3, device=device), torch.ones(3, device=device)
            with torch.enable_grad():
                # forward AND backward (torch 2.11's batch_norm backward insists on statistics of
                # the affine parameters' dtype although its forward does not)
                torch.nn.functional.batch_norm(x, rm, rv, w, b, training=True).float().sum().backward()
                torch.nn.functional.batch_norm(x, rm, rv, w, b, training=False).float().sum().backward()
            ok = bool(rm.abs().sum() > 0) and rm.dtype == torch.float32
        except Exception as e:                       # noqa: BLE001
            logger.info("fp32 BatchNorm statistics next to bf16 parameters are not supported here (%s): "
                        "running statistics are kept in bf16", str(e).splitlines()[0])
            ok = False
        _NORM_FP32_STATS[key] = ok
    return _NORM_FP32_STATS[key]


def resolve_precision(explicit: Optional[Precision] = None) -> Precision:
    if explicit is not None:
        return explicit
    return Precision(os.environ.get(PRECISION_ENV, "fp32").lower())


def resolve_layer_adaptation(explicit: Optional[LayerAdaptation] = None) -> LayerAdaptation:
    if explicit is not None:
        return LayerAdaptation(explicit)
    return LayerAdaptation(os.environ.get(LAYER_ADAPTATION_ENV, "none").lower())


def resolve_grad_accumulation(explicit: Optional[int] = None) -> int:
    """Microbatches per optimizer update: ``explicit``, else FRL_B200_GRAD_ACCUM, else 1.  Anything
    but an integer >= 1 (``0``, negatives, ``2.5``, ``True``, non-numeric strings) is a ValueError."""
    value: Any = explicit
    if value is None:
        raw = os.environ.get(GRAD_ACCUM_ENV, "1")
        try:
            value = int(raw.strip())
        except ValueError:
            raise ValueError("%s=%r: gradient accumulation must be an integer >= 1" % (GRAD_ACCUM_ENV, raw)) from None
    if isinstance(value, bool) or not isinstance(value, (int, np.integer)) or value < 1:
        raise ValueError("grad_accumulation=%r: gradient accumulation must be an integer >= 1" % (value,))
    return int(value)


def resolve_ema_decay(explicit: Optional[float] = None) -> float:
    """Weight EMA decay: ``explicit``, else FRL_B200_EMA_DECAY, else 0 (no EMA).  Anything but a
    real number in [0, 1) (``True``, negatives, ``1.0``, NaN, non-numeric strings) is a ValueError."""
    value: Any = explicit
    if value is None:
        raw = os.environ.get(EMA_DECAY_ENV, "0")
        try:
            value = float(raw.strip())
        except ValueError:
            raise ValueError("%s=%r: the EMA decay must be a real number in [0, 1)" % (EMA_DECAY_ENV, raw)) from None
    if (isinstance(value, bool) or not isinstance(value, (int, float, np.integer, np.floating))
            or not 0.0 <= float(value) < 1.0):
        raise ValueError("ema_decay=%r: the EMA decay must be a real number in [0, 1)" % (value,))
    return float(value)


def load_ema_checkpoint(ema, path: str, epoch: int) -> bool:
    """Resume ``ema`` (an ``ema.WeightEMA``) from the ``<checkpoint>.ema`` file at ``path`` if it
    exists and belongs to the checkpoint being resumed (saved at the same ``epoch``).  A file of
    another epoch (left by a later run without an EMA, or a save cut short between the two files) is
    not used: the EMA then starts from the loaded weights with 0 updates.  Returns True if loaded."""
    if not os.path.exists(path):
        return False
    blob = _torch_load(path, map_location="cpu")
    if int(blob["epoch"]) != int(epoch):
        logger.warning("%s was saved at epoch %d, the checkpoint being resumed at epoch %d: not used, "
                       "the weight EMA starts from the loaded weights", path, int(blob["epoch"]), int(epoch))
        return False
    if float(blob["decay"]) != ema.decay:
        logger.warning("%s was averaged with decay %r; continuing with %r", path, blob["decay"], ema.decay)
    ema.load_state_dict(blob)
    logger.info("Loaded the weight EMA from %s (%d updates)", path, ema.updates)
    return True


class Solver:
    # ------------------------------------------------------------------------------------------
    # per-rank bootstrap (child process)
    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _load_checkpoint(checkpoint_file: IO) -> Checkpoint:
        logger.info("Loading from check point %s", str(checkpoint_file))
        blob = _torch_load(checkpoint_file, map_location="cpu")
        logger.info("Loaded from check point, starting from epoch %d", blob["epoch"])
        return Checkpoint(epoch=blob["epoch"], modelState=blob["state_dict"],
                          optimizerState=blob["optimizer"])

    @staticmethod
    def _init_process_group(args: SolverWorkerArgs, device: torch.device) -> None:
        logger.info("Initializing process group with %s" % args.init_method)
        if torch.distributed.is_initialized():
            return                         # an external launcher (torchrun) already did
        torch.distributed.init_process_group(
            backend="nccl" if device.type == "cuda" else "gloo",
            init_method=args.init_method, world_size=args.world_size, rank=args.rank,
            group_name=args.group_name or "")

    @classmethod
    def build_worker(cls, args: SolverWorkerArgs):
        """Everything `_run_solver_worker` sets up, returned instead of run (bench/tests)."""
        run_opts, problem = args.run_opts, args.problem
        if args.run_device != Device.GPU:
            raise RuntimeError("frl_b200 has no CPU path: a CUDA (sm_90a) device is required")
        torch.cuda.set_device(args.local_rank)
        device = torch.device("cuda", args.local_rank)
        if args.world_size > 1 and os.environ.get("FRL_B200_NUMA_BIND", "1") != "0":
            bind_to_gpu_numa_node(args.local_rank)
        logger.info("Using device %s" % device)

        checkpoint: Optional[Checkpoint] = None
        try:
            with open(os.path.join(args.save_dir, CHECKPOINT_NAME), "rb") as f:
                checkpoint = cls._load_checkpoint(f)
        except FileNotFoundError:
            pass

        # model: build on the host (same RNG stream as the reference), load weights, move
        model = problem.get_model()
        if run_opts.initialModelPath is not None:
            _load_model_state(model, run_opts.initialModelPath,
                              strict=(run_opts.mode == Mode.EVAL))
        elif checkpoint:
            model.load_state_dict(checkpoint.modelState)
        model.to(device)
        criterion: BaseParallelCriterion = problem.get_criterion().to(device)
        from .criteria import GradNormWeightedCriterion
        accum = args.grad_accumulation if run_opts.mode == Mode.TRAIN else 1
        if accum > 1 and isinstance(criterion, GradNormWeightedCriterion):
            # GradNorm learns its task weights from each step's own gradients
            raise ValueError("grad_accumulation=%d cannot be combined with GradNormWeightedCriterion: "
                             "its task weights are learnt per step, not per accumulated group" % accum)

        distributed = args.world_size > 1
        if distributed:
            cls._init_process_group(args, device)

        # world > 1 without clipping: arena vectors other ranks reach go to symmetric/multicast
        # memory so all-reduce + update + broadcast can be one NVLS kernel per bucket
        ema_decay = args.ema_decay if run_opts.mode == Mode.TRAIN else 0.0
        symm_alloc = None
        if (distributed and not run_opts.optim.gradientClip
                and args.layer_adaptation == LayerAdaptation.NONE and accum == 1 and ema_decay == 0.0):
            from .symm import try_make_allocator
            symm_alloc = try_make_allocator(device, args.world_size)
        from .arena_linear import head_layout_groups
        arena = ParamArena(model.parameters(), criterion.parameters(), device=device,
                           precision=args.precision, shared_allocator=symm_alloc,
                           adjacent=head_layout_groups(model))
        if (args.precision.bf16_storage and any(b.is_floating_point() for b in model.buffers())
                and not _norm_accepts_fp32_stats(device)):
            # BatchNorm running statistics stay fp32 (what the reference's checkpoints hold: a
            # bf16 EMA with momentum 0.1 stalls on small deltas); only if this torch build
            # refuses bf16 activations/affine parameters next to fp32 statistics are the buffers
            # cast — and upcast again on export (arena.exported)
            for buf in model.buffers():
                if buf.is_floating_point():
                    buf.data = buf.data.to(torch.bfloat16)
        optimizer = create_fused_optimizer(arena, run_opts.optim, args.layer_adaptation)
        if checkpoint:
            optimizer.load_state_dict(checkpoint.optimizerState)
        ema = None
        if ema_decay > 0.0:
            # after the buffers took their final dtype; starts from the weights just loaded
            from .ema import WeightEMA
            ema = WeightEMA(arena, model, ema_decay)
            if checkpoint and run_opts.initialModelPath is None:
                load_ema_checkpoint(ema, os.path.join(args.save_dir, CHECKPOINT_NAME + EMA_SUFFIX),
                                    checkpoint.epoch)
        nvls_link = None
        if symm_alloc is not None:
            from .symm import make_link
            # grid of the fused NVLS step: each rank streams 1/world of a bucket, and every CTA it
            # parks on an SM while backward runs costs the cluster-scheduled GEMMs a wave, so the
            # grid shrinks with the world size: half the H100's 132 SMs at 2 GPUs (half of every
            # bucket per rank), 16 CTAs from 4 GPUs on.  Not yet tuned on a multi-GPU H100 box.
            default_blocks = 66 if args.world_size <= 2 else 16
            # the launch for the bucket that becomes ready last runs alone (backward has ended), so it
            # gets a wider grid
            default_tail = 64 if args.world_size >= 4 else 0
            nvls_link = make_link(symm_alloc, arena.grad,
                                  arena.lp if arena.lp is not None else arena.master,
                                  max_blocks=int(os.environ.get("FRL_B200_NVLS_BLOCKS", default_blocks)),
                                  tail_blocks=int(os.environ.get("FRL_B200_NVLS_TAIL_BLOCKS", default_tail)))
        pipeline = GradBucketPipeline(
            arena, optimizer, world_size=args.world_size, clip_norm=run_opts.optim.gradientClip,
            nvls_link=nvls_link,
            bucket_cap_mb=float(os.environ.get("FRL_B200_BUCKET_MB",
                                               "24" if nvls_link is not None else "48")),
            first_bucket_mb=None,
            eager_update=os.environ.get("FRL_B200_EAGER_UPDATE",
                                        "1" if args.world_size > 1 else "0") != "0",
            accumulation=accum, ema=ema)
        # GradNorm differentiates through the layers' backward (create_graph=True) and debugGrad
        # calls autograd.grad on them: those runs keep the stock nn.Linear autograd path
        if (os.environ.get("FRL_B200_DIRECT_GRADS", "1") != "0" and not run_opts.debugGrad
                and not isinstance(criterion, GradNormWeightedCriterion)):
            pipeline.patch_linears(model)
        buffers = None
        if distributed:
            pipeline.broadcast_parameters(src=0)
            buffers = BufferBroadcaster(model, world_size=args.world_size)
            buffers.sync()
        worker = SolverWorker(model, criterion, optimizer, device=device, run_opts=run_opts,
                              cache=args.cache, local_rank=args.local_rank,
                              node_idx=args.node_idx, node_count=args.node_count,
                              pipeline=pipeline, buffers=buffers, precision=args.precision,
                              serialize_state=(args.local_rank == 0),
                              graph_step=(args.graph_step if args.graph_step is not None
                                          else os.environ.get("FRL_B200_CUDA_GRAPH", "0") == "1"),
                              ema=ema)
        worker.save_every = args.save_every
        if args.rank == 0:
            # one line per run: which of the alternative paths this configuration took
            logger.info(
                "frl_b200 step: precision %s | step issue %s | gradient exchange %s | update %s | "
                "Linear layers with arena-born gradients %d (%d fused with their ReLU, %d in FP8) | "
                "other gradients %s | layer adaptation %s | gradient accumulation %s | weight EMA %s",
                args.precision.value,
                "CUDA-graph replay after 2 eager steps" if worker.graphed is not None else "eager launches",
                ("fused NVLS kernel per bucket (K7), %d buckets" % len(pipeline.buckets)) if pipeline.nvls is not None
                else ("ncclAllReduce in place + K2 per bucket, %d buckets" % len(pipeline.buckets)) if distributed
                else "none (1 GPU)",
                "per bucket on the side stream" if pipeline.eager else
                "in the dW GEMM's epilogue (K12) for trunk Linear weights that qualify, one tail launch for the rest"
                if pipeline.fused_dw_update else "one tail launch",
                len(pipeline.linear_sites), sum(s.relu is not None for s in pipeline.linear_sites),
                sum(s.fp8 for s in pipeline.linear_sites),
                "read in place through segment tables (K2-mt / one flatten launch per bucket)"
                if pipeline.mt_enabled else "copied into the arena per tensor",
                "none" if args.layer_adaptation == LayerAdaptation.NONE else
                "%s, %d of %d tensors adapted (K2-lw)" % (args.layer_adaptation.value,
                                                          sum(is_adapted(s) for s in arena.slots), len(arena.slots)),
                "none" if accum == 1 else
                "%d microbatches per update (K10, fp32 accumulator %.1f MiB)" % (
                    accum, pipeline.accumulator_bytes / 2 ** 20),
                "none" if ema is None else
                "decay %r, one K11 launch per update (%.1f MiB), held-out splits evaluated with it" % (
                    ema_decay, ema.nbytes / 2 ** 20))
        scheduler = create_lr_scheduler(run_opts, worker.optimizer,
                                        checkpoint.epoch if checkpoint else -1)
        return worker, scheduler, checkpoint

    @classmethod
    def _run_solver_worker(cls, args: SolverWorkerArgs) -> Iterator[FractionalPerformanceSummary]:
        """One of ``world_size`` instances, each training on its share of every epoch."""
        worker, scheduler, checkpoint = cls.build_worker(args)
        run_opts = args.run_opts
        if run_opts.mode == Mode.TRAIN:
            yield from worker.train(args.problem,
                                    startEpoch=checkpoint.epoch if checkpoint else 0,
                                    nEpochs=run_opts.nEpochs, batchSize=run_opts.batchSize,
                                    scheduler=scheduler)
        elif run_opts.mode == Mode.EVAL:
            yield from worker.eval(args.problem, batchSize=run_opts.batchSize)
        else:
            raise ValueError("unknown mode")

    @classmethod
    def _solver_worker_process(cls, solver_worker_args: SolverWorkerArgs,
                               comms_connection: Connection, cleanup_flag) -> None:
        """Child main: stream pickled per-epoch results, ``None`` on clean exit, the exception
        object on failure; then hold the pipe open until the parent has drained it."""
        root = logging.getLogger()
        root.setLevel(logging.DEBUG)
        try:
            for result in cls._run_solver_worker(solver_worker_args):
                comms_connection.send_bytes(pickle.dumps(result, protocol=pickle.HIGHEST_PROTOCOL))
            comms_connection.send(None)
        except Exception as e:
            logger.error(str(e))
            for line in traceback.format_exc().splitlines(False):
                logger.error(line)
            try:
                comms_connection.send(e)
            except Exception:
                comms_connection.send(RuntimeError(repr(e)))
            raise
        finally:
            cleanup_flag.wait()

    # ------------------------------------------------------------------------------------------
    # parent side: aggregation
    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _deserialize_sample_summaries(items: Sequence[SerializableSampleSummary]
                                      ) -> List[SampleSummary]:
        return [SampleSummary(image=s.image, text=s.text,
                              plot=json.loads(s.plot) if s.plot else None, source=s.source)
                for s in items]

    @classmethod
    def _aggregate_fractional_results(cls, run_opts: RunOpts, problem: Problem,
                                      fractional_results: List[FractionalPerformanceSummary]
                                      ) -> Dict[Split, EpochSplitPerformanceSummary]:
        splits = [d.data_type for d in problem.datasets]
        metric_sum = {s: defaultdict(float) for s in splits}
        loss_sum = {s: defaultdict(float) for s in splits}
        n_samples = {s: 0 for s in splits}
        picked = {s: [] for s in splits}
        worst = {s: [] for s in splits}
        for frac in fractional_results:
            for split, perf in frac.performance.items():
                for k, v in perf.metrics.items():
                    metric_sum[split][k] += v * perf.nSamples
                for k, v in perf.losses.items():
                    loss_sum[split][k] += v * perf.nSamples
                n_samples[split] += perf.nSamples
                picked[split] += cls._deserialize_sample_summaries(perf.samples)
                worst[split] += cls._deserialize_sample_summaries(perf.worstSamples)

        def finish_metrics(split: Split) -> Dict[str, float]:
            # sample-weighted MSE aggregates correctly but reads badly: report RMSE instead
            out: DefaultDict[str, float] = defaultdict(float)
            for name, total in metric_sum[split].items():
                value = total / n_samples[split]
                assert name.find("RMSE") == -1
                if "MSE" in name:
                    head, _, tail = name.rpartition("MSE")
                    out[head + "RMSE" + tail] = math.sqrt(value) if value > 0 else value
                else:
                    out[name] = value
            return out

        return {split: EpochSplitPerformanceSummary(
                    losses={k: v / n_samples[split] for k, v in loss_sum[split].items()},
                    metrics=finish_metrics(split),
                    sample_summary=SplitSampleSummary(
                        random=_aggregate_sample_summaries(picked[split]),
                        worst=_aggregate_sample_summaries(worst[split])))
                for split in splits}

    # ------------------------------------------------------------------------------------------
    # parent side: files
    # ------------------------------------------------------------------------------------------
    @classmethod
    def _save_epoch_summary(cls, epoch: int, save_dir: str,
                            epoch_stats: Dict[Split, EpochSplitPerformanceSummary]) -> None:
        for split, summary in epoch_stats.items():
            for group_name, group in (("random", summary.sample_summary.random),
                                      ("worst", summary.sample_summary.worst)):
                stem = os.path.join(save_dir, ".%s_%s_%04d" % (split.value, group_name, epoch))
                if group.image is not None:
                    with open(stem + ".png", "wb") as f:
                        f.write(group.image)
                if group.text is not None:
                    with open(stem + ".txt", "wb") as f:
                        f.write(group.text.encode("utf-8"))

    @classmethod
    def _save_checkpoint(cls, epoch: int, save_dir: str, run_opts: RunOpts, problem: Problem,
                         fractional_results: List[FractionalPerformanceSummary],
                         base_filename: str) -> None:
        # replicas are identical after every step, so one rank's state stands for all; the
        # rank with local_rank 0 is the one that serialised it
        donors = [r for r in fractional_results if r.modelBuffer]
        if not donors:
            raise RuntimeError("no worker serialised its model state")
        donor = donors[0]
        test_io = None
        for split in (Split.HELDOUT, Split.TEST, Split.TRAIN):
            if split in donor.performance:
                test_io = donor.performance[split].testIO
                break
        if test_io is None:
            raise RuntimeError("No splits found")
        test_input = [torch.stack([s.data[i] for s in test_io]) for i in range(len(test_io[0].data))]
        test_output = [torch.stack([s.output[i] for s in test_io])
                       for i in range(len(test_io[0].output))]
        model = _torch_load(io.BytesIO(donor.modelBuffer), map_location="cpu")
        optimizer_state = _torch_load(io.BytesIO(donor.optimizerStateBuffer), map_location="cpu")
        ema = optimizer_state.pop(EMA_STATE_KEY, None)       # the main checkpoint keeps its format

        logger.info("==> saving checkpoint to %s", str(save_dir))
        stem = os.path.join(save_dir, base_filename)
        with ExitStack() as stack:
            f_ckpt = stack.enter_context(open(stem, "wb"))
            f_model = stack.enter_context(open(stem + ".model", "wb"))
            f_data = stack.enter_context(open(stem + ".test_data", "wb"))
            f_anno = stack.enter_context(open(stem + ".annotate_param", "wb"))
            torch.save({"epoch": epoch, "optimizer": optimizer_state,
                        "state_dict": model.state_dict()}, f_ckpt)
            torch.save(model, f_model)       # whole module: loadable without the class layout
            torch.save({"test_input": test_input, "test_output": test_output}, f_data)
            torch.save(problem.anno_param._asdict() if problem.anno_param else {}, f_anno)
            if ema is not None:
                with open(stem + EMA_SUFFIX, "wb") as f_ema:
                    torch.save({"epoch": epoch, "decay": ema["decay"], "updates": ema["updates"],
                                "state_dict": ema["state_dict"]}, f_ema)

    # ------------------------------------------------------------------------------------------
    # parent side: collecting per-epoch results from the ranks
    # ------------------------------------------------------------------------------------------
    @classmethod
    def _collect_direct_fractional_results(cls, args: SolverWorkerArgs
                                           ) -> Iterator[List[FractionalPerformanceSummary]]:
        for res in cls._run_solver_worker(args):
            yield [res]

    @classmethod
    def _collect_process_fractional_results(cls, processes, parent_pipes: List[Connection],
                                            cleanup_flag
                                            ) -> Iterator[List[FractionalPerformanceSummary]]:
        pending: DefaultDict[int, List[FractionalPerformanceSummary]] = defaultdict(list)
        finished: List[Connection] = []
        try:
            while len(finished) < len(processes):
                for pipe in wait_pipes(parent_pipes, 5):
                    try:
                        msg = pipe.recv()
                    except EOFError:
                        if pipe not in finished:
                            raise Exception("Child process failed to exit cleanly.")
                        logger.info("Worker process has exited")
                        continue
                    if msg is None:
                        logger.info("Worker process ready to exit")
                        finished.append(pipe)
                    elif isinstance(msg, Exception):
                        logger.info("Received exception from child process")
                        raise msg
                    else:
                        pending[msg.epoch].append(msg)
                        if len(pending[msg.epoch]) == len(processes):
                            yield pending.pop(msg.epoch)
        except Exception:
            logger.exception("Unexpected error in solve")
            cleanup_flag.set()
            logger.info("Sending SIGTERM to all child processes.")
            for p in processes:
                logger.info("Killing process with pid " + str(p.pid))
                p.terminate()
            raise
        finally:
            cleanup_flag.set()
            logger.info("Joining worker processes")
            for p in processes:
                p.join()

    # ------------------------------------------------------------------------------------------
    # entry point
    # ------------------------------------------------------------------------------------------
    @classmethod
    def solve(cls, run_opts: RunOpts, problem: Problem, *, group_name: Optional[str],
              init_method: str, node_idx: int = 0, node_count: int = 1, memory_quota: int = 0,
              precision: Optional[Precision] = None, graph: Optional[bool] = None,
              layer_adaptation: Optional[LayerAdaptation] = None,
              grad_accumulation: Optional[int] = None,
              ema_decay: Optional[float] = None
              ) -> Iterator[PerformanceSummary]:
        """The reference's entry point (solver.py:728-739) plus two keyword-only extensions:

        ``precision``  ``Precision.FP32`` (default; parity with the reference's arithmetic) or
                       ``Precision.BF16`` (bf16 forward/backward/gradients, fp32 master weights and
                       optimizer state — the benchmarked configuration) or ``Precision.FP8``
                       (BF16 with the qualifying Linear layers' GEMMs on the FP8 tensor cores,
                       see ``types.Precision``).  None: FRL_B200_PRECISION.
        ``graph``      True: replay the training step from a CUDA graph once a batch signature
                       has run 2 eager steps (the Problem's forward must be capturable: static
                       shapes, no host syncs; a failed capture falls back to eager launches).
                       None: FRL_B200_CUDA_GRAPH (default off).
        ``layer_adaptation``  ``LayerAdaptation.LARS`` (with ``OptAlgorithm.SGD``) or ``.LAMB`` (with
                       ``OptAlgorithm.ADAM``, no amsgrad): layer-wise trust-ratio updates for large
                       batches, see ``types.LayerAdaptation``; any other combination raises
                       ``ValueError`` before a rank starts.  None: FRL_B200_LAYER_ADAPTATION
                       (default ``none``).  ``Mode.EVAL`` ignores it.
        ``grad_accumulation``  k >= 1 microbatches per optimizer update (gradient accumulation).
                       ``batchSize`` stays the rows of one per-rank microbatch.  Within a training
                       split the microbatches are grouped k at a time: microbatch j closes a group
                       if (j + 1) % k == 0 or it is the split's last, so the last group may be
                       short; no group crosses a split or epoch boundary (checkpoints keep their
                       format and a resumed run is exact).  With g_i the gradient of microbatch i's
                       (mean-reduced) loss, n_i its rows, B = batchSize and N the group's rows, the
                       update uses  G = (1/world) * sum_ranks sum_i (n_i/B) * g_i * (B/N),  summed
                       on the device into an fp32 accumulator (K10).  For MSE and cross-entropy
                       without ignored targets G is the gradient of one batch of N rows; with
                       ``ignore_index`` or a masked loss it is the row-weighted mean of the
                       per-microbatch means, as in every framework's accumulation.  Adam's / LAMB's
                       step count and the optimizer state dict count updates; the NaN guard, loss
                       log rows, ``lossLoggingFreq``, metrics, the watchdog, BatchNorm statistics
                       and the buffer broadcast stay per microbatch; the LR schedule stays per
                       epoch.  Not combinable with ``GradNormWeightedCriterion`` (ValueError).
                       None: FRL_B200_GRAD_ACCUM (default 1: no accumulator, today's step).  Any
                       value but an integer >= 1 raises ``ValueError`` before a rank starts.
                       ``Mode.EVAL`` ignores it.
        ``ema_decay``  d in [0, 1): keep an exponential moving average (EMA) of the weights; 0 is
                       off.  The same values as ``AveragedModel(model, multi_avg_fn=
                       get_ema_multi_avg_fn(d), use_buffers=True)`` with ``update_parameters``
                       called after every ``optimizer.step()``.  It covers the model's trainable
                       parameters (arena range ``[0, model_end)``; criterion parameters are not
                       averaged) and is updated once per optimizer update (with gradient
                       accumulation by the microbatch that closes a group): the first update
                       copies the fp32 master weights, every later one is
                       ``ema = lerp(ema, w, 1 - d)`` in fp32 on them, torch's lerp formula with
                       ``1 - d`` formed in double (K11, one launch).  Floating buffers (BatchNorm
                       statistics) get the same lerp through ``torch._foreach_lerp_``,
                       non-floating ones are copied.  In a TRAIN run every split other than
                       ``Split.TRAIN`` is evaluated with the EMA weights and buffers (swapped
                       into the arena and the bf16 shadow for the split, swapped back bit for
                       bit after it), so its losses, metrics and ``testIO`` samples, and hence
                       ``<stem>.test_data``, belong to the EMA model.  Every checkpoint gets a
                       ``<stem>.ema`` next to it: ``{"epoch", "decay", "updates",
                       "state_dict"}``, the state dict keyed like the main checkpoint's, so
                       ``initialModelPath=<stem>.ema`` with ``Mode.EVAL`` evaluates the EMA model;
                       the main checkpoint and ``<stem>.model`` keep the live weights and their
                       format.  A resume loads ``<save_dir>/.checkpoint.pth.ema`` if it exists
                       and was saved at the checkpoint's epoch (bit-exact continuation); without
                       it, with one of another epoch, or with ``initialModelPath``, the EMA starts
                       from the loaded weights with 0 updates.  Several GPUs: the EMA
                       turns the fused NVLS step (K7) off, every rank keeps the same averaged
                       parameters (buffers: see INTEGRATION.md; rank 0's are saved).
                       None: FRL_B200_EMA_DECAY (default 0).  Any value but a real number in
                       [0, 1) raises ``ValueError`` before a rank starts.  ``Mode.EVAL`` ignores it.
        """
        adapt = LayerAdaptation.NONE
        accum = 1
        decay = 0.0
        if run_opts.mode == Mode.TRAIN:
            adapt = resolve_layer_adaptation(layer_adaptation)
            check_layer_adaptation(run_opts.optim, adapt)
            accum = resolve_grad_accumulation(grad_accumulation)
            decay = resolve_ema_decay(ema_decay)
        n_visible = 0 if run_opts.cpuonly else _cuda_device_count_without_poisoning_fork()
        if n_visible == 0:
            raise RuntimeError(
                "frl_b200 runs the training step on H100 GPUs only (cpuonly=%s, visible CUDA "
                "devices=%d); there is no CPU path" % (run_opts.cpuonly, n_visible))
        run_device = Device.GPU
        if run_opts.singleThreaded:
            device_count, world_size = 1, 1
        else:
            device_count = n_visible
            world_size = device_count * node_count
        logger.info("World size %d, device count %d" % (world_size, device_count))
        num_workers = min(device_count, world_size)

        save_dir = problem.save_dir + (str(node_idx) if node_count > 1 else "")
        os.makedirs(save_dir, exist_ok=True)
        assert len(problem.datasets) > 0, "datasets cannot be empty"
        # big datasets checkpoint every epoch, small ones every fifth
        save_every = 1 if len(problem.datasets[0]) > 300_000 else 5
        prec = resolve_precision(precision)

        logger.info("Parent process has pid " + str(os.getpid()))
        # fork keeps un-picklable Problems working (as in the reference) but is only safe while
        # this process holds no CUDA context
        use_fork = run_opts.singleThreaded or _fork_is_safe()
        if not use_fork:
            logger.info("CUDA already touched in the parent: ranks are spawned (Problem must pickle)")
        ctx = multiprocessing.get_context("fork" if use_fork else "spawn")
        cleanup_flag = ctx.Event()
        processes, parent_pipes = [], []
        args: Optional[SolverWorkerArgs] = None
        for local_rank in range(num_workers):
            args = SolverWorkerArgs(
                run_opts=run_opts, problem=problem, save_dir=save_dir, run_device=run_device,
                node_idx=node_idx, node_count=node_count,
                rank=node_idx * device_count + local_rank, local_rank=local_rank,
                world_size=world_size, group_name=group_name, init_method=init_method,
                cache=None, precision=prec, save_every=save_every, graph_step=graph,
                layer_adaptation=adapt, grad_accumulation=accum, ema_decay=decay)
            if not run_opts.singleThreaded:
                parent_conn, child_conn = ctx.Pipe(duplex=False)
                proc = ctx.Process(target=cls._solver_worker_process,
                                   kwargs={"solver_worker_args": args,
                                           "comms_connection": child_conn,
                                           "cleanup_flag": cleanup_flag})
                proc.start()
                parent_pipes.append(parent_conn)
                processes.append(proc)
                logger.info("Started worker with rank: %d pid: %d", local_rank, proc.pid)
        assert args is not None
        if run_opts.singleThreaded:
            assert num_workers == 1, "Single threaded run cannot use multiple workers"
            results = cls._collect_direct_fractional_results(args)
        else:
            results = cls._collect_process_fractional_results(processes, parent_pipes, cleanup_flag)

        for res in results:
            epoch = res[0].epoch
            epoch_stats = cls._aggregate_fractional_results(run_opts, problem, res)
            if run_opts.mode == Mode.TRAIN:
                final = epoch == run_opts.nEpochs
                if epoch % save_every == 0 or final:
                    cls._save_epoch_summary(epoch, save_dir, epoch_stats)
                    cls._save_checkpoint(epoch, save_dir, run_opts, problem, res,
                                         "final_model.pth" if final else CHECKPOINT_NAME)
            yield PerformanceSummary(epoch=epoch, performance=epoch_stats, save_dir=str(save_dir))
