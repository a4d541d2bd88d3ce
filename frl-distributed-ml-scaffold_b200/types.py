"""Option records and enums of the scaffold plugin API.

Mirrors the public names of the reference's ``types.py`` (reference types.py:36-127) so a
``Problem`` written against the reference constructs the same ``RunOpts``/``OptimOpts`` here.
Field names, order and defaults are the contract; the plotly dependency of the reference's
``SampleSummary.plot`` is dropped (any JSON-serialisable figure dict is accepted).
"""
from enum import Enum
from typing import Any, NamedTuple, Optional

import numpy as np


# --- enums (values are the strings the reference uses on the wire / in logs) ---------------

class ShuffleType(Enum):
    RANDPERM = "randperm"
    PER_NODE_RANDPERM = "per_node_randperm"


class Split(Enum):
    TRAIN = "training"
    TEST = "testing"
    HELDOUT = "heldOut"


class Device(Enum):
    CPU = "cpu"
    GPU = "cuda"


class Mode(Enum):
    EVAL = "eval"
    TRAIN = "train"


class OptAlgorithm(Enum):
    RMSPROP = "rmsprop"
    SGD = "sgd"
    ADAM = "adam"


class LossType(Enum):
    MSE = "mse"
    CrossEntropy = "crossentropy"


class LRSchedulerAlgorithm(Enum):
    DropEpochs = "drop"
    WarmupMultiStepLR = "multistep"


class Precision(Enum):
    """Extension (not in the reference, which is fp32-only): arithmetic of the train step.

    FP32  - parameters, gradients and optimizer state fp32 (reference parity mode, 1e-5 rel).
    BF16  - bf16 shadow weights + bf16 gradients for forward/backward, fp32 master weights and
            optimizer state in the arena, written by the fused update kernel (1e-2 tolerance).
    FP8   - BF16 in every respect (storage, gradients, master weights, optimizer state,
            checkpoints), except that the exact ``nn.Linear`` layers that qualify (weight in the
            bf16 shadow, in/out features multiples of 16, and per call a row count that is a
            multiple of 16) run their forward, input-gradient and weight-gradient GEMMs on the
            FP8 tensor cores: e4m3 activations and weights, e5m2 output gradients, bf16 results.
            Scaling is current per-tensor scaling: each operand is quantised at a power-of-two
            scale derived on the device from its own amax in the same step (K9), so the run keeps
            no scaling state.  Other layers, the fused task heads and calls that do not qualify
            run exactly as in BF16.
    """
    FP32 = "fp32"
    BF16 = "bf16"
    FP8 = "fp8"

    @property
    def bf16_storage(self) -> bool:
        """bf16 shadow weights and bf16 gradients around fp32 master weights (BF16 and FP8)."""
        return self is not Precision.FP32


class LayerAdaptation(Enum):
    """Extension (not in the reference): layer-wise learning-rate adaptation for large-batch
    training, chosen with ``Solver.solve(..., layer_adaptation=...)`` or
    ``FRL_B200_LAYER_ADAPTATION``.  Per arena slot, in fp32, with ``g^ = g * grad_scale`` (times the
    clip coefficient when ``gradientClip`` is on, model parameters only), ``w`` the fp32 master
    weights before the update and ``lr`` the scheduled rate.

    A tensor is ADAPTED if it has 2 or more dimensions (Linear and conv weights, embeddings).  0-
    and 1-D tensors (biases, normalisation affine parameters, criterion parameters) get ratio 1
    and no weight decay.  The rule is fixed.

    NONE - the plain ``OptimOpts.algo`` update.
    LARS - layer adaptation on the SGD rule (You et al. 2017); needs ``algo == SGD``.  Trust
           coefficient eta = 0.001 (fixed), mu = ``momentum``, no dampening:
             adapted:     ratio = eta*||w|| / (||g^|| + wd*||w||) if ||w|| > 0 and ||g^|| > 0, else 1;
                          d = ratio * (g^ + wd*w)
             not adapted: d = g^
             buf = d on the first step, else mu*buf + d;  w -= lr*buf   (mu = 0: no buffer)
           The buffer has torch SGD's units: checkpoints load into ``torch.optim.SGD``.
    LAMB - layer adaptation on the Adam rule (You et al. 2019); needs ``algo == ADAM`` and
           ``amsgrad == False``.  beta = (0.9, 0.999), eps = ``epsilon``, lam = ``weightDecay`` if
           adapted else 0, t = the arena's step count (as for the fused Adam):
             m = m + (1-beta1)*(g^ - m);  v = beta2*v + (1-beta2)*g^^2
             u = (m / bc1) / (sqrt(v) / sqrt(bc2) + eps) + lam*w          bc_i = 1 - beta_i^t
             ratio = ||w|| / ||u|| if adapted and ||w|| > 0 and ||u|| > 0, else 1;  w -= lr*ratio*u
           The weight decay is DECOUPLED (part of u), unlike the L2-coupled decay of this
           package's Adam.  The state is Adam's: checkpoints load into ``torch.optim.Adam`` and an
           Adam checkpoint resumes under LAMB.

    A non-finite gradient still gives non-finite weights (the ratio-1 branch passes a NaN on), so
    the NaN-loss check fires.  Both run as two tile-parallel kernels over whole tensors (K2-lw), so
    the gradients are all-reduced per bucket and the update runs once after backward: no eager
    per-bucket update and no fused NVLS step.  ``Mode.EVAL`` ignores the setting.
    """
    NONE = "none"
    LARS = "lars"
    LAMB = "lamb"


class OptimizerState(Enum):
    """Extension (not in the reference): how Adam's optimizer state is stored, chosen with
    ``Solver.solve(..., optimizer_state=...)`` or ``FRL_B200_OPTIMIZER_STATE``.

    FP32 - ``exp_avg`` and ``exp_avg_sq`` as fp32 arena-shaped vectors (8 B per parameter).
    Q8   - 8-bit block-wise dynamic quantization (Dettmers et al., ICLR 2022): per moment one byte
           per parameter plus one fp32 absmax per block of 256 consecutive elements of a tensor
           (about 2.03 B per parameter).  ``exp_avg`` is sign + 7-bit index into a 128-entry
           magnitude table, ``exp_avg_sq`` an 8-bit index into a 256-entry table (the dynamic
           tree map; ``fused_optim.q8_tables``); values decode to ``table[k] * absmax``.  Every
           step decodes, applies this package's Adam rule in fp32 (weights and bf16 shadow from
           the fp32 moments of the step), then re-encodes each block to the nearest table entry
           (K2-q8, one launch after backward).  Needs ``algo == ADAM``, ``amsgrad == False`` and
           ``LayerAdaptation.NONE``.  The state dict is ``torch.optim.Adam``'s with decoded fp32
           moments.  Gradients are all-reduced per bucket and the update runs once after backward:
           no eager per-bucket update and no fused NVLS step.  ``Mode.EVAL`` ignores the setting.
           With ``channels_last=True`` a block is 256 consecutive elements of the conv weight's
           (O, kh, kw, I) order, so its elements, absmax and codes differ from an NCHW run's; the
           state dict is still torch's, and loads in either layout re-encode it.
    """
    FP32 = "fp32"
    Q8 = "8bit"


class MasterWeights(Enum):
    """Extension (not in the reference): where the authoritative copy of the model's weights lives
    in a BF16 / FP8 run, chosen with ``Solver.solve(..., master_weights=...)`` or
    ``FRL_B200_MASTER_WEIGHTS``.

    FP32 - an fp32 master vector beside the bf16 weights forward and backward read; every update
           reads and rewrites the master and writes the bf16 copy (round to nearest even).
    BF16 - the bf16 weights are the only copy of the model range ``[0, model_end)`` of the arena: 4 B
           per model parameter less resident memory.  Every update widens the bf16 weight to fp32,
           applies the unchanged fp32 rule and rounds the result stochastically back to bf16 (K2-sr /
           K2-mt-sr), so that the expected stored weight equals the fp32 result and updates below half
           a bf16 ulp are not lost.  The 16 random bits of arena element ``i`` at update ``t`` come
           from Philox4x32-10 keyed by the optimizer's ``sr_seed`` (include/frl_b200.h, K2-sr); the
           param group keeps ``sr_seed`` and ``sr_updates``, so a resumed run continues bit for bit.
           Criterion parameters keep their fp32 master.  Checkpoints keep their fp32 format (the
           values are bf16-exact) and load in either mode.  Allowed with SGD, Adam / AdamW and RMSprop
           in ``Precision.BF16`` / ``FP8``; refused with ``Precision.FP32``, layer adaptation, 8-bit
           optimizer state, Adafactor and Muon.  On one GPU with SGD the dW-GEMM update (K12) runs its
           stochastic-rounding form; with several GPUs the fused NVLS step (K7) is not used.  The EMA
           file keeps the fp32 EMA itself.  ``Mode.EVAL`` ignores the setting.
    """
    FP32 = "fp32"
    BF16 = "bf16"


class ScheduleFree(NamedTuple):
    """Extension (not in the reference): the settings of Schedule-Free optimization (Defazio et al.
    2024, *The Road Less Scheduled*), chosen with ``Solver.solve(..., schedule_free=ScheduleFree(...))``
    (``True`` for these defaults) or ``FRL_B200_SCHEDULE_FREE`` / ``FRL_B200_SCHEDULE_FREE_WARMUP``.

    warmup_steps     - updates over which lr ramps linearly up, (k+1)/warmup_steps, then stays flat
    r, weight_lr_power - the averaging weight of update k is (k+1)^r * lr_max^weight_lr_power (the
                       schedulefree package's defaults 0 and 2)
    """
    warmup_steps: int = 0
    r: float = 0.0
    weight_lr_power: float = 2.0


# --- records ---------------------------------------------------------------------------------

class SampleSummary(NamedTuple):
    image: Optional[np.ndarray] = None
    text: Optional[str] = None
    plot: Optional[Any] = None          # plotly Figure or a figure dict
    source: Optional[str] = None


class LRSchedulerOpts(NamedTuple):
    algo: LRSchedulerAlgorithm = LRSchedulerAlgorithm.DropEpochs


class OptimOpts(NamedTuple):
    """Optimizer options (reference types.py:85-93).  How the H100 step consumes them:

    algo          which fused update rule K2/K7 applies (``frl_sgd_momentum`` / ``frl_adam`` /
                  ``frl_rmsprop``); anything else raises ``ValueError`` like the reference
    lr            base rate; the per-epoch scheduler writes the current value into the kernel
                  arguments (or the device-resident ``dyn`` block under CUDA-graph replay)
    lr_scheduler  ``drop`` or ``multistep`` closed forms, stepped once per epoch
    weightDecay   L2-COUPLED decay folded into the gradient read, on every parameter (model and
                  criterion) — this is ``torch.optim``'s ``weight_decay``; for AdamW's decoupled
                  decay with Adam, pass ``Solver.solve(..., adamw=True)``
    momentum      SGD momentum AND RMSprop momentum (the reference feeds both from this field)
    epsilon       Adam only (RMSprop keeps torch's 1e-8), as in the reference's factory
    amsgrad       Adam: adds the running maximum of the second moment (a third state vector)
    gradientClip  > 0: global-norm clip of the MODEL parameters' gradients (K3 computes the
                  coefficient on the device, K2 applies it); turns the fused NVLS step off

    Layer-wise adaptation (LARS on SGD, LAMB on Adam) is not a field here but a keyword of
    ``Solver.solve``: see ``LayerAdaptation``.
    """
    algo: OptAlgorithm
    lr: float = 0.001
    lr_scheduler: LRSchedulerOpts = LRSchedulerOpts()
    weightDecay: float = 0.00001
    momentum: float = 0.9
    epsilon: float = 1e-8
    amsgrad: bool = False
    gradientClip: float = 0.0


class RunOpts(NamedTuple):
    """Run options (reference types.py:102-121).  Field names, order and defaults are the
    reference's; what each means on the H100 path:

    batchSize                   minibatch PER RANK (weak scaling, as DDP in the reference)
    cpuonly                     must stay False: there is no CPU path, ``Solver.solve`` raises
    nEpochs                     epochs to train; also fixes the LR drop / warm-up milestones
    maxEpochImages              > 0: train on the first N samples of each dataset only
    numThreads                  DataLoader workers of the per-sample input path; the batched
                                device input path (``pinned_fields`` datasets) ignores it
    numIOThreads                accepted for compatibility (storage-layer option)
    metricAmortizationSchedule  every N minibatches the retained outputs/targets are folded
                                into per-sample metrics — on a worker thread here, so the hook's
                                device-to-host read never stalls the step
    initialModelPath            ``state_dict`` to start from (strict in EVAL mode)
    mode                        TRAIN or EVAL (EVAL runs every split forward-only, writes nothing)
    numVisualizedSamples        random + worst-k samples kept per split for the summaries
    singleThreaded              run the single rank in the calling process instead of forking
    outputTTL                   accepted for compatibility (storage-layer option)
    lossLoggingFreq             > 0: log the loss row every N minibatches (a lagged read of the
                                pinned loss log, not a sync)
    debugGrad                   per-task gradient norms at the last shared parameter every 10
                                minibatches; keeps the step on eager launches and stock autograd
    shuffleType                 how ``ScaffoldSampler`` partitions the permutation across ranks
    minibatchTimeoutMs          watchdog: a minibatch longer than this raises ``TimeoutError``
    """
    optim: OptimOpts
    batchSize: int
    cpuonly: bool = False
    nEpochs: int = 75
    maxEpochImages: int = 0
    numThreads: int = 4
    numIOThreads: int = 5
    metricAmortizationSchedule: int = 10
    initialModelPath: Optional[str] = None
    mode: Mode = Mode.TRAIN
    numVisualizedSamples: int = 36
    singleThreaded: bool = False
    outputTTL: int = 0
    lossLoggingFreq: int = 0
    debugGrad: bool = False
    shuffleType: ShuffleType = ShuffleType.RANDPERM
    minibatchTimeoutMs: int = 1000 * 60 * 60


def _fill_namedtuple(cls, args, kwargs):
    merged = dict(cls._field_defaults)
    free = [name for name in cls._fields if name not in kwargs]
    merged.update(zip(free, args))
    merged.update(kwargs)
    return merged


class OptimOptsBase(OptimOpts):
    """Subclassable variant: positional args fill the fields not given by keyword."""

    def __new__(cls, *args, **kwargs):
        return super().__new__(cls, **_fill_namedtuple(cls, args, kwargs))


class RunOptsBase(RunOpts):
    def __new__(cls, *args, **kwargs):
        return super().__new__(cls, **_fill_namedtuple(cls, args, kwargs))
