"""Numeric modes of the CUDA engine (DESIGN.md section 4).  Every mode multiplies 16-bit operands on wgmma (same tensor rate
for fp16 and bf16) and accumulates in fp32 registers; they differ in what the 16 bits are:

  "bf16"     bf16 activations and weights.  8-bit significand: feature maps ~8e-3 (norm-wise) off the fp32 reference.  Cannot
             overflow on unnormalised activations.  BASELINE.json config 2 names this dtype; kept as a labelled bench line.
  "fp16"     IEEE-half activations and weights (11-bit significand): ~1.0e-3.
  "fp16_w2"  IEEE-half activations; every backbone / FPN weight is the SUM OF TWO halves (hi + lo, both multiplied with the same
             activation tile into one accumulator -- nrpn_conv_desc.wsplit), so only the activations carry rounding error:
             ~8e-4, the mode that meets north_star's "<= 1e-3 rel on feature maps" with margin.  The head keeps single fp16
             weights (it is tensor-pipe bound and comes after the feature maps).

The mode is an explicit constructor argument of the module mirrors (`precision=`), shows up in their repr and in bench.py's JSON
line; NRPN_PRECISION overrides the default for A/B runs.
"""
import os

MODES = ("bf16", "fp16", "fp16_w2")
DEFAULT = os.environ.get("NRPN_PRECISION", "fp16_w2")
if DEFAULT not in MODES:
    raise ValueError(f"NRPN_PRECISION must be one of {MODES}, got {DEFAULT!r}")


def resolve(precision=None) -> str:
    p = DEFAULT if precision is None else precision
    if p not in MODES:
        raise ValueError(f"precision must be one of {MODES}, got {p!r}")
    return p


def bench_dtype(precision: str) -> str:
    return {"bf16": "bf16", "fp16": "f16", "fp16_w2": "f16 (backbone weights as hi+lo f16 pairs)"}[precision]


class EngineHolder:
    """Mixin of the module mirrors that cache an engine (CUDA graphs, streams, ctypes objects): keeps it out of pickles and deep copies
    (torch.save(model), copy.deepcopy, spawn-based DDP), like the reference's plain nn.Modules support."""

    def __getstate__(self):
        d = self.__dict__.copy()
        for k in ("_engine", "_engine_key", "_train_engine"):
            if k in d:
                d[k] = None
        return d
