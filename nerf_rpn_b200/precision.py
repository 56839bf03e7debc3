"""Numeric modes of the CUDA engine (DESIGN.md section 4).  Every mode multiplies 16-bit operands on wgmma (same tensor rate
for fp16 and bf16) and accumulates in fp32 registers; they differ in what the 16 bits are:

  "bf16"     bf16 activations and weights.  8-bit significand: feature maps ~8e-3 (norm-wise) off the fp32 reference.  Cannot
             overflow on unnormalised activations.  BASELINE.json config 2 names this dtype; kept as a labelled bench line.
  "fp16"     IEEE-half activations and weights (11-bit significand): ~1.0e-3.
  "fp16_w2"  IEEE-half activations; the backbone / FPN weights are the SUM OF TWO halves (hi + lo, both multiplied with the same
             activation tile into one accumulator -- nrpn_conv_desc.wsplit), so only the activations carry rounding error:
             ~8e-4, the mode that meets north_star's "<= 1e-3 rel on feature maps" with margin.  The head keeps single fp16
             weights (it is tensor-pipe bound and comes after the feature maps); split_weights() names every exception.

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


def storage_dtype(precision: str):
    """16-bit format of the activations and the packed weights."""
    import torch
    return torch.bfloat16 if precision == "bf16" else torch.float16


def split_weights(precision: str, role: str, weight, stride: int = 1) -> bool:
    """Whether a layer's weights are packed as hi + lo fp16 planes.  Only under "fp16_w2", and there for every backbone / FPN layer
    (role "backbone") except:
      - 3^3 64 -> <= 64 stride-1 layers: they run on the halo-slab kernel, which takes single weights (conv3d_slab_eligible);
      - role "p2": the P2 output conv (15 % of the scene's FLOPs, tensor-pipe bound); its weight rounding alone contributes ~2e-4
        to P2 (measured by emulation, DESIGN.md section 4);
      - roles "stem" / "stem_s1" (own packed layouts) and "head": single halves."""
    if precision != "fp16_w2" or role != "backbone":
        return False
    cout, cin, taps = weight.shape[0], weight.shape[1], weight[0, 0].numel()
    return not (cin == 64 and cout <= 64 and taps >= 8 and stride == 1)


class EngineHolder:
    """Mixin of the module mirrors that cache an engine (CUDA graphs, streams, ctypes objects): keeps it out of pickles and deep copies
    (torch.save(model), copy.deepcopy, spawn-based DDP), like the reference's plain nn.Modules support."""

    def __getstate__(self):
        d = self.__dict__.copy()
        for k in ("_engine", "_engine_key", "_train_engine"):
            if k in d:
                d[k] = None
        return d

    def _engine_features(self, x):
        """forward() of the backbones: (N,4,W,L,H) fp32 CUDA -> [P2, P3, P4, P5], each (N,256,w,l,h) fp32 (channels_last_3d
        strides), from an engine over this backbone alone, cached per precision."""
        from .engine import RPNInferenceEngine
        precision = resolve(getattr(self, "precision", None))
        if self._engine is None or self._engine.precision != precision:
            self._engine = RPNInferenceEngine(self, precision=precision)
        plan = self._engine.forward_device(x.contiguous())
        return [f.permute(0, 4, 1, 2, 3).float() for f in plan.features]
