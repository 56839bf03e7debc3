"""The dynamic tile scheduler of the implicit-GEMM convolution (conv3d_igemm.cu).

Each CTA starts with its own tile and then claims the next from a per-launch counter that the launch's last CTA resets, so
which CTA runs which tile changes from run to run while every output element keeps its reduction order.  For every tile kind,
on layers with more tiles than resident CTAs:
  - two launches back to back, then replays of a captured CUDA graph: every output equals the first bit for bit, and no
    element is left unwritten (a counter that was not reset would make the next launch skip tiles);
  - a launch that starts while another stream's convolution holds part of the SMs, so that some of its CTAs start late:
    still the same bits."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

# (cin, cout, k, wsplit, instance nrpn_conv3d_variant names): 32^3 voxels = 256 tiles of 128 voxels per scene
CASES = {
    "long64": (128, 64, 3, False, "igemm<64,8,1,tma-epilogue>"),
    "long128": (128, 128, 3, False, "igemm<128,6,1,tma-epilogue>"),
    "long256": (128, 256, 3, False, "igemm<256,4,1,tma-epilogue>"),
    "long256_wsplit": (128, 256, 3, True, "igemm<256,2,1,tma-epilogue,wsplit>"),
    "short64": (256, 256, 1, False, "igemm<64,2,2,tma-epilogue>"),
}
DIMS, N = (32, 32, 32), 2


class Layer:
    def __init__(self, ops, cin, cout, k, wsplit, dims=DIMS, n=N, seed=0):
        from nerf_rpn_b200 import packing
        self.ops, self.cin, self.cout, self.dims, self.n = ops, cin, cout, dims, n
        g = torch.Generator(device="cuda").manual_seed(seed)
        w = torch.randn((cout, cin, k, k, k), device="cuda", generator=g) / math.sqrt(cin * k ** 3)
        self.wp, self.taps = packing.pack_conv_weight(w, dtype=torch.bfloat16, split=wsplit)
        self.shift = packing.pad_shift(torch.randn((cout,), device="cuda", generator=g), self.wp.shape[-2])
        self.x = torch.randn((n, *dims, cin), device="cuda", generator=g).to(torch.bfloat16)
        self.y = torch.empty((n, *dims, cout), device="cuda", dtype=torch.bfloat16)

    def args(self):
        return [self.ops.ConvLevelArgs(self.x, self.y, self.n, self.dims, self.dims, self.cout)]

    def variant(self):
        return self.ops.conv3d_variant(self.args(), self.wp, self.shift, self.cin, self.cout, self.taps, relu=True)

    def launch(self):
        self.ops.conv3d_fprop(self.args(), self.wp, self.shift, self.cin, self.cout, self.taps, relu=True)

    def run(self):
        """One launch into a NaN-filled output; returns its bits."""
        self.y.fill_(float("nan"))
        self.launch()
        torch.cuda.synchronize()
        return self.y.view(torch.int16).clone()


@pytest.fixture(scope="module")
def ops():
    from nerf_rpn_b200 import ops as o
    return o


def _check(first, got, what):
    assert torch.equal(got, first), f"{what}: {(got != first).sum().item()} elements differ from the first launch"


@pytest.mark.parametrize("case", list(CASES))
def test_repeat_and_graph_replay(ops, case):
    cin, cout, k, wsplit, name = CASES[case]
    layer = Layer(ops, cin, cout, k, wsplit)
    assert layer.variant() == name
    first = layer.run()
    assert not torch.isnan(layer.y.float()).any(), "tiles left unwritten"
    _check(first, layer.run(), "second launch")

    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        layer.launch()
        layer.launch()                       # two launches in one graph: the second takes the counter the first reset
    for i in range(4):
        layer.y.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        _check(first, layer.y.view(torch.int16), f"graph replay {i}")


@pytest.mark.parametrize("case", ["long256", "short64"])
def test_late_starting_ctas(ops, case):
    cin, cout, k, wsplit, _ = CASES[case]
    layer = Layer(ops, cin, cout, k, wsplit)
    first = layer.run()
    # a 3^3 256 -> 256 convolution over 64 tiles on a second stream: one CTA of ~225 KB shared memory on each of 64 SMs
    other = Layer(ops, 256, 256, 3, False, dims=(8, 32, 32), n=1, seed=1)
    assert other.variant() == "igemm<256,4,1,tma-epilogue>"
    other_first = None
    side = torch.cuda.Stream()
    for i in range(3):
        layer.y.fill_(float("nan"))
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            other.launch()
        layer.launch()
        torch.cuda.synchronize()
        _check(first, layer.y.view(torch.int16), f"launch {i} beside another stream's convolution")
        if other_first is None:
            other_first = other.y.view(torch.int16).clone()
        else:
            _check(other_first, other.y.view(torch.int16), f"second-stream convolution {i}")
