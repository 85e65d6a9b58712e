"""CUDA-graph capture of static-shape forwards of these modules (SURVEY.md §8(f)4, latent stack).

The latent self-attention stack of Perceiver IO runs L layers (6-26) of small kernels on a FIXED (B, N, D) latent
array: per layer a LayerNorm-folded QKV GEMM, the attention kernel, the output projection and the MLP — at N = 256 the
step is bound by launch latency and host-side bookkeeping (plan lookup, tensor-map encoding, Python), not by the
kernels.  Everything this package launches is capturable: it allocates through torch's caching allocator, encodes
tensor maps on the host, never synchronises, and its one-time work (work plans, `cudaFuncSetAttribute`, folded
weights) happens during the warm-up calls.  ``GraphedForward`` records the whole forward once and replays it with
one `cudaGraphLaunch` per call.

    block = encoder.self_attn_1                       # a SelfAttentionBlock of this package or a patched reference one
    fast = GraphedForward(lambda x: block(x).last_hidden_state, example_latents)
    y = fast(latents)                                 # same values as block(latents).last_hidden_state

Shapes, dtypes and the parameter TENSORS must stay the same between capture and replay (in-place parameter updates are
fine as long as the folded-weight caches are refreshed by an eager call before re-capturing); inputs are copied into the
static buffers the graph was recorded with, outputs are views of the graph's static outputs (valid until the next call).
"""
from __future__ import annotations

from typing import Callable, Sequence

import torch


def _tensors(x):
    if isinstance(x, torch.Tensor):
        return [x]
    if isinstance(x, (list, tuple)):
        return [t for i in x for t in _tensors(i)]
    raise TypeError("GraphedForward functions must return a tensor or a (nested) tuple / list of tensors")


class GraphedForward:
    def __init__(self, fn: Callable, *example_inputs: torch.Tensor, warmup: int = 3):
        if not example_inputs or not all(isinstance(t, torch.Tensor) and t.is_cuda for t in example_inputs):
            raise RuntimeError("GraphedForward needs CUDA example inputs (there is no CPU path)")
        # fn is not kept: a bound method of an owner that holds this object (GraphedDecoder) would make a reference cycle,
        # and the cycle collector could then destroy the graph while another stream is capturing, which invalidates
        # that capture.
        self._inputs = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream(device=self._inputs[0].device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(max(1, warmup)):   # plans, kernel attributes, folded weights, allocator pools
                fn(*self._inputs)
        torch.cuda.current_stream().wait_stream(side)
        self._graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self._graph):
            self._outputs = fn(*self._inputs)
        _tensors(self._outputs)

    def __call__(self, *inputs: torch.Tensor):
        if len(inputs) != len(self._inputs):
            raise ValueError(f"expected {len(self._inputs)} inputs")
        for dst, src in zip(self._inputs, inputs):
            if dst.shape != src.shape or dst.dtype != src.dtype:
                raise ValueError("GraphedForward replays a fixed shape / dtype; re-capture for new shapes")
            dst.copy_(src)
        self._graph.replay()
        return self._outputs


def graph_latent_block(block, example_latents: torch.Tensor, **kwargs) -> Callable[[torch.Tensor], torch.Tensor]:
    """Capture ``block(x, **kwargs).last_hidden_state`` for a SelfAttentionBlock on a fixed latent shape.

    While recording, the row threshold of the self-attention projections is lowered so that the LayerNorm-folded
    one-GEMM QKV projection and the tcgen05 o_proj are what gets captured (4 kernels per layer instead of 7): inside a
    graph there is no host-side dispatch cost to trade against."""
    from . import modules

    old = modules.kv_producer_config["min_rows_latent"]
    modules.kv_producer_config["min_rows_latent"] = modules.kv_producer_config["min_rows"]
    try:
        return GraphedForward(lambda x: block(x, **kwargs).last_hidden_state, example_latents)
    finally:
        modules.kv_producer_config["min_rows_latent"] = old
