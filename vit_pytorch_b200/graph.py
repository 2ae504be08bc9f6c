"""CUDA-graph replay of a fused forward at a fixed input shape (small-batch serving).

At batch 512 the 65 launches of a ViT-B/16 forward are hidden behind 20 ms of GPU work; at batch 1-64 the host side
(ctypes calls, tensor-map look-ups, Python) is what the GPU waits for.  `GraphedForward` captures one fused forward --
every launch of libb200vit.so goes to torch's current stream, which is the capture stream inside `torch.cuda.graph` --
and replays it with static input / output buffers:

    fwd = GraphedForward(model, example_images)        # model: ViT / SimpleViT family, eval, CUDA bf16
    logits = fwd(images)                               # same shape / dtype / device as the example

Only fixed-shape models qualify (NaViT builds its index arrays on the host per call).  The output tensor is reused by
the next call; clone it if it has to survive.
"""
from __future__ import annotations

import torch


class GraphedForward:
    def __init__(self, model: torch.nn.Module, example: torch.Tensor, warmup: int = 3) -> None:
        reason = model.fused_reason(example) if hasattr(model, "fused_reason") else "model has no fused path"
        with torch.inference_mode():
            reason = model.fused_reason(example) if hasattr(model, "fused_reason") else reason
        if reason is not None:
            raise RuntimeError(f"GraphedForward needs a call that takes the fused path: {reason}")
        # a model whose fused forward varies from call to call at a fixed shape (CaiT's layer dropout) says why here
        reason = model.graph_reason() if hasattr(model, "graph_reason") else None
        if reason is not None:
            raise RuntimeError(f"GraphedForward cannot replay this model: {reason}")
        self.model = model
        self.static_in = example.clone()
        self.graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream(device=example.device)
        side.wait_stream(torch.cuda.current_stream(example.device))
        with torch.cuda.device(example.device), torch.inference_mode():
            with torch.cuda.stream(side):                       # weights prepared, attributes set, descriptors cached
                for _ in range(warmup):
                    model(self.static_in)
            torch.cuda.current_stream(example.device).wait_stream(side)
            torch.cuda.synchronize(example.device)
            with torch.cuda.graph(self.graph):
                self.static_out = model(self.static_in)

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        if x.shape != self.static_in.shape or x.dtype != self.static_in.dtype or x.device != self.static_in.device:
            raise ValueError(f"GraphedForward was captured for {tuple(self.static_in.shape)} {self.static_in.dtype} on "
                             f"{self.static_in.device}, got {tuple(x.shape)} {x.dtype} on {x.device}")
        self.static_in.copy_(x, non_blocking=True)
        self.graph.replay()
        return self.static_out
