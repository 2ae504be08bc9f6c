"""`Extractor` with the interface of `vit_pytorch.extractor.Extractor` (reference extractor.py:18-92): returns the
logits together with the output (or input) of one layer, `vit.transformer` by default.

With the default layer the wrapped model stays on the fused sm_90a path: its forward notices the hook on the
Transformer module and passes the tokens through that module call (engine.hooked_transformer_tokens).  A layer strictly
inside the transformer needs the materialised PyTorch graph, which the model's dispatch then runs for that call.
"""
from __future__ import annotations

from torch import nn


def _map(fn, val):
    return tuple(fn(v) for v in val) if isinstance(val, tuple) else fn(val)


class Extractor(nn.Module):
    def __init__(self, vit, device=None, layer=None, layer_name='transformer', layer_save_input=False,
                 return_embeddings_only=False, detach=True) -> None:
        super().__init__()
        self.vit = vit
        self.data = None
        self.latents = None
        self.hooks = []
        self.hook_registered = False
        self.ejected = False
        self.device = device
        self.layer = layer
        self.layer_name = layer_name
        self.layer_save_input = layer_save_input
        self.return_embeddings_only = return_embeddings_only
        self.detach_fn = (lambda t: t.clone().detach()) if detach else (lambda t: t)

    def _hook(self, _, inputs, output) -> None:
        self.latents = _map(self.detach_fn, inputs if self.layer_save_input else output)

    def _register_hook(self) -> None:
        if self.layer is None:
            assert hasattr(self.vit, self.layer_name), \
                'layer whose output to take as embedding not found in vision transformer'
            layer = getattr(self.vit, self.layer_name)
        else:
            layer = self.layer
        self.hooks.append(layer.register_forward_hook(self._hook))
        self.hook_registered = True

    def eject(self):
        self.ejected = True
        for hook in self.hooks:
            hook.remove()
        self.hooks.clear()
        return self.vit

    def clear(self) -> None:
        self.latents = None

    def forward(self, img, return_embeddings_only=False):
        assert not self.ejected, 'extractor has been ejected, cannot be used anymore'
        self.clear()
        if not self.hook_registered:
            self._register_hook()
        pred = self.vit(img)
        target = self.device if self.device is not None else img.device
        latents = _map(lambda t: t.to(target), self.latents)
        if return_embeddings_only or self.return_embeddings_only:
            return latents
        return pred, latents
