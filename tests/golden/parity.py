"""The reference-parity recipe every drop-in family shares.  A family's `<name>_spec.py` holds its case table and one
`Family` record; make_family_golden.py runs the UNMODIFIED reference (vit_pytorch) on the cases and writes
tests/golden/<name>.pt, and the tests rebuild the same weights and inputs from the seeds for the drop-in
(vit_pytorch_b200).  The weights are not stored: the drop-in's constructor consumes the RNG exactly like the
reference's (the seeded-init digests check it), and every case keeps a digest of its rebuilt weights and input, so a
drift in the recipe fails loudly instead of comparing different models.

The recipe of a case: seed torch with its seed and build the model; from a generator seeded with 1000 + seed, add
0.1 N(0, 1) to every 1-D `weight` and 0.05 N(0, 1) to every 1-D `bias` (LayerNorm affines and biases, so they are
exercised), the family's `extra` rule to any other parameter, then run its `after` rule; round every parameter to a
bf16-representable value, so a bf16 copy of the model holds the same numbers.  The input is N(0, 1) from a generator
seeded with 100 + seed, rounded to bf16."""
from __future__ import annotations

import hashlib
import importlib
import inspect
import os
import random
import sys
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import torch

TESTS = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)
from conftest import signature as class_signature, state_digest  # noqa: E402,F401  (tests/conftest.py)

REFERENCE, DROPIN = "vit_pytorch", "vit_pytorch_b200"
FAMILY_NAMES = ("pit", "cct", "cait", "deepvit", "xcit", "cross_vit", "vivit", "vit_nd", "vit_small")


def families() -> Dict[str, "Family"]:
    """Every family's record, from tests/golden/<name>_spec.py."""
    return {n: importlib.import_module(f"{n}_spec").FAMILY for n in FAMILY_NAMES}


def load(package: str, path: str):
    """`module.attr` of the reference (`vit_pytorch`) or the drop-in (`vit_pytorch_b200`) package."""
    module, attr = path.rsplit(".", 1)
    return getattr(importlib.import_module(f"{package}.{module}"), attr)


def signature(fn) -> list:
    """(name, repr(default)) of every parameter: of cls.__init__ for a class, of the function itself otherwise."""
    if inspect.isclass(fn):
        return class_signature(fn)
    return [(k, repr(v.default)) for k, v in inspect.signature(fn).parameters.items()]


def seeded_model(make, kwargs: dict, seed: int, *, extra=None, after=None):
    """`make(**kwargs)` built and perturbed by the shared recipe (module docstring).  `extra(name, p, g)` perturbs a
    parameter the 1-D weight / bias rules skip and `after(model, g)` runs before the rounding, both drawing from the
    same generator, in this order."""
    torch.manual_seed(seed)
    model = make(**kwargs).eval()
    g = torch.Generator().manual_seed(1000 + seed)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1 and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1 and n.endswith("bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
            elif extra is not None:
                extra(n, p, g)
        if after is not None:
            after(model, g)
        for p in model.parameters():
            p.copy_(p.bfloat16().float())
    return model


def seeded_input(seed: int, shape: tuple) -> torch.Tensor:
    g = torch.Generator().manual_seed(100 + seed)
    return torch.randn(*shape, generator=g).bfloat16()


def round_buffers(model) -> None:
    """Round every floating-point buffer to a bf16-representable value, as the parameters are."""
    for b in model.buffers():
        if b.is_floating_point():
            b.copy_(b.bfloat16().float())


def seed_layer_dropout(spec: dict) -> None:
    """Seed the generators layer dropout draws from (torch's CPU generator, and `random` when every layer would be
    dropped) right before a forward, so that every run of the case keeps the same layers."""
    if "drop_seed" in spec:
        torch.manual_seed(spec["drop_seed"])
        random.seed(spec["drop_seed"])


def weights_digest(model) -> str:
    """One sha256 over every state_dict entry (name, shape, dtype, bytes) in registration order."""
    h = hashlib.sha256()
    for k, v in model.state_dict().items():
        h.update(f"{k}{tuple(v.shape)}{v.dtype}".encode())
        h.update(v.detach().float().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def input_digest(x: torch.Tensor) -> str:
    return hashlib.sha256(x.float().contiguous().numpy().tobytes()).hexdigest()


@dataclass(frozen=True)
class Family:
    """One drop-in family's parity cases and the rules only it has.

    `model` is the `module.Class` of the model under both packages.  `make(package, spec)`, when given, picks the
    class or factory a case constructs instead (a seeded-init variant passes spec = {"kind": variant}).  `init` maps
    each seeded-init variant to its constructor keywords; a family with one variant (key None) stores its digest
    unnamed.  `signatures(package)`, when given, returns the stored signature fields instead of
    {"signature": signature(model)}.  `forwards(spec)` lists the forwards a case stores logits for, as (key in
    logits_fp32, None for the only one; keyword arguments).  `stored(model, spec)` adds fields stored before the
    logits and `embed(model, x, spec)` fields stored after them.  `before_forward(spec)` runs right before every
    forward."""
    name: str                                             # tests/golden/<name>.pt
    model: str
    cases: Dict[str, dict]
    case_kwargs: Callable[[dict], dict]
    input_shape: Callable[[dict], tuple]                  # of a case's input, batch first
    init_seed: int
    init: Dict[Optional[str], dict]
    make: Optional[Callable[[str, dict], Callable]] = None
    signatures: Optional[Callable[[str], dict]] = None
    extra: Optional[Callable] = None                      # extra(name, p, g, spec), see seeded_model
    after: Optional[Callable] = None                      # after(model, g, spec), see seeded_model
    before_forward: Optional[Callable[[dict], None]] = None
    forwards: Callable[[dict], List[Tuple[Optional[str], dict]]] = lambda spec: [(None, {})]
    stored: Optional[Callable] = None                     # stored(model, spec) -> dict
    embed: Optional[Callable] = None                      # embed(model, x, spec) -> dict

    def constructor(self, package: str, spec: dict):
        return self.make(package, spec) if self.make is not None else load(package, self.model)

    def build(self, spec: dict, package: str = DROPIN):
        """The fp32 model of a case, bf16-representable."""
        extra = None if self.extra is None else (lambda n, p, g: self.extra(n, p, g, spec))
        after = None if self.after is None else (lambda m, g: self.after(m, g, spec))
        return seeded_model(self.constructor(package, spec), self.case_kwargs(spec), spec["seed"], extra=extra,
                            after=after)

    def input(self, spec: dict) -> torch.Tensor:
        """The bf16 input of a case."""
        return seeded_input(spec["seed"], self.input_shape(spec))

    def signature_fields(self, package: str) -> dict:
        if self.signatures is not None:
            return self.signatures(package)
        return {"signature": signature(load(package, self.model))}

    def init_state(self, package: str, variant: Optional[str]) -> dict:
        """state_dict of the unperturbed model the seeded-init variant builds."""
        make = self.constructor(package, {"kind": variant})
        torch.manual_seed(self.init_seed)
        return make(**self.init[variant]).state_dict()

    def outputs(self, model, x: torch.Tensor, spec: dict) -> dict:
        """What the fixture stores for a case after the spec and digests; run under inference mode."""
        out = {} if self.stored is None else self.stored(model, spec)
        logits = {}
        for key, kwargs in self.forwards(spec):
            if self.before_forward is not None:
                self.before_forward(spec)
            logits[key] = model(x.float(), **kwargs).clone()
        out["logits_fp32"] = logits[None] if list(logits) == [None] else logits
        if self.embed is not None:
            out.update(self.embed(model, x, spec))
        return out
