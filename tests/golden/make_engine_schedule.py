"""Generate tests/golden/engine_schedule.json: the launch sequence TransformerEngine.run_blocks issues, per model family,
LayerNorm mode and host loop, recorded on CPU without a GPU:

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_engine_schedule.py

Every _lib entry point run_blocks can reach is replaced by a recorder and torch.cuda.current_stream is stubbed, so the
engine runs on CPU tensors and nothing computes.  A call is stored with its arguments bound against the real function's
signature (defaults applied).  A tensor is stored by its role when its storage is one the caller owns (`x`, a workspace
buffer `ws.<name>`, the rope table, the key mask, the varlen arrays) with its byte offset, shape and stride; any other
tensor (a prepared weight) by its key in TransformerEngine.prepared(), dtype, shape, stride and a digest of its bytes.
encoder_blocks' ctypes layer array is expanded field by field.

The weights are multiples of 1/64 in [-1, 1] and the temperatures 0 or -ln 2, so every prepared weight is computed
exactly (or rounded once, deterministically) on any CPU and the digests do not depend on the host.
"""
from __future__ import annotations

import contextlib
import ctypes
import hashlib
import inspect
import json
import math
import os
import sys
import types
from typing import Callable, Dict, List, NamedTuple, Optional

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from vit_pytorch_b200 import _lib  # noqa: E402

FIXTURE = os.path.join(HERE, "engine_schedule.json")

# every _lib entry point TransformerEngine.run_blocks can reach
ENTRY_POINTS = ("gemm", "gemm_headnorm", "layernorm", "rowstats_cast", "rope_qk", "attention", "attention_varlen",
                "attention_axial", "attention_headmix", "attention_xca", "local_patch_interaction", "encoder_blocks",
                "cast_f32_bf16")

D, HEADS, DH, MLP = 64, 2, 32, 128


def quantize_(module: torch.nn.Module, seed: int) -> None:
    """Weights k/64 (|k| <= 64), BatchNorm running variances in [1/4, 2], temperatures alternately 0 and -ln 2."""
    g = torch.Generator().manual_seed(seed)
    temps = 0
    with torch.no_grad():
        for name, p in list(module.named_parameters()) + list(module.named_buffers()):
            if not p.is_floating_point():
                continue
            if name.endswith("temperature"):
                p.fill_(-math.log(2.0) if temps % 2 else 0.0)
                temps += 1
            elif name.endswith("running_var"):
                p.copy_(torch.randint(16, 129, p.shape, generator=g).float() / 64)
            elif isinstance(p, torch.nn.Parameter) or name.endswith("running_mean"):
                p.copy_(torch.randint(-64, 65, p.shape, generator=g).float() / 64)


def varlen_index() -> _lib.VarlenIndex:
    """A packed batch of three images of 12, 4 and 5 patches (patch size 4)."""
    images = [torch.empty(3, 16, 12), torch.empty(3, 8, 8), torch.empty(3, 4, 20)]
    return _lib.VarlenIndex(images, 4, torch.device("cpu"))


class Case(NamedTuple):
    name: str
    module: Callable[[], torch.nn.Module]
    rows: int                                     # rows of x
    kwargs: Callable[[], dict]                    # run_blocks' keyword arguments besides x
    c_loop: bool                                  # the one-call C loop applies in fold mode


def _vit(heads=HEADS, dh=DH):
    from vit_pytorch_b200.vit import Transformer
    return Transformer(D, 2, heads, dh, MLP)


def _qk_norm():
    from vit_pytorch_b200.simple_vit_with_qk_norm import Transformer
    return Transformer(D, 2, HEADS, DH, MLP)


def _navit_nested():
    from vit_pytorch_b200.na_vit_nested_tensor import Transformer
    return Transformer(D, 2, HEADS, DH, MLP)


def _navit():
    from vit_pytorch_b200.na_vit import Transformer
    return Transformer(D, 2, HEADS, DH, MLP)


def _rotary():
    from vit_pytorch_b200.vit_nd_rotary import Transformer
    return Transformer(D, 2, HEADS, DH, MLP)


def _small():
    from vit_pytorch_b200.vit_for_small_dataset import Transformer
    return Transformer(D, 2, HEADS, DH, MLP)


def _factorized():
    from vit_pytorch_b200.vivit import FactorizedTransformer
    return FactorizedTransformer(D, 2, HEADS, DH, MLP)


def _temporal():
    from vit_pytorch_b200.vivit import Transformer
    return Transformer(D, 2, HEADS, DH, MLP)


def _deepvit():
    from vit_pytorch_b200.deepvit import Transformer
    return Transformer(D, 2, 4, DH, MLP)


def _cait():
    from vit_pytorch_b200.cait import Transformer
    return Transformer(D, 3, 4, DH, MLP)


def _xcit():
    from vit_pytorch_b200.xcit import XCATransformer
    return XCATransformer(D, 3, HEADS, DH, MLP, local_patch_kernel_size=3)


def _mask(rows: List[List[int]]) -> torch.Tensor:
    return torch.tensor(rows, dtype=torch.uint8)


def _rope(rows: int) -> tuple:
    return torch.zeros(rows, HEADS, DH // 2, 2), rows


# ViViT factorized self-attention: b = 2 videos of f = 3 frames of N = 5 tokens; the factorized encoder's temporal
# transformer: b = 2 sequences of Lt = 4 (cls + 3 frames)
CASES = [
    Case("vit cls", _vit, 2 * 17, lambda: dict(B=2, N=17), True),
    Case("vit cls primed", _vit, 2 * 17, lambda: dict(B=2, N=17, primed=True), True),
    Case("vit identity out", lambda: _vit(heads=1, dh=D), 2 * 17, lambda: dict(B=2, N=17, primed=True), True),
    Case("vit long", _vit, 2 * 520, lambda: dict(B=2, N=520), True),
    Case("simple_vit qk rmsnorm", _qk_norm, 2 * 16, lambda: dict(B=2, N=16, primed=True), True),
    Case("navit nested varlen", _navit_nested, 21, lambda: dict(primed=True, varlen=varlen_index()), False),
    Case("navit varlen", _navit, 21, lambda: dict(primed=True, varlen=varlen_index()), False),
    Case("vit_nd rotary", _rotary, 2 * 12, lambda: dict(B=2, N=12, primed=True, rope=_rope(12)), True),
    Case("vit small dataset", _small, 2 * 17, lambda: dict(B=2, N=17, primed=True), True),
    Case("vivit factorized self-attention", _factorized, 30, lambda: dict(B=6, N=5, primed=True,
                                                                          axial=(5, 3, None, True)), False),
    Case("vivit factorized self-attention masked", _factorized, 30,
         lambda: dict(B=6, N=5, primed=True, axial=(5, 3, _mask([[1, 0, 1], [1, 1, 0]]), False)), False),
    Case("vivit temporal", _temporal, 8, lambda: dict(B=2, N=4), True),
    Case("vivit temporal masked zero rows", _temporal, 8,
         lambda: dict(B=2, N=4, axial=(1, 4, _mask([[1, 1, 0, 1], [1, 0, 0, 0]]), True)), False),
    Case("vivit temporal masked", _temporal, 8,
         lambda: dict(B=2, N=4, axial=(1, 4, _mask([[1, 1, 0, 1], [1, 0, 0, 0]]), False)), False),
    Case("deepvit", _deepvit, 2 * 17, lambda: dict(B=2, N=17, primed=True), False),
    Case("cait layer subset", _cait, 2 * 16, lambda: dict(B=2, N=16, primed=True, layers=[0, 2]), False),
    Case("xcit layer subset", _xcit, 2 * 12, lambda: dict(B=2, N=12, primed=True, layers=[0, 2], grid=(3, 4)), False),
]


def runs(case: Case) -> List[tuple]:
    """(LayerNorm mode, host loop) pairs the case is recorded in."""
    return [("fold", "c")] * case.c_loop + [("fold", "python"), ("exact", "python")]


def build(case: Case, seed: int = 0):
    torch.manual_seed(seed)
    mod = case.module().eval()
    quantize_(mod, seed)
    return mod


# ------------------------------------------------------------------------------------------------------ recording
def _digest(t: torch.Tensor) -> str:
    return hashlib.sha256(t.detach().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()[:12]


class Recorder:
    """Encodes the arguments of the engine's library calls; `owners()` lists (role, tensor) of the caller's buffers."""

    def __init__(self, eng, owners: Callable[[], List[tuple]]) -> None:
        self.eng, self.owners, self.calls = eng, owners, []

    def weight_key(self, ptr: int, t: Optional[torch.Tensor] = None) -> Optional[str]:
        for k, v in self.eng.prepared().items():
            if isinstance(v, torch.Tensor) and v.data_ptr() == ptr and (
                    t is None or (v.shape == t.shape and v.stride() == t.stride())):
                return k
        return None

    def tensor(self, t: torch.Tensor) -> dict:
        base = t.untyped_storage().data_ptr()
        for role, o in self.owners():
            if isinstance(o, torch.Tensor) and o.untyped_storage().data_ptr() == base:
                return {"role": role, "offset": t.data_ptr() - base, "shape": list(t.shape), "stride": list(t.stride())}
        return {"key": self.weight_key(t.data_ptr(), t), "dtype": str(t.dtype).replace("torch.", ""),
                "shape": list(t.shape), "stride": list(t.stride()), "sha": _digest(t)}

    def pointer(self, ptr: Optional[int]):
        """A device pointer inside a ctypes struct: the workspace buffer or prepared weight it addresses."""
        if ptr is None:
            return None
        for role, o in self.owners():
            if isinstance(o, torch.Tensor) and o.data_ptr() == ptr:
                return role
        k = self.weight_key(ptr)
        return None if k is None else {"key": k, "sha": _digest(self.eng.prepared()[k])}

    def value(self, v):
        if v is None or isinstance(v, (bool, int, float, str)):
            return v
        if isinstance(v, torch.Tensor):
            return self.tensor(v)
        if isinstance(v, (tuple, list)):
            return [self.value(e) for e in v]
        if isinstance(v, ctypes.Array):
            return [self.value(e) for e in v]
        if isinstance(v, ctypes.Structure):
            return {f: (self.pointer(getattr(v, f)) if ty is ctypes.c_void_p else getattr(v, f))
                    for f, ty in v._fields_}
        raise TypeError(f"cannot record {type(v)}")

    @staticmethod
    def bind(sig: inspect.Signature, args: tuple, kwargs: dict) -> dict:
        """A call's arguments by parameter name, bound against the real function's signature, defaults applied."""
        bound = sig.bind(*args, **kwargs)
        bound.apply_defaults()
        return dict(bound.arguments)

    def recorder(self, name: str, real: Callable) -> Callable:
        sig = inspect.signature(real)

        def record(*args, **kwargs):
            self.calls.append({"call": name, **{k: self.value(v) for k, v in self.bind(sig, args, kwargs).items()}})
        return record


@contextlib.contextmanager
def recording(eng, owners: Callable[[], List[tuple]], ln_mode: str, host_loop: str, extra_entry_points=(),
              recorder=Recorder):
    """Within: ENTRY_POINTS and `extra_entry_points` of _lib record into the yielded `recorder(eng, owners)`'s
    `calls`, torch.cuda.current_stream is stubbed and B200VIT_LN_MODE / B200VIT_HOST_LOOP are set."""
    rec = recorder(eng, owners)
    saved = {n: getattr(_lib, n) for n in ENTRY_POINTS + tuple(extra_entry_points)}
    saved_stream = torch.cuda.current_stream
    saved_env = {k: os.environ.get(k) for k in ("B200VIT_LN_MODE", "B200VIT_HOST_LOOP")}
    try:
        for n, f in saved.items():
            setattr(_lib, n, rec.recorder(n, f))
        torch.cuda.current_stream = lambda device=None: types.SimpleNamespace(cuda_stream=0)
        os.environ["B200VIT_LN_MODE"], os.environ["B200VIT_HOST_LOOP"] = ln_mode, host_loop
        yield rec
    finally:
        for n, f in saved.items():
            setattr(_lib, n, f)
        torch.cuda.current_stream = saved_stream
        for k, v in saved_env.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def caller_buffers(eng, x: torch.Tensor, kw: dict) -> Callable[[], List[tuple]]:
    """(role, tensor) of every buffer the caller of run_blocks owns, read when a call is recorded."""
    def owners():
        out = [("x", x)] + [(f"ws.{k}", v) for k, v in eng.slot.t.items()]
        if kw.get("rope") is not None:
            out.append(("rope", kw["rope"][0]))
        if kw.get("axial") is not None and kw["axial"][2] is not None:
            out.append(("key_mask", kw["axial"][2]))
        if kw.get("varlen") is not None:
            out.append(("varlen", kw["varlen"].cu))
        if eng._vl is not None:
            out += [("varlen.cu", eng._vl[0]), ("varlen.tile_prefix", eng._vl[1])]
        return out
    return owners


def record(case: Case, ln_mode: str, host_loop: str) -> List[dict]:
    mod = build(case)
    eng = mod.engine()
    x = torch.zeros(case.rows, D)
    kw = case.kwargs()
    with recording(eng, caller_buffers(eng, x, kw), ln_mode, host_loop) as rec:
        eng.run_blocks(x, **kw)
    return rec.calls


def run_name(case: Case, ln_mode: str, host_loop: str) -> str:
    return f"{case.name} | {ln_mode} | {host_loop}"


def generate(cases=CASES) -> Dict[str, List[dict]]:
    return {run_name(c, m, h): record(c, m, h) for c in cases for m, h in runs(c)}


def dumps(schedule: Dict[str, List[dict]]) -> str:
    """JSON with one line per call."""
    out = ["{"]
    for i, (name, calls) in enumerate(schedule.items()):
        out.append(f"{json.dumps(name)}: [")
        out += ["  " + json.dumps(c) + ("," if j + 1 < len(calls) else "") for j, c in enumerate(calls)]
        out.append("]" + ("," if i + 1 < len(schedule) else ""))
    out.append("}")
    return "\n".join(out) + "\n"


if __name__ == "__main__":
    if not _lib.LIB_PATH.exists():
        from vit_pytorch_b200 import build as _build
        _build.build()
    text = dumps(generate())
    with open(FIXTURE, "w") as f:
        f.write(text)
    print(f"wrote {FIXTURE} ({len(text)} bytes)")
