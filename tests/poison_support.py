"""Poisoned allocations: every ``torch.empty`` / ``torch.empty_like`` filled with one byte pattern.  TEST INFRASTRUCTURE ONLY.

The library takes its outputs and workspaces from ``torch.empty``, so they hold whatever the caching allocator's block
held last.  A kernel that reads a byte nobody wrote can still give the right answer on the memory the suite happens to
get (0 x finite garbage = 0), and the wrong one once the block held a NaN.  ``same_under_poison`` runs a call with every
new tensor's storage filled with each of ``PATTERNS`` and asserts that the results do not depend on the pattern:

- ``0x00``: zeros everywhere (the friendliest garbage);
- ``0xFF``: NaN in fp32, bf16 and fp16, -1 in int32 (an index that points before its array);
- ``0x7F``: 3.39e38 in fp32 and bf16 (finite, but inf once doubled), NaN in fp16, 0x7F7F7F7F in int32.

The fill is a tensor op on the current stream, so an allocation made while a CUDA graph is being captured gets its fill
as a captured node and every replay poisons it again."""
import contextlib

import torch

PATTERNS = (0x00, 0xFF, 0x7F)

_EMPTY, _EMPTY_LIKE = torch.empty, torch.empty_like


def fill_storage(t: torch.Tensor, byte: int) -> torch.Tensor:
    """Every byte of ``t``'s storage set to ``byte``, whatever ``t``'s strides (channels-last, views, zero-size)."""
    st = t.untyped_storage()
    if st.nbytes():
        _EMPTY((0,), dtype=torch.uint8, device=t.device).set_(st).fill_(byte)
    return t


@contextlib.contextmanager
def poisoned(byte: int):
    """``torch.empty`` and ``torch.empty_like`` return tensors whose whole storage holds ``byte``; restored on exit."""

    def empty(*args, **kwargs):
        return fill_storage(_EMPTY(*args, **kwargs), byte)

    def empty_like(*args, **kwargs):
        return fill_storage(_EMPTY_LIKE(*args, **kwargs), byte)

    torch.empty, torch.empty_like = empty, empty_like
    try:
        yield
    finally:
        torch.empty, torch.empty_like = _EMPTY, _EMPTY_LIKE


def _tensors(out):
    """The tensors of a (nested) result, in order, each detached."""
    if isinstance(out, torch.Tensor):
        return [out.detach()]
    if isinstance(out, dict):
        return [t for k in sorted(out) for t in _tensors(out[k])]
    if isinstance(out, (tuple, list)):
        return [t for x in out for t in _tensors(x)]
    if hasattr(out, "_fields"):
        return _tensors(tuple(out))
    return []


def _bits(t: torch.Tensor) -> torch.Tensor:
    """The bytes of ``t``'s elements (not its storage), comparable with ``torch.equal`` whatever the dtype, NaN included."""
    t = t.contiguous()
    return t.reshape(-1).view(torch.uint8) if t.numel() else t.reshape(-1).to(torch.uint8)


def same_under_poison(fn, *args, masks=None, patterns=PATTERNS, case=""):
    """Run ``fn(*args)`` under each byte pattern and assert every returned tensor is bit-identical across them.

    ``args`` are made by the caller, outside the poison.  ``masks``: {index of the output tensor, in the flattened order
    of ``_tensors``: bool mask of the entries the results may leave unspecified}; the test that passes one names the
    comment that documents those entries.  Returns the first pattern's outputs."""
    masks = masks or {}
    runs = []
    for byte in patterns:
        with poisoned(byte):
            out = fn(*args)
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        runs.append([t.clone() for t in _tensors(out)])
    first = runs[0]
    assert first, f"{case}: the call returned no tensor"
    for byte, run in zip(patterns[1:], runs[1:]):
        assert len(run) == len(first), case
        for i, (a, b) in enumerate(zip(first, run)):
            assert a.shape == b.shape and a.dtype == b.dtype, f"{case}: output {i} {tuple(a.shape)} vs {tuple(b.shape)}"
            if i in masks:
                keep = ~masks[i].to(a.device).expand(a.shape)
                a, b = a[keep], b[keep]
            ba, bb = _bits(a), _bits(b)
            if not torch.equal(ba, bb):
                n = int((ba.reshape(a.numel(), -1) != bb.reshape(b.numel(), -1)).any(1).sum())
                raise AssertionError(f"{case}: output {i} {tuple(a.shape)} {a.dtype} differs in {n} elements between fill "
                                     f"0x{patterns[0]:02X} and fill 0x{byte:02X}")
    return first
