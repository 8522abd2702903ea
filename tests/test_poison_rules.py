"""CPU: the poisoned-allocation helper of tests/poison_support.py catches what it is there to catch.

The fill reaches every byte of a new tensor's storage (dense, channels-last, zero-size, every dtype the library
allocates), ``torch.empty`` is itself again after the context, and ``same_under_poison`` fails a planted "kernel" that
reads one element it never wrote, even one that multiplies that element by zero, while passing a correct one."""
import pytest
import torch

from poison_support import PATTERNS, _EMPTY, _EMPTY_LIKE, fill_storage, poisoned, same_under_poison

DTYPES = (torch.float32, torch.bfloat16, torch.float16, torch.int32, torch.int64, torch.uint8)


def _storage_bytes(t):
    return torch.tensor([], dtype=torch.uint8).set_(t.untyped_storage())


@pytest.mark.parametrize("byte", PATTERNS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_fill_covers_every_byte(byte, dtype):
    with poisoned(byte):
        dense = torch.empty((3, 5, 7, 2), dtype=dtype)
        cl = torch.empty((2, 3, 5, 7), dtype=dtype, memory_format=torch.channels_last)
        like = torch.empty_like(cl)
        flat = torch.empty(13, dtype=dtype)
        zero = torch.empty((0, 4), dtype=dtype)
        zero_like = torch.empty_like(zero)
    assert not cl.is_contiguous() and like.stride() == cl.stride()
    for t in (dense, cl, like, flat):
        raw = _storage_bytes(t)
        assert raw.numel() == t.numel() * t.element_size()
        assert bool((raw == byte).all())
    assert zero.numel() == 0 and zero_like.numel() == 0


def test_patterns_are_the_documented_values():
    """0xFF is NaN in each float type and -1 in int32; 0x7F is 3.39e38 in fp32 and bf16, NaN in fp16."""
    with poisoned(0xFF):
        ff = {d: torch.empty(4, dtype=d) for d in (torch.float32, torch.bfloat16, torch.float16, torch.int32)}
    with poisoned(0x7F):
        sf = {d: torch.empty(4, dtype=d) for d in (torch.float32, torch.bfloat16, torch.float16, torch.int32)}
    for d in (torch.float32, torch.bfloat16, torch.float16):
        assert bool(torch.isnan(ff[d]).all())
    assert bool((ff[torch.int32] == -1).all())
    assert float(sf[torch.float32][0]) == pytest.approx(3.3961e38, rel=1e-4)
    assert float(sf[torch.bfloat16][0].float()) == pytest.approx(3.39e38, rel=1e-2)
    assert bool(torch.isnan(sf[torch.float16]).all())
    assert int(sf[torch.int32][0]) == 0x7F7F7F7F


def test_context_restores_torch_empty():
    with poisoned(0xFF):
        assert torch.empty is not _EMPTY and torch.empty_like is not _EMPTY_LIKE
    assert torch.empty is _EMPTY and torch.empty_like is _EMPTY_LIKE
    with pytest.raises(RuntimeError):
        with poisoned(0x7F):
            raise RuntimeError("inside")
    assert torch.empty is _EMPTY and torch.empty_like is _EMPTY_LIKE


def test_fill_storage_of_a_view_fills_its_base():
    base = _EMPTY(10, dtype=torch.float32)
    fill_storage(base[2:4], 0x00)
    assert bool((base == 0).all())


# ---- planted kernels: each takes its workspace and output from torch.empty, as ops.py does ----------------------------
def _correct(x):
    ws = torch.empty(x.numel() + 8)
    ws[: x.numel()] = x.reshape(-1) * 2
    out = torch.empty_like(x)
    out.copy_(ws[: x.numel()].reshape(x.shape))
    return out


def _reads_one_stale(x):
    """Stages n elements into a workspace of n + 8 and sums n + 1 of them: the last one was never written."""
    ws = torch.empty(x.numel() + 8)
    ws[: x.numel()] = x.reshape(-1)
    out = torch.empty(1)
    out[0] = ws[: x.numel() + 1].sum()
    return out


def _multiplies_stale_by_zero(x):
    """Reads an unwritten workspace row only to multiply it by a structural zero: right on zeroed memory, NaN on 0xFF."""
    ws = torch.empty((2, x.numel()))
    ws[0] = x.reshape(-1)
    taps = torch.tensor([1.0, 0.0])
    return taps @ ws


def _leaves_one_output_unwritten(x):
    out = torch.empty_like(x)
    out.reshape(-1)[1:] = x.reshape(-1)[1:]
    return out


def _int_counter_not_cleared(x):
    """An int32 count accumulated into a workspace nobody cleared."""
    cnt = torch.empty(1, dtype=torch.int32)
    cnt += int((x > 0).sum())
    return cnt


@pytest.mark.parametrize("bug", [_reads_one_stale, _multiplies_stale_by_zero, _leaves_one_output_unwritten, _int_counter_not_cleared])
def test_planted_bugs_fail_the_comparison(bug):
    x = torch.randn(3, 5, generator=torch.Generator().manual_seed(0))
    with pytest.raises(AssertionError, match="differs in"):
        same_under_poison(bug, x, case=bug.__name__)


def test_multiply_by_zero_is_right_on_clean_memory():
    """The zero-multiply bug is invisible on zeroed memory: the reason the helper runs more than one pattern."""
    x = torch.randn(3, 5, generator=torch.Generator().manual_seed(1))
    with poisoned(0x00):
        assert torch.equal(_multiplies_stale_by_zero(x), x.reshape(-1))
    with poisoned(0xFF):
        assert bool(torch.isnan(_multiplies_stale_by_zero(x)).all())


def test_correct_kernel_passes():
    x = torch.randn(4, 3, generator=torch.Generator().manual_seed(2))
    out = same_under_poison(_correct, x, case="correct")
    assert torch.equal(out[0], x * 2)


def test_mask_excuses_only_the_documented_entries():
    x = torch.randn(6, generator=torch.Generator().manual_seed(3))
    first = torch.zeros(6, dtype=torch.bool)
    first[0] = True
    same_under_poison(_leaves_one_output_unwritten, x, masks={0: first}, case="masked")
    second = torch.zeros(6, dtype=torch.bool)
    second[1] = True
    with pytest.raises(AssertionError, match="differs in 1 elements"):
        same_under_poison(_leaves_one_output_unwritten, x, masks={0: second}, case="wrong mask")


def test_nan_results_compare_by_bits():
    """A result that is NaN under every pattern (the same NaN) passes; NaN payloads and -0.0 are told apart."""
    x = torch.tensor([float("nan"), 1.0])
    same_under_poison(lambda v: v * 1.0, x)
    flip = iter([0.0, -0.0, -0.0])
    with pytest.raises(AssertionError):
        same_under_poison(lambda v: torch.full_like(v, next(flip)), torch.ones(2))
