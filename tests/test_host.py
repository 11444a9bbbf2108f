"""``_host.to_host``, the transfer format of the command modules: its packing of CUDA tensors (``_pack`` / ``_unpack``)
run on CPU tensors, and its CPU path.  ``tests/test_gpu_host.py`` repeats the round trip on CUDA tensors and counts the
calls of each command."""
import numpy as np
import pytest
import torch

from transformer_explainability_b200 import _host

DTYPES = [torch.bool, torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float16, torch.float32,
          torch.float64, torch.complex64, torch.complex128]


def sample(dtype, shape, seed):
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.bool:
        return torch.rand(shape, generator=g) < 0.5
    if dtype.is_complex:
        return torch.randn(shape, dtype=dtype, generator=g)
    if dtype.is_floating_point:
        t = torch.randn(shape, generator=g).to(dtype)
        if t.numel() >= 3:                                        # NaN, -0 and inf travel as bits
            t.view(-1)[:3] = torch.tensor([float("nan"), -0.0, float("inf")], dtype=dtype)
        return t
    info = torch.iinfo(dtype)
    return torch.randint(info.min, info.max, shape, dtype=dtype, generator=g)


def packed(*tensors):
    """``to_host``'s packing of CUDA tensors, run on CPU tensors."""
    return _host._unpack(_host._pack(tensors).numpy(), tensors)


def check(arrays, tensors):
    assert len(arrays) == len(tensors)
    for a, t in zip(arrays, tensors):
        want = t.numpy()
        assert a.dtype == want.dtype and a.shape == want.shape
        assert a.tobytes() == np.ascontiguousarray(want).tobytes()
        assert a.ctypes.data % a.dtype.alignment == 0


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_round_trip_every_dtype(dtype):
    tensors = [sample(dtype, (3, 5), 1), sample(dtype, (), 2), sample(dtype, (0, 4), 3), sample(dtype, (7,), 4)]
    check(_host.to_host(*tensors), tensors)
    check(packed(*tensors), tensors)


def test_mixed_dtypes_odd_byte_counts_and_non_contiguous():
    t = [sample(torch.bool, (3,), 1), sample(torch.float64, (2, 3), 2), sample(torch.uint8, (5,), 3),
         sample(torch.float16, (3,), 4), sample(torch.int64, (4, 6), 5)[:, ::2], sample(torch.float64, (), 6),
         sample(torch.int32, (3, 4), 7).t(), sample(torch.float32, (0,), 8), sample(torch.float64, (3,), 9)]
    assert not t[4].is_contiguous() and not t[6].is_contiguous()
    check(packed(*t), t)
    check(_host.to_host(*t), t)


def test_cpu_tensors_are_returned_as_views():
    t = torch.arange(6, dtype=torch.int32).reshape(2, 3)
    a, = _host.to_host(t)
    assert np.shares_memory(a, t.numpy())
    assert _host.to_host() == ()


def test_rejects_what_numpy_cannot_hold():
    with pytest.raises(ValueError, match="bfloat16"):
        _host.to_host(torch.zeros(2), torch.zeros(3, dtype=torch.bfloat16))
    for bad in (np.zeros(2), [1, 2], 3.0, None):
        with pytest.raises(ValueError, match="tensors expected"):
            _host.to_host(torch.zeros(2), bad)
