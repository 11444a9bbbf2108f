"""Device results to the host: the one transfer format of the command modules."""
import torch


def to_host(*tensors):
    """The tensors as numpy arrays of their own dtypes and shapes, bit for bit.  All CUDA tensors of the call reach the
    host in one device-to-host copy of ``_pack``'s buffer, and their arrays are views of that one host buffer; CPU
    tensors are returned as ``numpy()`` views, without a trip to the device.  CUDA tensors on two devices, a dtype numpy
    cannot hold (bfloat16) and arguments that are not tensors raise ``ValueError``."""
    for t in tensors:
        if not torch.is_tensor(t):
            raise ValueError("to_host: tensors expected, got %s" % type(t).__name__)
        _numpy_dtype(t)
    cuda = [t for t in tensors if t.is_cuda]
    if len({t.device for t in cuda}) > 1:
        raise ValueError("to_host: the CUDA tensors of one call must live on one device")
    views = iter(_unpack(_pack(cuda).cpu().numpy(), cuda) if cuda else ())
    return tuple(next(views) if t.is_cuda else t.detach().numpy() for t in tensors)


def _numpy_dtype(t):
    try:
        return torch.empty(0, dtype=t.dtype).numpy().dtype
    except TypeError:
        raise ValueError("to_host: numpy has no dtype for %s" % t.dtype) from None


def _pack(tensors):
    """The tensors' bytes, in order, each padded to a multiple of 8 bytes so that every view ``_unpack`` takes is
    aligned (the padding bytes are never read), as one uint8 tensor on their device: one concatenation, none for one
    tensor."""
    parts = []
    for t in tensors:
        b = t.detach().contiguous().view(-1).view(torch.uint8)
        parts += [b, b.new_empty(-b.numel() % 8)]
    return torch.cat(parts) if len(tensors) > 1 else parts[0]


def _unpack(host, tensors):
    """The tensors' arrays as views of ``_pack``'s buffer on the host (a uint8 ndarray)."""
    out, o = [], 0
    for t in tensors:
        n = t.numel() * t.element_size()
        out.append(host[o:o + n].view(_numpy_dtype(t)).reshape(t.shape))
        o += n + (-n % 8)
    return out
