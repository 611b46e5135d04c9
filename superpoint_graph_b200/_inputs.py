"""How the partition pipelines' device stages take their array arguments (DESIGN.md §4).

Every argument is a numpy array or a tensor.  The stage runs on the device of its first CUDA tensor argument, else on
the current device.  A wrong dtype is refused with TypeError, never rounded; CPU tensors and numpy arrays are copied to
the device (spg_delaunay alone refuses a CPU tensor).  The checks are apart from the upload because most stages check
every argument before they pick a device, and that order decides which error an input with several faults raises.
"""
import numpy as np
import torch

MAX_POINTS = 2 ** 31 - 1


def device_of(*xs):
    """The device of the first CUDA tensor among xs, else the current device."""
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    return torch.device("cuda", torch.cuda.current_device())


def n_points(shape):
    """The point count of a cloud of this shape; ValueError unless it is [n, 3] with n < 2^31 - 1."""
    if len(shape) != 2 or shape[1] != 3:
        raise ValueError("xyz must be [n, 3] (got shape %s)" % (tuple(shape),))
    if shape[0] >= MAX_POINTS:
        raise ValueError("%d points; clouds of 2^31 - 1 points or more are not supported" % shape[0])
    return int(shape[0])


def check_dtype(a, name, dtype):
    """The shape of a, whose dtype must be the one named `dtype` ("float32", "uint8"), numpy's or torch's."""
    if torch.is_tensor(a):
        if a.dtype != getattr(torch, dtype):
            raise TypeError("%s must be %s (got %s)" % (name, dtype, a.dtype))
        return tuple(a.shape)
    a = np.asarray(a)
    if a.dtype != dtype:
        raise TypeError("%s must be %s (got %s)" % (name, dtype, a.dtype))
    return a.shape


def check_ints(a, name):
    """The shape of a, which must hold integers (bool, floating and complex dtypes are refused)."""
    if torch.is_tensor(a):
        if a.dtype.is_floating_point or a.dtype.is_complex or a.dtype == torch.bool:
            raise TypeError("%s must hold integers (got %s)" % (name, a.dtype))
        return tuple(a.shape)
    a = np.asarray(a)
    if a.dtype.kind not in "iu":
        raise TypeError("%s must hold integers (got %s)" % (name, a.dtype))
    return a.shape


def on_device(a, dev, int64=False):
    """a as a contiguous tensor on dev, copied there at most once.  int64=True widens checked integer ids to int64;
    nothing else is cast."""
    if torch.is_tensor(a):
        return a.to(device=dev, dtype=torch.int64 if int64 else None).contiguous()
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64 if int64 else None)).to(dev)


def simplices_on(s, dev):
    """A triangulation's simplices, integers [T, 4], on dev: int32 stays int32 (what spg_delaunay gives), other
    integer types become int64."""
    shape = tuple(s.shape)
    if len(shape) != 2 or shape[1] != 4:
        raise ValueError("simplices must be [T, 4] (got shape %s)" % (shape,))
    check_ints(s, "simplices")
    return on_device(s, dev, int64=s.dtype not in (torch.int32, np.int32))
