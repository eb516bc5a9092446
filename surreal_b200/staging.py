"""Pinned host staging for the host <-> device copies of the plugin API (numpy observations and actions of the agents, the
exp-sender wrappers' host rows, numpy batches of the learners, host inserts and sampled indices of the replays).

Each owner keeps one ``Staging``; its buffers are named by the owner, allocated (zeroed) on first use and reused by name,
and replaced only when the requested shape or dtype changes, so repeated calls allocate nothing.  A numpy array that is
already pinned, C-contiguous, writeable and of the requested dtype is the DMA source itself; anything else is copied
into the named pinned buffer first.  Such an array is read by the copy after the call returns, like the pinned buffers.

The pool adds no synchronisation.  A named pinned buffer is rewritten only after a host synchronisation that follows its
last copy, and each owner relies on one it already has:
  * agents (observations in, actions / pd / cells out) and exp-sender wrappers (host rows of a step): the act entry's
    D2H of the actions, which ends in a stream synchronisation, comes between two uses;
  * learners (numpy batches): the read-back of the statistics at the end of every learn();
  * FIFOReplay.insert: the host read of the slot ``sb200_fifo_push`` assigned;
  * UniformReplay.insert: its copy of the record is synchronous; UniformReplay.sample: the event recorded after the
    H2D of the indices, which sample_indices waits on before it draws into the buffer again.
Device buffers (``device``) are the fixed landing places of staged copies; the stream orders their reuse."""
import ctypes as C
import math

import numpy as np
import torch

# the dtypes staged: float32 rows, float64 rewards (SSAR n-step sums), uint8 frames, int64 actions / replay indices
_PAIRS = ((np.float32, torch.float32), (np.float64, torch.float64), (np.uint8, torch.uint8), (np.int64, torch.int64))
_TORCH = {**{n: t for n, t in _PAIRS}, **{np.dtype(n): t for n, t in _PAIRS}}     # numpy type or dtype -> torch dtype
_NUMPY = {t: np.dtype(n) for n, t in _PAIRS}


def _direct(arr, dtype, shape):
    """``arr`` may be the DMA source itself: a pinned, C-contiguous, writeable numpy array of ``dtype`` holding
    prod(shape) elements (torch.from_numpy needs a writeable array)."""
    return (isinstance(arr, np.ndarray) and arr.dtype == dtype and arr.size == math.prod(shape)
            and arr.flags['C_CONTIGUOUS'] and arr.flags['WRITEABLE'] and torch.from_numpy(arr).is_pinned())


class Staging:
    def __init__(self, device):
        self._cuda = device
        self._pinned, self._device = {}, {}

    @staticmethod
    def _get(table, name, shape, dtype, alloc):
        """Buffer ``name`` of ``table``, keyed with its shape and torch dtype so that a repeated request is one lookup; a
        request with another shape or dtype replaces it."""
        key = (name, tuple(shape), _TORCH[dtype])
        buf = table.get(key)
        if buf is None:
            for k in [k for k in table if k[0] == name]:
                del table[k]
            buf = table[key] = alloc(*key[1:])
        return buf

    def pinned(self, name, shape, dtype=np.float32):
        """The pinned host tensor ``name`` [shape] of numpy ``dtype`` (D2H landing buffers, staged records)."""
        return self._get(self._pinned, name, shape, dtype, lambda s, t: torch.zeros(s, dtype=t, pin_memory=True))

    def device(self, name, shape, dtype=np.float32):
        """The device tensor ``name`` [shape] of numpy ``dtype``: where a staged copy lands."""
        return self._get(self._device, name, shape, dtype, lambda s, t: torch.zeros(s, dtype=t, device=self._cuda))

    def host_ptr(self, name, arr, shape, dtype=np.float32):
        """Host address (c_void_p) of ``arr`` as [shape] ``dtype``, for a C entry that issues its own H2D: ``arr``'s own
        when it can be the DMA source, else that of pinned buffer ``name`` holding ``np.asarray(arr, dtype)``."""
        dtype = np.dtype(dtype)
        if _direct(arr, dtype, shape):
            return C.c_void_p(arr.ctypes.data)
        pin = self.pinned(name, shape, dtype)
        pin.numpy()[...] = np.asarray(arr, dtype=dtype).reshape(pin.shape)
        return C.c_void_p(pin.data_ptr())

    def upload(self, name, src, dst):
        """Fill device tensor ``dst`` from ``src`` without blocking: a CUDA tensor is copied on the device (not at all when
        it is ``dst``), a CPU tensor straight from its memory, a numpy array (or anything np.asarray takes) from itself
        or through pinned buffer ``name`` as ``host_ptr`` decides.  Returns the bytes that crossed PCIe."""
        if isinstance(src, torch.Tensor):
            if src.is_cuda and src.data_ptr() == dst.data_ptr():
                return 0
            dst.copy_(src.reshape(dst.shape), non_blocking=True)
            return 0 if src.is_cuda else dst.numel() * dst.element_size()
        dtype = _NUMPY[dst.dtype]
        if _direct(src, dtype, dst.shape):
            host = torch.from_numpy(src).view(dst.shape)
        else:
            host = self.pinned(name, dst.shape, dtype)
            host.numpy()[...] = np.asarray(src, dtype=dtype).reshape(host.shape)
        dst.copy_(host, non_blocking=True)
        return dst.numel() * dst.element_size()
