"""Guard-banded device buffers shared by the GPU tests: a read outside an input brings a NaN into the result, a write
outside an output changes a guard."""
import torch

GUARD = 64   # elements on each side


class Guarded:
    """n values at element GUARD + off of a buffer of n + 2 GUARD whose guards hold NaN.  For complex64, off = 0 starts
    the view on a 16-byte boundary and off = 1 on an 8-byte one; the view ends where its guard begins."""

    def __init__(self, n, off, fill=None, dtype=torch.complex64):
        self.buf = torch.full((n + 2 * GUARD,), complex(float("nan"), float("nan")), dtype=dtype, device="cuda")
        self.lo, self.hi = GUARD + off, GUARD + off + n
        self.view = self.buf[self.lo:self.hi]
        if dtype == torch.complex64:
            assert (self.view.data_ptr() % 16 == 0) == (off == 0)
        if fill is not None:
            self.view.copy_(torch.as_tensor(fill, dtype=dtype))
        self._guards = self._guard_bits().clone()

    def _guard_bits(self):
        b = torch.view_as_real(self.buf).view(torch.int32)   # one row of int32 words per element
        return torch.cat([b[:self.lo], b[self.hi:]])

    def intact(self):
        return torch.equal(self._guard_bits(), self._guards)

    def numpy(self):
        return self.view.cpu().numpy()
