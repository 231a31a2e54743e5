"""Guarded, poisoned output buffers for the GPU tests (DESIGN section 9).

Every output, gradient and workspace is a view inside a larger allocation filled with one NaN bit pattern; after the
call the bytes around each view must still hold it (no write outside the buffer), and every element of an output view
must be finite (no element left unwritten, which a zero-filled buffer would hide where the right answer is 0).  Calls
whose right answer may hold NaN or inf take a `poison` pattern of their own, one no kernel writes (the signalling NaN
POISON_SNAN); their output views must then hold no element with that bit pattern.
"""
import numpy as np
import torch

POISON32 = 0x7FC0DEAD           # a quiet NaN as fp32
POISON16 = 0x7FC07FC0           # two quiet NaNs as fp16 and as bf16
POISON_SNAN = 0x7F80DEAD        # a signalling NaN as fp32: arithmetic never produces it
LEAD, TAIL = 256, 256           # guard bytes in front of / behind every view
SENTINEL = 12345.0              # finite value of elements a call must leave alone


class Arena(object):
    """Views carved out of poisoned allocations, and the check that nothing outside them changed."""

    def __init__(self, poison=None):
        """poison: the fp32 bit pattern of the output views (default POISON32, and finite outputs required); with a
        pattern given, output views are checked for elements still holding it instead of for finiteness."""
        self.items = []
        self.poison = poison

    def _alloc(self, nbytes, misalign, poison):
        words = (LEAD + misalign + nbytes + TAIL + 3) // 4
        raw = torch.full((words,), poison, dtype=torch.int32, device="cuda")
        return raw, LEAD + misalign

    def out(self, shape, dtype=torch.float32, misalign=0, fill=None):
        """An output view: poisoned (or `fill`ed), guarded; must come back finite."""
        es = torch.empty((), dtype=dtype).element_size()
        n = int(np.prod(shape))
        if self.poison is not None:
            assert es == 4, "a poison pattern is for fp32 outputs"
        raw, start = self._alloc(n * es, misalign, self.poison if self.poison is not None else
                                 POISON32 if es == 4 else POISON16)
        v = raw.view(torch.uint8)[start:start + n * es].view(dtype).view(shape)
        if fill is not None:
            v.fill_(fill)
        self.items.append((raw, raw.clone(), start, n * es, v, "output %s" % (tuple(shape),)))
        return v

    def workspace(self, nbytes):
        """A workspace of exactly nbytes (None for 0); its contents are scratch, only its guards are checked."""
        if not nbytes:
            return None
        raw, start = self._alloc(nbytes, 0, POISON32)
        v = raw.view(torch.uint8)[start:start + nbytes]
        self.items.append((raw, raw.clone(), start, nbytes, None, "workspace of %d bytes" % nbytes))
        return v

    def check(self):
        torch.cuda.synchronize()
        for raw, orig, start, nbytes, view, what in self.items:
            b, o = raw.view(torch.uint8), orig.view(torch.uint8)
            assert torch.equal(b[:start], o[:start]), "%s: the guard in front was written" % what
            assert torch.equal(b[start + nbytes:], o[start + nbytes:]), "%s: the guard behind was written" % what
            if view is not None and self.poison is not None:
                left = view.view(torch.int32) == self.poison - (1 << 32 if self.poison >= 1 << 31 else 0)
                assert not bool(left.any()), "%s: %d elements still hold the poison (never written?)" % (
                    what, int(left.sum()))
            elif view is not None:
                assert bool(torch.isfinite(view).all()), "%s: %d elements not finite (never written?)" % (
                    what, int((~torch.isfinite(view)).sum()))
