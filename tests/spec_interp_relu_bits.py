"""TEST INFRASTRUCTURE: the CPU interpreter of ``spec_interp`` extended with restatements of the two op types of the
bit-mask refinement step program (``lama_b200.relu_bits``).  The interpreter keeps a bit mask as one 0 / 1 value per
element of a (B, H, W, C) float64 buffer; the device stores it as uint32 words (include/ffc_b200.h:
ffcb_relu_mask_pack)."""
from spec_interp import SpecInterpreter, storage_nbytes


class BitsSpecInterpreter(SpecInterpreter):
    def MaskPackOp(self, op, ext):
        self.write(op.bits, (self.read(op.y) > 0).double())

    def ReluBwdBitsOp(self, op, ext):
        self.write(op.out, self.read(op.dy) * self.read(op.bits))


def storage_nbytes_bits(b):
    """Device bytes of a buffer's storage, bit masks included (uint32 words, ceil(C/32) per pixel)."""
    if b.bits:
        return b.B * b.H * b.W * -(-b.C // 32) * 4
    return storage_nbytes(b)
