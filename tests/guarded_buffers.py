"""Operands and outputs of the GPU kernel tests placed inside larger guarded buffers: an operand inside NaN shows a kernel that
reads past the extents it was given, an output inside a sentinel shows one that writes past them."""
import torch


class Guarded:
    """``view`` at row 1, column 16 of a larger buffer (row pitch a multiple of ``pitch_multiple`` elements, at least 56
    columns wider than the view, one extra row above and two below); the rest of the buffer holds ``fill``.  A 1-D source
    sits at offset 16 of a buffer 48 elements longer."""

    def __init__(self, src: torch.Tensor, fill, interior=None, pitch_multiple: int = 16):
        self.src_shape = tuple(src.shape)
        if src.dim() == 1:
            self.buf = torch.full((src.numel() + 48,), fill, dtype=src.dtype, device="cuda")
            self.view = self.buf[16:16 + src.numel()]
        else:
            rows, cols = src.shape
            pitch = (cols + 16 + 40 + pitch_multiple - 1) // pitch_multiple * pitch_multiple
            self.buf = torch.full((rows + 3, pitch), fill, dtype=src.dtype, device="cuda")
            self.view = self.buf[1:1 + rows, 16:16 + cols]
        self.view.copy_(src if interior is None else interior)
        self.snap = self.buf.clone()

    def guards_intact(self) -> bool:
        """Every element outside the view still holds its initial bits."""
        b = self.buf.clone()
        b[self._region()] = self.snap[self._region()]
        bits = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[b.element_size()]
        return torch.equal(b.view(bits), self.snap.view(bits))

    def _region(self):
        if len(self.src_shape) == 1:
            return slice(16, 16 + self.src_shape[0])
        return (slice(1, 1 + self.src_shape[0]), slice(16, 16 + self.src_shape[1]))
