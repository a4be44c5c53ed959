"""`Sequential`: plain modules around exactly one quantizer of this package, called in order, with the quantizer's extra
outputs returned after the last module's output (the reference's utils.Sequential).  `QUANTIZE_KLASSES` is what counts as
a quantizer: every quantizer of the reference that this package has except `LatentQuantize`, which it does not accept (yet);
`BinaryMapper` is not one, as in the reference."""
from torch import nn

from .fsp import FSP
from .fsq import FSQ
from .hierarchical_vq import HierarchicalVQ
from .lfq import LFQ
from .random_projection_quantizer import RandomProjectionQuantizer
from .residual_fsq import GroupedResidualFSQ, ResidualFSQ
from .residual_lfq import GroupedResidualLFQ, ResidualLFQ
from .residual_sim_vq import ResidualSimVQ
from .residual_vq import GroupedResidualVQ, ResidualVQ
from .sim_vq import SimVQ
from .vector_quantize import VectorQuantize

QUANTIZE_KLASSES = (VectorQuantize, ResidualVQ, GroupedResidualVQ, RandomProjectionQuantizer, FSQ, LFQ, SimVQ, ResidualSimVQ,
                    ResidualLFQ, GroupedResidualLFQ, ResidualFSQ, GroupedResidualFSQ, FSP, HierarchicalVQ)


def _is_quantizer(module) -> bool:
    return isinstance(module, QUANTIZE_KLASSES)


class Sequential(nn.Module):
    def __init__(self, *fns: nn.Module):
        super().__init__()
        n_quantizers = sum(1 for fn in fns if _is_quantizer(fn))
        assert n_quantizers == 1, 'this special Sequential must contain exactly one quantizer'
        self.fns = nn.ModuleList(fns)

    def forward(self, x, **kwargs):
        """Runs the modules in order; `kwargs` go to the quantizer alone.  Returns (output of the last module, *the
        quantizer's outputs after its first)."""
        extra = ()
        for fn in self.fns:
            if not _is_quantizer(fn):
                x = fn(x)
                continue
            # Unpacked like a tuple whatever the quantizer returns, as the reference does: RandomProjectionQuantizer's bare
            # index tensor splits along its first (batch) axis.  Kept so that code written against the reference's
            # Sequential gets the same values here.
            x, *extra = fn(x, **kwargs)
        return (x, *extra)
