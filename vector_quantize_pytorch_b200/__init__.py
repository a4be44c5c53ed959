"""H100-native (sm_90a) nearest-code search / gather / EMA kernels behind the vector-quantize-pytorch API.

Drop-in for ONE path of lucidrains/vector-quantize-pytorch: `VectorQuantize`, `ResidualVQ`,
`GroupedResidualVQ` forward (`(quantized, indices, commit_loss)`), the `Codebook` surface, `SimVQ`'s search,
`ResidualSimVQ`, finite scalar quantization (`FSQ`, `ResidualFSQ`, `GroupedResidualFSQ`),
lookup-free quantization (`LFQ`, `ResidualLFQ`, `GroupedResidualLFQ`), finite scalar perturbation (`FSP`)
the binary mapper (`BinaryMapper`), multi-scale residual VQ over feature maps (`HierarchicalVQ`), the BEST-RQ random-projection
quantizer (`RandomProjectionQuantizer`), latent quantization (`LatentQuantize`) and the one-quantizer container
`Sequential`.
The hot path is hand-written CUDA (wgmma / TMA / mbarrier) in `csrc/`, bound through the C ABI in
`include/vqb200.h`.  No Triton, no CPU fallback.
"""
from .codebook import Codebook, EuclideanCodebook, CosineSimCodebook  # noqa: E402
from .vector_quantize import VectorQuantize  # noqa: E402
from .residual_vq import ResidualVQ, GroupedResidualVQ  # noqa: E402
from .sim_vq import SimVQ  # noqa: E402
from .residual_sim_vq import ResidualSimVQ  # noqa: E402
from .fsq import FSQ  # noqa: E402
from .residual_fsq import ResidualFSQ, GroupedResidualFSQ  # noqa: E402
from .lfq import LFQ  # noqa: E402
from .residual_lfq import ResidualLFQ, GroupedResidualLFQ  # noqa: E402
from .fsp import FSP  # noqa: E402
from .binary_mapper import BinaryMapper  # noqa: E402
from .hierarchical_vq import HierarchicalVQ  # noqa: E402
from .random_projection_quantizer import RandomProjectionQuantizer  # noqa: E402
from .latent_quantize import LatentQuantize  # noqa: E402
from .utils import Sequential  # noqa: E402

__all__ = ["Codebook", "EuclideanCodebook", "CosineSimCodebook", "VectorQuantize", "ResidualVQ", "GroupedResidualVQ", "SimVQ",
           "ResidualSimVQ", "FSQ", "ResidualFSQ", "GroupedResidualFSQ",
           "LFQ", "ResidualLFQ", "GroupedResidualLFQ", "FSP", "BinaryMapper", "HierarchicalVQ",
           "RandomProjectionQuantizer", "LatentQuantize", "Sequential"]
