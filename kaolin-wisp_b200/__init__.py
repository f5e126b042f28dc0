"""wisp_b200 -- Hopper (sm_90a) volumetric render path behind the kaolin-wisp API.

Import as `wisp_b200` (the directory is named kaolin-wisp_b200 per the repo layout; the top-level `wisp_b200`
package aliases it).  Host-side classes mirror the reference's names and arguments; all compute goes through
libwispb200.so (hand-written CUDA behind a C ABI, include/wispb200.h).  There is no CPU fallback.
"""
from . import _cabi, ops, spc, parallel, raygen                                                   # noqa: F401
from ._cabi import WispB200Error                                                # noqa: F401
from .core import Rays, RenderBuffer                                            # noqa: F401
from .accelstructs import OctreeAS, AxisAlignedBBoxAS, ASQueryResults, ASRaymarchResults, ASRaytraceResults   # noqa: F401
from .grids import HashGrid, MultiTable, TriplanarGrid, TriplanarFeatureVolume, OctreeGrid, CodebookOctreeGrid                                         # noqa: F401
from .nefs import NeuralRadianceField, NeuralSDF, BasicDecoder, PositionalEmbedder, get_positional_embedder   # noqa: F401
from .tracers import PackedRFTracer, PackedSDFTracer                                             # noqa: F401
from .pipeline import Pipeline                                                  # noqa: F401
from . import trainers                                                          # noqa: F401
from .trainers import MultiviewStep, NativeAdam, NativeAdamW, NativeRMSprop, SDFStep   # noqa: F401

__version__ = "0.1.0"
