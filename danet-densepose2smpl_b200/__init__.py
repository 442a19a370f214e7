"""H100-native DaNet inference hot path (HRNet IUV estimator -> part regressors -> SMPL LBS ->
IUV rasteriser) behind the reference's call surface.  See DESIGN.md."""
__version__ = "0.1.0"

from . import constants  # noqa: F401
from .smpl import SMPL, ModelOutput_, mpjpe_h36m  # noqa: F401
from .renderer import IUV_Renderer  # noqa: F401
from . import geometry, iuvmap  # noqa: F401
from .danet import DaNet, build_synthetic_danet  # noqa: F401
from . import synthetic  # noqa: F401
from . import parallel, evaluate, losses, regressor, conv, layers, stn  # noqa: F401
from . import optim, targets, training  # noqa: F401
from . import estimator  # noqa: F401
from .estimator import iuv_estimator  # noqa: F401
from .part_utils import PartRenderer  # noqa: F401
