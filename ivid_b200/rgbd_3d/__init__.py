from .renderer import AggregationRenderer, SimpleRenderer, DeviceWarp
from . import utils
from . import glm_compat
from . import fusion
from .fusion import tsdf_integrate, extract_surface, fuse_views, write_ply
