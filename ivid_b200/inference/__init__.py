from .sample import sample_all, shard, build_modelviews, async_save, image_grid_u8
from .utils import parse_int_list, save_scene, load_scene, load_scene_views, reorder, colorize_depth
from .render import swing_trajectory, random_views, render_scene
from .superres import superresolve_views
