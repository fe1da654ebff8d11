"""Pi3 on Hopper (wgmma) tensor cores behind the reference's model surface, and the Backend's accurate loop closure."""
from .model import Pi3, interpolate_pos_embed, param_shapes, svd_pose  # noqa: F401  (registers the C signatures)
from .loop_closure import accurate_loop_closure, score_window, window_input  # noqa: F401
