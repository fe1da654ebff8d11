"""MASt3R pair inference on Hopper (wgmma) tensor cores behind the reference's model surface."""
from . import ops  # noqa: F401  (registers the C signatures)
from .model import FULL_CFG, AsymmetricMASt3R, forward_pair  # noqa: F401
from .graph import BENCH_PAIRS_PER_GPU, GraphedForwardPair  # noqa: F401,E402
from . import curope, wrappers  # noqa: F401,E402
