"""Mirror of `bio::stats` on the H100 engine: the pair HMM (`pairhmm`)."""
from . import pairhmm  # noqa: F401
