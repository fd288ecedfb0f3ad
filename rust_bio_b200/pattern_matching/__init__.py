"""Mirror of `bio::pattern_matching` on the H100 engine: the Myers bit-parallel search (`myers`)."""
from . import myers  # noqa: F401
