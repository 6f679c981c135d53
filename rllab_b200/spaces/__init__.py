from .box import Box  # noqa: F401
from .discrete import Discrete  # noqa: F401
