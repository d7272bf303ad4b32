"""Same public names as reference estimator/models/multi_task_learning/__init__.py:4-5."""
from .mixture_of_experts import MMoE  # noqa: F401
from .esmm import ESMM  # noqa: F401
