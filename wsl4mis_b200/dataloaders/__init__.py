"""GPU input pipeline (SURVEY 8(f) rank 2): resident slice store + batch augmentation kernel."""
from .dataset import BaseDataSets, GpuLoader, RandomGenerator, SliceStore  # noqa: F401
from .random_walker import random_walker_labels  # noqa: F401
