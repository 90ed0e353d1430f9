from wsl4mis_b200.dataloaders.dataset_semi import *  # noqa: F401,F403
from wsl4mis_b200.dataloaders.dataset_semi import BaseDataSets, RandomGenerator, TwoStreamBatchSampler  # noqa: F401
