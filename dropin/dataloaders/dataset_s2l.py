from wsl4mis_b200.dataloaders.dataset import BaseDataSets_s2l, RandomGenerator_s2l  # noqa: F401
