"""Stand-in for matplotlib: dataloaders/dataset_s2l.py imports matplotlib.pyplot at module level but never calls it."""
