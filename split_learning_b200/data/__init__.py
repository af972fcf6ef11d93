"""Datasets and loaders: ``data_loader(data_name, batch_size, distribution, train)``
(reference src/dataset/dataloader.py:124-133) plus synthetic stand-ins of identical shape."""
from .distribution import label_counts
from .loaders import DATASET_SHAPES, SyntheticDataset, data_loader, resident_test_loader, synthetic_loader

__all__ = ["label_counts", "data_loader", "resident_test_loader", "synthetic_loader", "SyntheticDataset", "DATASET_SHAPES"]
