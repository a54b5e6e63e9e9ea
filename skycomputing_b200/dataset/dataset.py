"""Registered datasets.

* ``SynthMNLIDataset`` - synthetic MNLI-shaped data (three int64 ``[S]`` tensors + a label in
  ``num_classes``): the workload of every benchmark here (there is no network for GLUE).
* ``RandomMlpDataset`` / ``CIFAR10Dataset`` - parity with scaelum/dataset/dataset.py:14-48.
"""
from __future__ import annotations

import random

import torch
from torch.utils.data import Dataset

from ..registry import DATASET


@DATASET.register_module
class SynthMNLIDataset(Dataset):
    """Random token ids with MNLI-like structure: ``[CLS] a [SEP] b [SEP] pad...``.

    ``label_rule="random"`` (default) draws labels independently of the tokens; ``"token"`` sets
    ``label = input_ids[:, 1] % num_classes``, a task a model can learn and be evaluated on.

    Items are ``((input_ids, token_type_ids, attention_mask), label)`` - the order
    ``BertEmbeddings.forward`` consumes.  ``reference_order=True`` yields the reference
    ``GlueDataset`` order ``(input_ids, input_mask, segment_ids)`` instead
    (scaelum/dataset/bert_dataset.py:34-37,85-90; see SURVEY §2.7 for the mismatch it causes).
    """

    def __init__(self, num_samples: int = 1024, max_seq_length: int = 128, vocab_size: int = 30522,
                 num_classes: int = 3, seed: int = 0, full_length: bool = True,
                 reference_order: bool = False, label_rule: str = "random"):
        g = torch.Generator().manual_seed(seed)
        S = max_seq_length
        low = 1000 if vocab_size > 2000 else max(1, vocab_size // 10)
        self.input_ids = torch.randint(low, vocab_size, (num_samples, S), generator=g)
        if full_length:
            lens = torch.full((num_samples,), S, dtype=torch.long)
        else:
            lens = torch.randint(max(8, S // 4), S + 1, (num_samples,), generator=g)
        pos = torch.arange(S).unsqueeze(0)
        self.input_mask = (pos < lens.unsqueeze(1)).long()
        split = (lens // 2).unsqueeze(1)
        self.segment_ids = ((pos >= split) & (pos < lens.unsqueeze(1))).long()
        self.input_ids = self.input_ids * self.input_mask
        self.input_ids[:, 0] = min(101, vocab_size - 1)  # [CLS]
        self.labels = torch.randint(0, num_classes, (num_samples,), generator=g)
        if label_rule == "token":
            # a learnable task: the label is a function of the first token after [CLS]; another
            # seed draws another sample of the same task (a held-out split)
            self.labels = self.input_ids[:, 1] % num_classes
        elif label_rule != "random":
            raise ValueError("label_rule must be 'random' or 'token', got {!r}".format(label_rule))
        self.reference_order = reference_order

    def __len__(self):
        return self.input_ids.size(0)

    def __getitem__(self, idx):
        if self.reference_order:
            data = (self.input_ids[idx], self.input_mask[idx], self.segment_ids[idx])
        else:
            data = (self.input_ids[idx], self.segment_ids[idx], self.input_mask[idx])
        return data, self.labels[idx]


@DATASET.register_module
class RandomMlpDataset(Dataset):
    def __init__(self, num=1000, dim=1024):
        self.dim = dim
        self.data = torch.rand(num, dim)

    def __len__(self):
        return self.data.size(0)

    def __getitem__(self, idx):
        return self.data[idx], random.randint(0, self.dim - 1)


@DATASET.register_module
class RandomImageDataset(Dataset):
    """CIFAR-shaped random images for the ResNet layer library (offline stand-in for CIFAR10)."""

    def __init__(self, num=512, channels=3, size=32, num_classes=100, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.data = torch.rand(num, channels, size, size, generator=g)
        self.labels = torch.randint(0, num_classes, (num,), generator=g)

    def __len__(self):
        return self.data.size(0)

    def __getitem__(self, idx):
        return self.data[idx], self.labels[idx]


@DATASET.register_module
class CIFAR10Dataset(Dataset):
    """torchvision CIFAR10 with the reference's augmentation; needs torchvision + local data."""

    def __init__(self, mean, std, *args, **kwargs):
        try:
            import torchvision
            import torchvision.transforms as transforms
        except Exception as e:  # pragma: no cover
            raise ImportError("CIFAR10Dataset needs torchvision, which is not installed") from e
        transform_train = transforms.Compose([
            transforms.RandomCrop(32, padding=4),
            transforms.RandomHorizontalFlip(),
            transforms.RandomRotation(15),
            transforms.ToTensor(),
            transforms.Normalize(mean, std),
        ])
        self.cifar10dataset = torchvision.datasets.CIFAR10(transform=transform_train, *args, **kwargs)

    def __len__(self):
        return len(self.cifar10dataset)

    def __getitem__(self, idx):
        return self.cifar10dataset[idx]
