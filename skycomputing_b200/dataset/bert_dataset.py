"""GlueDataset: tokenises a local GLUE split (``train.tsv`` by default) and caches the features.

Capability parity with scaelum/dataset/bert_dataset.py:16-94 (processor by name, feature cache
pickle next to the data, four int64 tensors).  Offline only: ``vocab_file`` must exist locally.
``reference_order=True`` (default, = the reference) yields ``((input_ids, input_mask,
segment_ids), label)``; ``False`` yields the order ``BertEmbeddings.forward`` consumes.
``split="dev"`` reads the processor's dev file (``dev_matched.tsv`` for MNLI), ``"dev_mismatched"``
MNLI's mismatched dev set; the feature cache of a split other than train carries its name.
"""
from __future__ import annotations

import os
import pickle

import torch
from torch.utils.data import Dataset, TensorDataset

from ..registry import DATASET
from .glue import PROCESSORS, BertTokenizer, convert_examples_to_features


@DATASET.register_module
class GlueDataset(Dataset):
    def __init__(self, data_dir, bert_model, vocab_file, max_seq_length, do_lower_case, processor,
                 reference_order: bool = True, split: str = "train"):
        self.processor = PROCESSORS[processor]()
        self.split = split
        self.tokenizer = BertTokenizer(vocab_file, do_lower_case=do_lower_case, max_len=512)
        self.reference_order = reference_order
        self.dataset = self._build(data_dir, bert_model, max_seq_length, do_lower_case)

    def __getitem__(self, idx):
        input_ids, input_mask, segment_ids, label = self.dataset[idx]
        if self.reference_order:
            return (input_ids, input_mask, segment_ids), label
        return (input_ids, segment_ids, input_mask), label

    def __len__(self):
        return len(self.dataset)

    def _build(self, data_dir, bert_model, max_seq_length, do_lower_case):
        name = "{0}_{1}_{2}".format(bert_model, max_seq_length, do_lower_case)
        if self.split != "train":
            name += "_" + self.split
        cached = os.path.join(data_dir, name)
        try:
            with open(cached, "rb") as reader:
                feats = pickle.load(reader)
        except Exception:
            examples = self.processor.get_split_examples(data_dir, self.split)
            feats = convert_examples_to_features(examples, self.processor.get_labels(),
                                                 max_seq_length, self.tokenizer)
            try:
                with open(cached, "wb") as writer:
                    pickle.dump(feats, writer)
            except OSError:
                pass
        return TensorDataset(
            torch.tensor([f.input_ids for f in feats], dtype=torch.long),
            torch.tensor([f.input_mask for f in feats], dtype=torch.long),
            torch.tensor([f.segment_ids for f in feats], dtype=torch.long),
            torch.tensor([f.label_id for f in feats], dtype=torch.long),
        )
