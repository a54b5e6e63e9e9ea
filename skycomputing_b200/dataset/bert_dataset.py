"""GlueDataset and MaskedLMDataset.

GlueDataset: tokenises a local GLUE split (``train.tsv`` by default) and caches the features.

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
from .dataset import _item_generator, bert_mask
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


@DATASET.register_module
class MaskedLMDataset(Dataset):
    """Masked-language-model data from a local text file: the text is tokenised with
    ``BertTokenizer`` (``vocab_file``, which must hold [CLS], [SEP], [MASK] and [PAD]), packed
    into ``[CLS] ... [SEP]`` sequences of at most ``max_seq_length`` tokens (the last one padded)
    and masked the BERT way (``bert_mask``): ``mask_prob`` of the non-special tokens, at least one
    per sequence, 80 % [MASK] / 10 % a random vocabulary token / 10 % unchanged, never [CLS],
    [SEP] or padding.  The masking of item ``i`` depends only on ``(seed, i)``.

    Items are ``((input_ids, token_type_ids, attention_mask), labels[S])`` with -100 on every
    position that is not predicted; ``reference_order=True`` yields ``(input_ids, input_mask,
    segment_ids)`` instead."""

    def __init__(self, text_file, vocab_file, max_seq_length, mask_prob: float = 0.15,
                 seed: int = 0, do_lower_case: bool = True, reference_order: bool = False):
        if max_seq_length < 3:
            raise ValueError("max_seq_length must be at least 3")
        tok = BertTokenizer(vocab_file, do_lower_case=do_lower_case, max_len=1 << 30)
        special = {}
        for name in ("[CLS]", "[SEP]", "[MASK]", "[PAD]"):
            if name not in tok.vocab:
                raise ValueError("{} has no {} token".format(vocab_file, name))
            special[name] = tok.vocab[name]
        self.cls_id, self.sep_id = special["[CLS]"], special["[SEP]"]
        self.mask_id, self.pad_id = special["[MASK]"], special["[PAD]"]
        self.vocab_size = len(tok.vocab)
        self.mask_prob, self.seed = mask_prob, seed
        self.reference_order = reference_order
        ids = []
        with open(text_file, encoding="utf-8") as f:
            for line in f:
                ids.extend(tok.convert_tokens_to_ids(tok.tokenize(line)))
        S, body = max_seq_length, max_seq_length - 2
        n = (len(ids) + body - 1) // body
        self.input_ids = torch.full((n, S), self.pad_id, dtype=torch.long)
        self.input_mask = torch.zeros((n, S), dtype=torch.long)
        for i in range(n):
            chunk = ids[i * body:(i + 1) * body]
            row = [self.cls_id] + chunk + [self.sep_id]
            self.input_ids[i, :len(row)] = torch.tensor(row, dtype=torch.long)
            self.input_mask[i, :len(row)] = 1
        self.segment_ids = torch.zeros_like(self.input_ids)
        self._special = torch.tensor(sorted(set(tok.vocab[t] for t in tok.vocab
                                                if t.startswith("[") and t.endswith("]"))))

    def __len__(self):
        return self.input_ids.size(0)

    def __getitem__(self, idx):
        ids, mask = self.input_ids[idx], self.input_mask[idx]
        maskable = (mask == 1) & ~torch.isin(ids, self._special)
        ids, labels = bert_mask(ids, maskable, self.mask_id, 0, self.vocab_size, self.mask_prob,
                                _item_generator(self.seed, idx))
        if self.reference_order:
            return (ids, mask, self.segment_ids[idx]), labels
        return (ids, self.segment_ids[idx], mask), labels
