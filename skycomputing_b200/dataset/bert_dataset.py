"""GlueDataset, MaskedLMDataset and PreTrainingDataset.

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
from .dataset import _item_generator, bert_mask, pretraining_item
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


@DATASET.register_module
class PreTrainingDataset(Dataset):
    """Masked-LM + next-sentence data from a local text file in the input format of BERT's
    ``create_pretraining_data``: one sentence per line, a blank line between documents.  The
    text is tokenised with ``BertTokenizer`` (``vocab_file`` must hold [CLS], [SEP], [MASK] and
    [PAD]).  Item i starts segment A at the i-th sentence of the corpus and takes a random run of
    sentences of its document; B is, chosen 50/50, the sentences that follow A (next-sentence
    label 0; an A that would start at its document's last sentence starts one sentence earlier)
    or a run from a random other document (label 1; always for a one-sentence document).  The
    pair is truncated to S - 3 tokens, longer side first, and masked as ``MaskedLMDataset`` does
    (never [CLS], [SEP] or padding).  Item i depends only on ``(seed, i)``.  Items are
    ``((input_ids, token_type_ids, attention_mask), labels [S + 1])``
    (``ops.functions.split_pretraining_labels``).  A file with fewer than two documents raises
    ``ValueError``: the random B needs another document."""

    def __init__(self, text_file, vocab_file, max_seq_length, mask_prob: float = 0.15,
                 seed: int = 0, do_lower_case: bool = True):
        if max_seq_length < 5:
            raise ValueError("max_seq_length must be at least 5 ([CLS] A [SEP] B [SEP])")
        tok = BertTokenizer(vocab_file, do_lower_case=do_lower_case, max_len=1 << 30)
        for name in ("[CLS]", "[SEP]", "[MASK]", "[PAD]"):
            if name not in tok.vocab:
                raise ValueError("{} has no {} token".format(vocab_file, name))
        self.cls_id, self.sep_id = tok.vocab["[CLS]"], tok.vocab["[SEP]"]
        self.mask_id, self.pad_id = tok.vocab["[MASK]"], tok.vocab["[PAD]"]
        self.vocab_size = len(tok.vocab)
        self.S, self.mask_prob, self.seed = max_seq_length, mask_prob, seed
        docs, cur = [], []
        with open(text_file, encoding="utf-8") as f:
            for line in f:
                if not line.strip():
                    if cur:
                        docs.append(cur)
                    cur = []
                    continue
                ids = tok.convert_tokens_to_ids(tok.tokenize(line))
                if ids:
                    cur.append(ids)
        if cur:
            docs.append(cur)
        if len(docs) < 2:
            raise ValueError("{} holds {} document(s); next-sentence pairs need at least two "
                             "(documents are separated by blank lines)".format(text_file, len(docs)))
        self.docs = docs
        self.index = [(d, k) for d, doc in enumerate(docs) for k in range(len(doc))]

    def __len__(self):
        return len(self.index)

    def __getitem__(self, idx):
        g = _item_generator(self.seed, idx)
        target = self.S - 3
        d, k = self.index[idx]
        doc = self.docs[d]
        is_random = float(torch.rand(1, generator=g)) < 0.5 or len(doc) < 2
        if not is_random:
            # B follows A: A starts early enough to leave at least one sentence after it
            k = min(k, len(doc) - 2)
            n_a = int(torch.randint(1, len(doc) - k, (1,), generator=g))
        else:
            n_a = int(torch.randint(1, len(doc) - k + 1, (1,), generator=g))
        a = [t for s in doc[k:k + n_a] for t in s]
        if not is_random:
            rest = doc[k + n_a:]
        else:
            other = int(torch.randint(0, len(self.docs) - 1, (1,), generator=g))
            other += other >= d
            odoc = self.docs[other]
            rest = odoc[int(torch.randint(0, len(odoc), (1,), generator=g)):]
        b = []
        for s in rest:
            if len(a) + len(b) >= target:
                break
            b.extend(s)
        while len(a) + len(b) > target:
            (a if len(a) > len(b) else b).pop()
        if not b:   # A alone filled the budget: keep one B token
            a.pop()
            b = rest[0][:1]
        return pretraining_item(a, b, int(is_random), self.S, self.cls_id, self.sep_id,
                                self.pad_id, self.mask_id, 0, self.vocab_size, self.mask_prob, g)
