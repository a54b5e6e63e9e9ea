"""GLUE task processors and feature conversion (parity with scaelum/dataset/glue/processor.py:
10-310): MRPC / MNLI / CoLA / SST-2 readers for local ``train.tsv`` / ``dev.tsv`` files and the
``[CLS] a [SEP] b [SEP]`` + padding feature builder."""
from __future__ import annotations

import csv
import os
from typing import Dict, List, Optional


class InputExample:
    def __init__(self, guid, text_a, text_b=None, label=None):
        self.guid, self.text_a, self.text_b, self.label = guid, text_a, text_b, label


class InputFeatures:
    def __init__(self, input_ids, input_mask, segment_ids, label_id):
        self.input_ids, self.input_mask = input_ids, input_mask
        self.segment_ids, self.label_id = segment_ids, label_id


class DataProcessor:
    def get_train_examples(self, data_dir):
        raise NotImplementedError

    def get_dev_examples(self, data_dir):
        raise NotImplementedError

    def get_labels(self):
        raise NotImplementedError

    @classmethod
    def _read_tsv(cls, input_file, quotechar=None):
        with open(input_file, "r", encoding="utf-8") as f:
            return [line for line in csv.reader(f, delimiter="\t", quotechar=quotechar)]


class _ColumnProcessor(DataProcessor):
    labels: List[str] = []
    col_a, col_b, col_label, skip_header = 0, None, -1, True
    dev_file = "dev.tsv"
    extra_splits: Dict[str, str] = {}

    def _create(self, lines, set_type):
        out = []
        for i, line in enumerate(lines):
            if i == 0 and self.skip_header:
                continue
            text_b = None if self.col_b is None else line[self.col_b]
            out.append(InputExample("%s-%s" % (set_type, i), line[self.col_a], text_b,
                                    line[self.col_label]))
        return out

    def get_train_examples(self, data_dir):
        return self._create(self._read_tsv(os.path.join(data_dir, "train.tsv")), "train")

    def get_dev_examples(self, data_dir):
        return self._create(self._read_tsv(os.path.join(data_dir, self.dev_file)), "dev")

    def get_split_examples(self, data_dir, split: str):
        """``train``, ``dev`` or one of ``extra_splits`` (file name by split name)."""
        if split == "train":
            return self.get_train_examples(data_dir)
        if split == "dev":
            return self.get_dev_examples(data_dir)
        if split in self.extra_splits:
            return self._create(self._read_tsv(os.path.join(data_dir, self.extra_splits[split])),
                                split)
        raise ValueError("unknown split {!r} (known: {})".format(
            split, ["train", "dev"] + sorted(self.extra_splits)))

    def get_labels(self):
        return list(self.labels)


class MrpcProcessor(_ColumnProcessor):
    labels = ["0", "1"]
    col_a, col_b, col_label = 3, 4, 0


class MnliProcessor(_ColumnProcessor):
    labels = ["contradiction", "entailment", "neutral"]
    col_a, col_b, col_label = 8, 9, -1
    dev_file = "dev_matched.tsv"
    extra_splits = {"dev_mismatched": "dev_mismatched.tsv"}


class ColaProcessor(_ColumnProcessor):
    labels = ["0", "1"]
    col_a, col_b, col_label, skip_header = 3, None, 1, False


class Sst2Processor(_ColumnProcessor):
    labels = ["0", "1"]
    col_a, col_b, col_label = 0, None, 1


PROCESSORS = {"cola": ColaProcessor, "mnli": MnliProcessor, "mrpc": MrpcProcessor,
              "sst-2": Sst2Processor}


def _truncate_seq_pair(tokens_a, tokens_b, max_length):
    while len(tokens_a) + len(tokens_b) > max_length:
        (tokens_a if len(tokens_a) > len(tokens_b) else tokens_b).pop()


def convert_examples_to_features(examples, label_list, max_seq_length, tokenizer):
    label_map = {label: i for i, label in enumerate(label_list)}
    features = []
    for example in examples:
        tokens_a = tokenizer.tokenize(example.text_a)
        tokens_b: Optional[list] = tokenizer.tokenize(example.text_b) if example.text_b else None
        if tokens_b:
            _truncate_seq_pair(tokens_a, tokens_b, max_seq_length - 3)
        elif len(tokens_a) > max_seq_length - 2:
            tokens_a = tokens_a[: max_seq_length - 2]
        tokens = ["[CLS]"] + tokens_a + ["[SEP]"]
        segment_ids = [0] * len(tokens)
        if tokens_b:
            tokens += tokens_b + ["[SEP]"]
            segment_ids += [1] * (len(tokens_b) + 1)
        input_ids = tokenizer.convert_tokens_to_ids(tokens)
        input_mask = [1] * len(input_ids)
        pad = [0] * (max_seq_length - len(input_ids))
        features.append(InputFeatures(input_ids + pad, input_mask + pad, segment_ids + pad,
                                      label_map[example.label]))
    return features
