"""SQuAD v1.1 extractive question answering: ``SquadDataset`` and the official answer scores.

``SquadDataset`` reads a local SQuAD v1.1 JSON file and builds the features of the HF / Google
BERT v1 recipe: whitespace words with a character-to-word map, WordPiece sub-tokens, the improved
answer span, and ``[CLS] question [SEP] window [SEP]`` windows over the document that advance by
``doc_stride``.  Items are ``((input_ids, token_type_ids, attention_mask), labels [5])`` in the
layout of ``ops.functions.split_span_labels``.

``normalize_answer`` / ``exact_match_score`` / ``f1_score`` are the official SQuAD v1.1 evaluation
formulas; ``SquadDataset.text_scores`` applies them to the spans an evaluation pass predicted.
"""
from __future__ import annotations

import collections
import json
import re
import string

import torch
from torch.utils.data import Dataset

from ..registry import DATASET
from .glue import BertTokenizer

IGNORE_INDEX = -100


def normalize_answer(s: str) -> str:
    """Lower case, no punctuation, no articles (a / an / the), collapsed whitespace."""
    s = "".join(ch for ch in s.lower() if ch not in set(string.punctuation))
    s = re.sub(r"\b(a|an|the)\b", " ", s)
    return " ".join(s.split())


def exact_match_score(prediction: str, ground_truth: str) -> float:
    return float(normalize_answer(prediction) == normalize_answer(ground_truth))


def f1_score(prediction: str, ground_truth: str) -> float:
    pred, gold = normalize_answer(prediction).split(), normalize_answer(ground_truth).split()
    same = sum((collections.Counter(pred) & collections.Counter(gold)).values())
    if same == 0:
        return 0.0
    p, r = same / len(pred), same / len(gold)
    return 2 * p * r / (p + r)


def _is_whitespace(c: str) -> bool:
    return c in " \t\r\n" or ord(c) == 0x202F


def _words(text: str):
    """Whitespace words of ``text`` and the word index of every character."""
    words, char_to_word, prev_ws = [], [], True
    for c in text:
        if _is_whitespace(c):
            prev_ws = True
        else:
            if prev_ws:
                words.append(c)
            else:
                words[-1] += c
            prev_ws = False
        char_to_word.append(len(words) - 1)
    return words, char_to_word


def _improve_answer_span(doc_tokens, start: int, end: int, tokenizer, answer: str):
    """The sub-token span that matches the tokenised answer exactly, if one lies inside the
    word-level span (e.g. "1895" inside "(1895-1943)."), else the word-level span."""
    target = " ".join(tokenizer.tokenize(answer))
    for s in range(start, end + 1):
        for e in range(end, s - 1, -1):
            if " ".join(doc_tokens[s:e + 1]) == target:
                return s, e
    return start, end


def _max_context_window(windows, position: int) -> int:
    """Index of the window in which ``position`` has the most context: the largest min(left,
    right) context plus 0.01 x the window length, the first window on a tie."""
    best, best_score = None, None
    for k, (start, length) in enumerate(windows):
        end = start + length - 1
        if position < start or position > end:
            continue
        score = min(position - start, end - position) + 0.01 * length
        if best_score is None or score > best_score:
            best, best_score = k, score
    return best


@DATASET.register_module
class SquadDataset(Dataset):
    """Features of a local SQuAD v1.1 JSON file (HF ``BertForQuestionAnswering``'s v1 recipe).

    Every question yields one feature per window.  Labels per window (``split_span_labels``):
    the gold answer's first and last token in the window; ``start_lo .. start_hi``, the part of
    the window's context in which this window has the most context of all windows (a ValueError
    if that part is not contiguous); ``end_hi``, the window's last context token.  A training
    window without the answer is labelled (0, 0), the [CLS] token; a dev window without the
    first gold answer gets ``ignore_index`` in the two gold columns, so the device metrics count
    only windows that contain it.  ``text_scores`` scores predicted spans against every gold
    answer with the official SQuAD v1.1 metric.  SQuAD v2 entries (``is_impossible``) raise
    ValueError."""

    def __init__(self, json_file, vocab_file, max_seq_length: int = 384, doc_stride: int = 128,
                 max_query_length: int = 64, split: str = "train", do_lower_case: bool = True):
        if split not in ("train", "dev"):
            raise ValueError("split must be 'train' or 'dev', got {!r}".format(split))
        self.tokenizer = tok = BertTokenizer(vocab_file, do_lower_case=do_lower_case, max_len=1 << 30)
        for name in ("[CLS]", "[SEP]"):
            if name not in tok.vocab:
                raise ValueError("{} has no {} token".format(vocab_file, name))
        cls_id, sep_id = tok.vocab["[CLS]"], tok.vocab["[SEP]"]
        with open(json_file, encoding="utf-8") as f:
            data = json.load(f)["data"]
        self.examples = []     # (doc words, gold answer texts)
        self.features = []     # (example index, window start, query length, tok_to_orig)
        ids_l, types_l, mask_l, labels_l = [], [], [], []
        S = max_seq_length
        for article in data:
            for para in article["paragraphs"]:
                words, char_to_word = _words(para["context"])
                tok_to_orig, orig_to_tok, doc_tokens = [], [], []
                for i, w in enumerate(words):
                    orig_to_tok.append(len(doc_tokens))
                    for sub in tok.tokenize(w):
                        tok_to_orig.append(i)
                        doc_tokens.append(sub)
                for qa in para["qas"]:
                    if qa.get("is_impossible"):
                        raise ValueError("question {} is a SQuAD v2 entry (is_impossible): only "
                                         "SQuAD v1.1 is supported".format(qa.get("id")))
                    answers = qa["answers"]
                    if not answers:
                        raise ValueError("question {} has no answer".format(qa.get("id")))
                    ans = answers[0]
                    a_start = char_to_word[ans["answer_start"]]
                    a_end = char_to_word[ans["answer_start"] + len(ans["text"]) - 1]
                    t_start = orig_to_tok[a_start]
                    t_end = (orig_to_tok[a_end + 1] - 1 if a_end < len(words) - 1
                             else len(doc_tokens) - 1)
                    t_start, t_end = _improve_answer_span(doc_tokens, t_start, t_end, tok,
                                                          ans["text"])
                    query = tok.tokenize(qa["question"])[:max_query_length]
                    room = S - len(query) - 3
                    if room < 1:
                        raise ValueError("max_seq_length {} leaves no room for the document "
                                         "after a question of {} tokens".format(S, len(query)))
                    windows, off = [], 0
                    while off < len(doc_tokens):
                        length = min(len(doc_tokens) - off, room)
                        windows.append((off, length))
                        if off + length == len(doc_tokens):
                            break
                        off += min(length, doc_stride)
                    ex = len(self.examples)
                    self.examples.append((words, [a["text"] for a in answers]))
                    q = len(query) + 2          # position of the window's first token
                    for k, (start, length) in enumerate(windows):
                        row = ([cls_id] + tok.convert_tokens_to_ids(query) + [sep_id]
                               + tok.convert_tokens_to_ids(doc_tokens[start:start + length])
                               + [sep_id])
                        n = len(row)
                        ids = torch.zeros(S, dtype=torch.long)
                        ids[:n] = torch.tensor(row)
                        types = torch.zeros(S, dtype=torch.long)
                        types[q:n] = 1
                        mask = torch.zeros(S, dtype=torch.long)
                        mask[:n] = 1
                        best = [q + i for i in range(length)
                                if _max_context_window(windows, start + i) == k]
                        if best and best[-1] - best[0] + 1 != len(best):
                            raise ValueError("the max-context positions of a window are not "
                                             "contiguous: {}".format(best))
                        lo, hi = (best[0], best[-1]) if best else (0, -1)
                        if start <= t_start and t_end <= start + length - 1:
                            gold = (t_start - start + q, t_end - start + q)
                        else:
                            gold = (0, 0) if split == "train" else (IGNORE_INDEX, IGNORE_INDEX)
                        ids_l.append(ids)
                        types_l.append(types)
                        mask_l.append(mask)
                        labels_l.append(torch.tensor([gold[0], gold[1], lo, hi, q + length - 1]))
                        self.features.append((ex, start, q, tok_to_orig))
        self.input_ids = torch.stack(ids_l) if ids_l else torch.zeros(0, S, dtype=torch.long)
        self.segment_ids = torch.stack(types_l) if types_l else torch.zeros(0, S, dtype=torch.long)
        self.input_mask = torch.stack(mask_l) if mask_l else torch.zeros(0, S, dtype=torch.long)
        self.labels = torch.stack(labels_l) if labels_l else torch.zeros(0, 5, dtype=torch.long)

    def __len__(self):
        return self.input_ids.size(0)

    def __getitem__(self, idx):
        return (self.input_ids[idx], self.segment_ids[idx], self.input_mask[idx]), self.labels[idx]

    def answer_text(self, idx: int, i: int, j: int) -> str:
        """The original whitespace words that token positions ``i..j`` of feature ``idx`` cover
        ("" for the empty span (-1, -1) or a span outside the window's document tokens)."""
        ex, start, q, tok_to_orig = self.features[idx]
        words = self.examples[ex][0]
        a, b = start + i - q, start + j - q
        if i < q or j < i or a < 0 or b >= len(tok_to_orig):
            return ""
        return " ".join(words[tok_to_orig[a]:tok_to_orig[b] + 1])

    def text_scores(self, spans, scores) -> dict:
        """Official SQuAD v1.1 ``text_exact_match`` and ``text_f1`` (percent) of predicted spans
        ``[len(self), 2]`` with their scores ``[len(self)]``: per question the window with the
        highest score wins (the first on a tie), its answer is the words the span covers, and EM
        and F1 are the maxima over the gold answers, averaged over every question."""
        spans = torch.as_tensor(spans).reshape(-1, 2).tolist()
        scores = torch.as_tensor(scores).reshape(-1).tolist()
        if len(spans) != len(self) or len(scores) != len(self):
            raise ValueError("text_scores needs one span and score per feature ({})".format(len(self)))
        best = {}
        for idx, (ex, _, _, _) in enumerate(self.features):
            if ex not in best or scores[idx] > scores[best[ex]]:
                best[ex] = idx
        em = f1 = 0.0
        for ex, (_, golds) in enumerate(self.examples):
            pred = self.answer_text(best[ex], *spans[best[ex]]) if ex in best else ""
            em += max(exact_match_score(pred, g) for g in golds)
            f1 += max(f1_score(pred, g) for g in golds)
        n = max(len(self.examples), 1)
        return dict(text_exact_match=100.0 * em / n, text_f1=100.0 * f1 / n)
