"""Registered datasets.

* ``SynthMNLIDataset`` - synthetic MNLI-shaped data (three int64 ``[S]`` tensors + a label in
  ``num_classes``): the workload of every benchmark here (there is no network for GLUE).
* ``SynthMLMDataset`` - a learnable synthetic masked-language-model task (labels ``[S]``).
* ``SynthQADataset`` - a learnable synthetic extractive question-answering task (labels ``[5]``).
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


def bert_mask(ids: torch.Tensor, maskable: torch.Tensor, mask_id: int, random_low: int,
              vocab_size: int, mask_prob: float, g: torch.Generator):
    """BERT masking of one sequence: ``mask_prob`` of the maskable positions (at least one) are
    labelled with their token; of those 80 % become ``mask_id``, 10 % a random token from
    ``[random_low, vocab_size)`` and 10 % stay unchanged.  Returns ``(input_ids, labels)`` with
    -100 on every unlabelled position."""
    pos = torch.nonzero(maskable, as_tuple=False)[:, 0]
    labels = torch.full_like(ids, -100)
    if pos.numel() == 0:
        return ids.clone(), labels
    n = max(1, int(round(mask_prob * pos.numel())))
    chosen = pos[torch.randperm(pos.numel(), generator=g)[:n]]
    labels[chosen] = ids[chosen]
    out = ids.clone()
    r = torch.rand(n, generator=g)
    out[chosen[r < 0.8]] = mask_id
    rnd = chosen[(r >= 0.8) & (r < 0.9)]
    out[rnd] = torch.randint(random_low, vocab_size, (rnd.numel(),), generator=g)
    return out, labels


def _item_generator(seed: int, idx: int) -> torch.Generator:
    return torch.Generator().manual_seed(int(seed) * 1000003 + int(idx))


@DATASET.register_module
class SynthMLMDataset(Dataset):
    """Synthetic masked-language-model data that a model can learn: every sequence is
    ``[CLS] t_1 ... t_{S-2} [SEP]`` with ``t_i = first + (start + i * step) mod (V - first)``, a
    random ``start`` and a random ``step`` in ``1..max_step``, so a masked token follows from its
    neighbours.
    Masking is ``bert_mask``'s (15 % of the body tokens, 80/10/10), deterministic for a given
    ``(seed, index)``; another ``seed`` draws a held-out split of the same task.

    Items are ``((input_ids, token_type_ids, attention_mask), labels[S])`` (labels -100 where not
    masked); ``reference_order=True`` yields ``(input_ids, input_mask, segment_ids)`` instead.
    Vocabularies above 2000 use the BERT ids [CLS] 101, [SEP] 102, [MASK] 103 and body tokens from
    1000; smaller ones 1, 2, 3 and body tokens from 4."""

    def __init__(self, num_samples: int = 1024, max_seq_length: int = 128,
                 vocab_size: int = 30528, mask_prob: float = 0.15, seed: int = 0,
                 reference_order: bool = False, max_step: int = 4):
        if max_seq_length < 3:
            raise ValueError("max_seq_length must be at least 3")
        big = vocab_size > 2000
        self.cls_id, self.sep_id, self.mask_id = (101, 102, 103) if big else (1, 2, 3)
        self.first = 1000 if big else 4
        if vocab_size <= self.first:
            raise ValueError("vocab_size {} leaves no body tokens".format(vocab_size))
        self.vocab_size, self.mask_prob, self.seed = vocab_size, mask_prob, seed
        self.reference_order = reference_order
        g = torch.Generator().manual_seed(seed)
        S, span = max_seq_length, vocab_size - self.first
        start = torch.randint(0, span, (num_samples, 1), generator=g)
        step = torch.randint(1, max_step + 1, (num_samples, 1), generator=g)
        body = self.first + (start + torch.arange(S - 2).unsqueeze(0) * step) % span
        cls = torch.full((num_samples, 1), self.cls_id, dtype=torch.long)
        sep = torch.full((num_samples, 1), self.sep_id, dtype=torch.long)
        self.input_ids = torch.cat([cls, body, sep], dim=1)
        self.input_mask = torch.ones_like(self.input_ids)
        self.segment_ids = torch.zeros_like(self.input_ids)

    def __len__(self):
        return self.input_ids.size(0)

    def __getitem__(self, idx):
        ids = self.input_ids[idx]
        maskable = torch.ones_like(ids, dtype=torch.bool)
        maskable[0] = maskable[-1] = False
        ids, labels = bert_mask(ids, maskable, self.mask_id, self.first, self.vocab_size,
                                self.mask_prob, _item_generator(self.seed, idx))
        if self.reference_order:
            return (ids, self.input_mask[idx], self.segment_ids[idx]), labels
        return (ids, self.segment_ids[idx], self.input_mask[idx]), labels


def pretraining_item(a, b, is_random: int, S: int, cls_id: int, sep_id: int, pad_id: int,
                     mask_id: int, random_low: int, vocab_size: int, mask_prob: float,
                     g: torch.Generator):
    """One masked-LM + next-sentence item from the token lists ``a`` and ``b`` (their total
    already at most S - 3): ``[CLS] a [SEP] b [SEP]`` padded to S, token types 0 up to the first
    [SEP] and 1 after it, ``bert_mask`` over the body tokens only.  Returns ``((input_ids,
    token_type_ids, attention_mask), labels [S + 1])``, the next-sentence label ``is_random`` in
    the last column (``ops.functions.split_pretraining_labels``)."""
    row = [cls_id] + list(a) + [sep_id] + list(b) + [sep_id]
    n = len(row)
    ids = torch.full((S,), pad_id, dtype=torch.long)
    ids[:n] = torch.tensor(row, dtype=torch.long)
    types = torch.zeros(S, dtype=torch.long)
    types[len(a) + 2:n] = 1
    mask = torch.zeros(S, dtype=torch.long)
    mask[:n] = 1
    maskable = mask.bool()
    maskable[0] = maskable[len(a) + 1] = maskable[n - 1] = False
    ids, labels = bert_mask(ids, maskable, mask_id, random_low, vocab_size, mask_prob, g)
    return (ids, types, mask), torch.cat([labels, torch.tensor([int(is_random)])])


@DATASET.register_module
class SynthPretrainingDataset(Dataset):
    """Synthetic masked-LM + next-sentence data that a model can learn.  An item is ``[CLS] A
    [SEP] B [SEP]`` (S tokens, no padding): A is an arithmetic progression as in
    ``SynthMLMDataset`` of random length; for next-sentence label 0 B continues A's progression,
    for label 1 B is the same progression shifted by a random non-zero offset, so it never
    continues A.  The labels are exactly balanced (an odd ``num_samples`` leaves one more 0) and
    drawn with everything else from ``seed``; the masking (``bert_mask``, never a special token)
    depends only on ``(seed, index)``.  Items are ``((input_ids, token_type_ids,
    attention_mask), labels [S + 1])``, the layout of ``ops.functions.split_pretraining_labels``.
    Token ids are ``SynthMLMDataset``'s."""

    def __init__(self, num_samples: int = 1024, max_seq_length: int = 128,
                 vocab_size: int = 30528, mask_prob: float = 0.15, seed: int = 0,
                 max_step: int = 4):
        if max_seq_length < 5:
            raise ValueError("max_seq_length must be at least 5 ([CLS] A [SEP] B [SEP])")
        big = vocab_size > 2000
        self.cls_id, self.sep_id, self.mask_id = (101, 102, 103) if big else (1, 2, 3)
        self.first = 1000 if big else 4
        if vocab_size <= self.first + 1:
            raise ValueError("vocab_size {} leaves too few body tokens".format(vocab_size))
        self.vocab_size, self.mask_prob, self.seed = vocab_size, mask_prob, seed
        self.S = max_seq_length
        g = torch.Generator().manual_seed(seed)
        span = vocab_size - self.first
        self.span = span
        self.start = torch.randint(0, span, (num_samples,), generator=g)
        self.step = torch.randint(1, max_step + 1, (num_samples,), generator=g)
        self.len_a = torch.randint(1, max_seq_length - 3, (num_samples,), generator=g)
        self.offset = torch.randint(1, span, (num_samples,), generator=g)
        self.nsp = (torch.randperm(num_samples, generator=g) >= (num_samples + 1) // 2).long()

    def __len__(self):
        return self.start.numel()

    def __getitem__(self, idx):
        S, la = self.S, int(self.len_a[idx])
        pos = torch.arange(S - 3)
        seq = self.first + (self.start[idx] + pos * self.step[idx]) % self.span
        a = seq[:la]
        b = seq[la:]
        if int(self.nsp[idx]):
            b = self.first + (b - self.first + self.offset[idx]) % self.span
        return pretraining_item(a.tolist(), b.tolist(), int(self.nsp[idx]), S, self.cls_id,
                                self.sep_id, 0, self.mask_id, self.first, self.vocab_size,
                                self.mask_prob, _item_generator(self.seed, idx))


@DATASET.register_module
class SynthQADataset(Dataset):
    """Synthetic extractive question answering that a model can learn.  An item is ``[CLS] q1 q2
    [SEP] context [SEP] pad...``: the context holds the token q1 and, later, the token q2 exactly
    once each, and the answer is the 1..``max_answer_tokens`` tokens between them.  The context
    length varies, so padding and the attention mask are exercised.  Token types are 0 for the
    question part and 1 for the context and its final [SEP].

    Labels are ``[start, end, start_lo, start_hi, end_hi]`` (``ops.functions.split_span_labels``):
    the answer's first and last position, and the context's first and last position as the
    search range.  Item i depends only on ``(seed, i)``; another seed draws a held-out split of
    the same task.  Token ids are ``SynthMLMDataset``'s."""

    def __init__(self, num_samples: int = 1024, max_seq_length: int = 384,
                 vocab_size: int = 30528, seed: int = 0, max_answer_tokens: int = 8):
        if max_answer_tokens < 1 or max_seq_length < max_answer_tokens + 7:
            raise ValueError("max_seq_length must be at least max_answer_tokens + 7 ([CLS] q1 q2 "
                             "[SEP] q1 answer q2 [SEP])")
        big = vocab_size > 2000
        self.cls_id, self.sep_id = (101, 102) if big else (1, 2)
        self.first = 1000 if big else 4
        if vocab_size < self.first + 3:
            raise ValueError("vocab_size {} leaves too few body tokens".format(vocab_size))
        self.num_samples, self.S, self.seed = num_samples, max_seq_length, seed
        self.vocab_size, self.max_answer_tokens = vocab_size, max_answer_tokens

    def __len__(self):
        return self.num_samples

    def __getitem__(self, idx):
        if not 0 <= idx < self.num_samples:
            raise IndexError(idx)
        g = _item_generator(self.seed, idx)
        S, A = self.S, self.max_answer_tokens
        span = self.vocab_size - self.first
        q = torch.randperm(span, generator=g)[:2] + self.first            # q1, q2: distinct
        n_ans = int(torch.randint(1, A + 1, (1,), generator=g))
        n_ctx = int(torch.randint(n_ans + 2, S - 5 + 1, (1,), generator=g))
        # filler and answer tokens: body tokens other than q1 and q2
        ctx = torch.randint(0, span - 2, (n_ctx,), generator=g) + self.first
        for t in sorted(q.tolist()):
            ctx = ctx + (ctx >= t).long()
        p1 = int(torch.randint(0, n_ctx - n_ans - 1, (1,), generator=g))   # q1's context index
        ctx[p1], ctx[p1 + n_ans + 1] = q[0], q[1]
        row = torch.cat([torch.tensor([self.cls_id]), q, torch.tensor([self.sep_id]), ctx,
                         torch.tensor([self.sep_id])])
        n = row.numel()
        ids = torch.zeros(S, dtype=torch.long)
        ids[:n] = row
        types = torch.zeros(S, dtype=torch.long)
        types[4:n] = 1
        mask = torch.zeros(S, dtype=torch.long)
        mask[:n] = 1
        start = 4 + p1 + 1
        last = 4 + n_ctx - 1
        labels = torch.tensor([start, start + n_ans - 1, 4, last, last])
        return (ids, types, mask), labels


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
