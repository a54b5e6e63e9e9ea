"""Host-side checks of the wrappers in front of the embedding kernels (no GPU needed)."""
import ctypes
import types

import numpy as np
import pytest
import torch


def _int64_at(ptr, n):
    return np.frombuffer(ctypes.string_at(ptr, 8 * n), dtype=np.int64).copy()


@pytest.mark.parametrize("ids_dtype,mask_dtype", [(torch.int32, torch.bool),
                                                  (torch.int32, torch.int32),
                                                  (torch.int64, torch.bool),
                                                  (torch.int64, torch.int64)])
def test_embeddings_fn_hands_int64_indices_to_the_kernel(monkeypatch, ids_dtype, mask_dtype):
    """embed_fwd reads ids, token types and the mask as contiguous int64: EmbeddingsFn must
    convert int32 ids and bool / int32 masks instead of passing their storage through."""
    from skycomputing_b200.models import BertConfig
    from skycomputing_b200.models.bert_layers import BertEmbeddings
    from skycomputing_b200.ops import functions

    B, S = 2, 8
    ep = functions.EmbeddingParams(BertEmbeddings(BertConfig(64, hidden_size=16).__dict__))
    ids = torch.arange(B * S).reshape(S, B).t()           # non-contiguous
    tts = (torch.arange(B * S) % 2).reshape(B, S)
    mask = torch.ones(B, S)
    mask[1, 5:] = 0
    seen = {}

    def embed_fwd(**kw):
        seen.update({k: _int64_at(kw[k], B * S) for k in ("ids", "tts", "amask")})

    monkeypatch.setattr(functions.nat, "ext", lambda: types.SimpleNamespace(embed_fwd=embed_fwd))
    monkeypatch.setattr(torch.cuda, "current_stream",
                        lambda *a: types.SimpleNamespace(cuda_stream=0))
    functions.EmbeddingsFn.apply(ep, False, None, 0, ids.to(ids_dtype), tts.to(ids_dtype),
                                 mask.to(mask_dtype), *ep.all_params())
    assert np.array_equal(seen["ids"], ids.reshape(-1).numpy())
    assert np.array_equal(seen["tts"], tts.reshape(-1).numpy())
    assert np.array_equal(seen["amask"], mask.reshape(-1).long().numpy())
