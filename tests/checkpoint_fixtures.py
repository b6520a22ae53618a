"""Synthetic checkpoints for tests/test_tree_extents.py and tools/extents_bench.py: the tensor names and shapes of a
Llama-style decoder, and safetensors headers that put the tensors in a chosen order with the header length in a
chosen class mod 16 (the class decides the device-address alignment of every tensor byte within a leaf)."""
from __future__ import annotations

import json
import struct
from typing import List, Sequence, Tuple


def llama_shapes(hidden: int = 4096, inter: int = 14336, layers: int = 32, vocab: int = 128256,
                 kv: int = 1024) -> List[Tuple[str, Tuple[int, ...]]]:
    """The Llama-3-8B layout by default: 291 tensors, about 16 GB in fp16."""
    out = [("model.embed_tokens.weight", (vocab, hidden))]
    for i in range(layers):
        p = f"model.layers.{i}."
        out += [(p + "self_attn.q_proj.weight", (hidden, hidden)), (p + "self_attn.k_proj.weight", (kv, hidden)),
                (p + "self_attn.v_proj.weight", (kv, hidden)), (p + "self_attn.o_proj.weight", (hidden, hidden)),
                (p + "mlp.gate_proj.weight", (inter, hidden)), (p + "mlp.up_proj.weight", (inter, hidden)),
                (p + "mlp.down_proj.weight", (hidden, inter)), (p + "input_layernorm.weight", (hidden,)),
                (p + "post_attention_layernorm.weight", (hidden,))]
    out += [("model.norm.weight", (hidden,)), ("lm_head.weight", (vocab, hidden))]
    return out


SMALL = dict(hidden=2048, inter=5632, layers=8, vocab=32000, kv=512)    # the same structure, about 1 GB in fp16


def header_in_order(entries: Sequence[Tuple[str, str, Sequence[int], int]], mod16: int) -> bytes:
    """A safetensors header whose data_offsets follow `entries` [(name, dtype, shape, nbytes)] in order, with a
    __metadata__ pad chosen so that the whole header length is = mod16 (0 or 8) modulo 16."""
    for k in range(16):
        doc = {"__metadata__": {"pad": "x" * k}}
        off = 0
        for name, dt, shape, nbytes in entries:
            doc[name] = {"dtype": dt, "shape": list(shape), "data_offsets": [off, off + nbytes]}
            off += nbytes
        text = json.dumps(doc, separators=(",", ":")).encode()
        text += b" " * (-len(text) % 8)
        if (8 + len(text)) % 16 == mod16:
            return struct.pack("<Q", len(text)) + text
    raise AssertionError("unreachable: the pad walks through both classes")
