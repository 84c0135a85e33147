"""Write the InternVideo2 text-tower golden data under tests/golden/, from the reference's own, unmodified bert/xbert.py and
bert/tokenization_bert.py imported at generation time:

* internvideo2_text_tokens.json: the reference tokenizer's `tokenize` + `convert_tokens_to_ids` over a corpus (ASCII, accents, CJK,
  emoji, control characters, non-ASCII punctuation, over-long words, empty and whitespace-only strings) with the synthetic vocabulary
  tests/golden/bert_vocab_synth.txt, which this script also writes.
* internvideo2_text_ref.npz: BertModel(mode="text") + text_proj + L2 norm (get_txt_feat, internvideo2_mm.py:219-241) at full width
  (hidden 1024, 16 heads of 64, intermediate 4096) and depth 2, built with num_hidden_layers=3 and fusion_layer=2 so that a
  cross-attention layer exists and text mode skips it; seeded weights (tests rebuild them with
  cosmos_curate_b200.models.internvideo2.seeded_text_weights); texts of different lengths, one exactly 40 tokens and one truncated.
  Stored: the token ids and lengths, the float32 embeddings and the reference's bf16 embeddings (for scale).

The [CLS] / [SEP] / truncation / [PAD] assembly is the transformers-4 rule the reference was written against ([CLS] + pieces[:38] +
[SEP], [PAD] to 40): under transformers 5 the reference tokenizer's __call__ leaves out [SEP], so only its tokenize and
convert_tokens_to_ids are used.  Shims for transformers 5 (the reference pins transformers < 5): apply_chunking_to_forward and
prune_linear_layer live in transformers.pytorch_utils, find_pruneable_heads_and_indices is gone (unused in eval), _is_control /
_is_punctuation / _is_whitespace live in transformers.tokenization_python, get_head_mask is gone ([None] * layers stands in), and
init_weights is stubbed (every tensor is overwritten anyway).

    python -m oracle.make_internvideo2_text_golden
"""

from __future__ import annotations

import importlib
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from cosmos_curate_b200.models.internvideo2 import text_reference_keys  # noqa: E402
from oracle import internvideo2_text as O  # noqa: E402
from oracle import ref_import  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
VOCAB_FILE = "bert_vocab_synth.txt"
SEED = 21
DEPTH = 2
MAX_LEN = 40

_WORDS = ("a an the of on in at with and is are to from by for it this that his her their man woman men women child children "
          "dog dogs cat cats car cars bike street road city park beach water sea sky tree trees house room kitchen table ball game "
          "red blue green white black small large young old people person group video clip scene shot camera view close up "
          "walk walks walking run runs running play plays playing ride rides riding sit sits sitting stand stands standing talk "
          "cafe resume naive over under left right front back top down one two three day night sun snow rain un re").split()  # fmt: skip
_SUFFIXES = "s ing ed er es ly ness able aff ful ion".split()
_CJK = "中国人大小日本猫狗水"
_PUNCT = "—–“”‘’…¿¡«»·•€£¥§¶†"


def synthetic_vocab() -> list[str]:
    """BERT's layout for the special ids ([PAD] 0, [unused*], [UNK] 100, [CLS] 101, [SEP] 102, [MASK] 103), then single characters,
    their ## continuations, words and suffixes."""
    v = ["[PAD]"] + [f"[unused{i}]" for i in range(99)] + ["[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    chars = [chr(c) for c in range(33, 127) if not chr(c).isupper()] + list(_CJK) + list(_PUNCT)
    v += chars + ["##" + c for c in "abcdefghijklmnopqrstuvwxyz0123456789"]
    v += [w for w in _WORDS if w not in v]
    v += [s for s in ("##" + x for x in _SUFFIXES) if s not in v]
    assert len(v) == len(set(v))
    return v


TOKENIZER_CORPUS = [
    "a man walks his dog on the beach",
    "Two children PLAYING ball in the park!",
    "The cat's toy, under the table.",
    "résumé naïve café Ångström ÉLAN",
    "中国人 walking in 日本",
    "大小猫狗水",
    "a dog 🐶 runs 🏃‍♂️ fast 😀",
    "tab\there\nnew line\r\nend",
    "nul\x00char and \ufffd replacement",
    "bell\x07 and escape\x1b[0m codes",
    "zero\u200bwidth\u200djoiner\ufeff soft\u00adhyphen",
    "line\u2028separator\u2029paragraph\u00a0nbsp\u3000ideographic\u2003em",
    "“quoted” — dash – en… ¿qué? ¡sí! «guillemets» · bullet • €5 £3 ¥9",
    "unaffable unplayable rerunning",
    "a" * 100,
    "a" * 101,
    "ok " + "b" * 150 + " ok",
    "supercalifragilisticexpialidocious",
    "",
    "   ",
    "\t\n \u3000 ",
    "a [MASK] dog and [CLS] [SEP] tokens",
    "x^2 + y_1 = $5 `code` ~tilde~ |pipe|",
    "ǅ ß ǆ ﬁ ① ½ Ⅻ ǲ",
    "e\u0301 a\u0300 combining marks \u0301 alone \u0308",
    "ΣΟΦΙΑ Москва العربية हिन्दी 한국어 ひらがな カタカナ",
    "the quick brown fox jumps over the lazy dog 0123456789",
]

# the tower batch: several lengths, one text of exactly 40 tokens ([CLS] + 38 + [SEP]) and one truncated
TOWER_TEXTS = [
    "a dog",
    "a man walks his dog on the beach at night",
    " ".join(["red"] * 38),
    "two children playing ball in the park while people sit on the grass and a woman rides a bike down the street near "
    "the sea under a blue sky with white snow on the trees and a black car",
    "中国人",
    "cafe resume: un naive walking video clip, close up!",
]


def _shim_transformers() -> None:
    import transformers.modeling_utils as mu
    import transformers.pytorch_utils as pu

    for name in ("apply_chunking_to_forward", "prune_linear_layer"):
        if not hasattr(mu, name):
            setattr(mu, name, getattr(pu, name))
    if not hasattr(mu, "find_pruneable_heads_and_indices"):
        def find_pruneable_heads_and_indices(*args, **kwargs):
            raise NotImplementedError("head pruning is not used in eval")

        mu.find_pruneable_heads_and_indices = find_pruneable_heads_and_indices
    import transformers.tokenization_python as tp
    import transformers.tokenization_utils as tu

    for name in ("_is_control", "_is_punctuation", "_is_whitespace"):
        if not hasattr(tu, name):
            setattr(tu, name, getattr(tp, name))


def reference_bert():
    ref_import._install_stubs()
    _shim_transformers()
    return importlib.import_module("cosmos_curate.models.internvideo2_multi_modality.bert.xbert")


def reference_tokenizer(vocab_path: Path):
    ref_import._install_stubs()
    _shim_transformers()
    mod = importlib.import_module("cosmos_curate.models.internvideo2_multi_modality.bert.tokenization_bert")
    return mod.BertTokenizer(str(vocab_path), do_lower_case=True)


def assemble(pieces: list[int], cls_id: int, sep_id: int, pad_id: int, max_len: int) -> tuple[list[int], int]:
    """transformers-4 padding="max_length", truncation=True for one sequence."""
    seq = [cls_id, *pieces[: max_len - 2], sep_id]
    return seq + [pad_id] * (max_len - len(seq)), len(seq)


def reference_model(cfg: O.TextConfig, w: dict):
    """BertModel(add_pooling_layer=False) in text mode plus text_proj, with `w` loaded under the reference's keys."""
    xbert = reference_bert()
    xbert.BertModel.init_weights = lambda self: None
    xbert.BertModel.get_head_mask = lambda self, head_mask, n, *a, **k: [None] * n
    bc = xbert.BertConfig(vocab_size=cfg.vocab, hidden_size=cfg.hidden, num_hidden_layers=cfg.layers + 1, num_attention_heads=cfg.heads,
                          intermediate_size=cfg.mlp, hidden_act="gelu", hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                          max_position_embeddings=cfg.max_pos, type_vocab_size=2, layer_norm_eps=cfg.ln_eps, pad_token_id=0,
                          position_embedding_type="absolute")  # fmt: skip
    bc.fusion_layer, bc.encoder_width, bc.cross_module = cfg.layers, cfg.hidden, "ca"
    bert = xbert.BertModel(bc, add_pooling_layer=False)
    text_proj = torch.nn.Linear(cfg.hidden, cfg.embed_dim)
    assert bert.encoder.layer[cfg.layers].has_cross_attention and not bert.encoder.layer[cfg.layers - 1].has_cross_attention
    sd = {k: torch.randn_like(v) * 0.02 if v.is_floating_point() else v for k, v in bert.state_dict().items()}  # unused tensors: any values
    sd["embeddings.token_type_embeddings.weight"][1] = 0.0
    for name, a in w.items():
        keys = text_reference_keys(name)
        t = torch.from_numpy(a)
        if keys[0].startswith("text_proj."):
            getattr(text_proj, keys[0].split(".")[1]).data.copy_(t)
            continue
        keys = [k[len("text_encoder.bert.") :] for k in keys]
        if name == "type_emb":
            sd[keys[0]][0] = t
            continue
        for k, part in zip(keys, t.chunk(len(keys), 0)):
            assert k in sd and sd[k].shape == part.shape, (k, part.shape)
            sd[k] = part.clone()
    bert.load_state_dict(sd)
    return bert.eval(), text_proj.eval()


@torch.no_grad()
def reference_embeddings(bert, text_proj, ids: np.ndarray, lengths: np.ndarray, dtype) -> np.ndarray:
    """encode_text (internvideo2_mm.py:115-136) with mode="text", the [CLS] row, text_proj, / norm (get_txt_feat)."""
    bert, text_proj = bert.to(dtype), text_proj.to(dtype)
    input_ids = torch.from_numpy(ids).long()
    mask = (torch.arange(ids.shape[1])[None, :] < torch.from_numpy(lengths)[:, None]).long()
    out = bert(input_ids, attention_mask=mask, return_dict=True, mode="text").last_hidden_state
    e = text_proj(out[:, 0]).float()
    return (e / e.norm(dim=-1, keepdim=True)).numpy()


def main() -> None:
    vocab_path = GOLDEN / VOCAB_FILE
    vocab_path.write_text("".join(t + "\n" for t in synthetic_vocab()), encoding="utf-8")
    tok = reference_tokenizer(vocab_path)
    cases = []
    for text in TOKENIZER_CORPUS:
        tokens = tok.tokenize(text)
        cases.append({"text": text, "tokens": tokens, "ids": [int(i) for i in tok.convert_tokens_to_ids(tokens)]})
    meta = {"vocab": VOCAB_FILE, "cases": cases}
    (GOLDEN / "internvideo2_text_tokens.json").write_text(json.dumps(meta, ensure_ascii=False, indent=0) + "\n", encoding="utf-8")
    print(f"tokenizer: {len(cases)} texts, {sum(len(c['ids']) for c in cases)} tokens")

    ids_l, lens = [], []
    v = tok.vocab
    for text in TOWER_TEXTS:
        seq, n = assemble(tok.convert_tokens_to_ids(tok.tokenize(text)), v["[CLS]"], v["[SEP]"], v["[PAD]"], MAX_LEN)
        ids_l.append(seq)
        lens.append(n)
    ids, lengths = np.array(ids_l, dtype=np.int32), np.array(lens, dtype=np.int32)
    assert MAX_LEN in lens and len(tok.tokenize(TOWER_TEXTS[3])) > MAX_LEN - 2 and len(tok.tokenize(TOWER_TEXTS[2])) == MAX_LEN - 2
    cfg = O.IV2_TEXT.with_(layers=DEPTH, vocab=len(v))
    w = O.random_weights(cfg, SEED)
    bert, text_proj = reference_model(cfg, w)
    emb = reference_embeddings(bert, text_proj, ids, lengths, torch.float32)
    emb_bf16 = reference_embeddings(bert, text_proj, ids, lengths, torch.bfloat16)
    print(f"tower: lengths {lens}; reference bf16 vs float32 min cosine {(emb * emb_bf16).sum(-1).min():.6f}, max-abs {np.abs(emb - emb_bf16).max():.2e}")
    tower_meta = {"seed": SEED, "depth": DEPTH, "vocab": len(v), "texts": TOWER_TEXTS}
    path = GOLDEN / "internvideo2_text_ref.npz"
    np.savez_compressed(path, ids=ids, lengths=lengths, emb=emb, emb_bf16=emb_bf16,
                        meta=np.frombuffer(json.dumps(tower_meta).encode(), dtype=np.uint8))  # fmt: skip
    print(f"wrote {path} ({path.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
