"""CLIP score on the H100 path: the host mirror of `gen_clipscore` (utils_ret.py:1046-1066; called by
diff_retrieval.py:485-487 for the query and the gallery loaders).

    for images, caps in loader:                                   utils_ret.py:1053
        caps = clip.tokenize(caps, 77, True)                      :1055  -> SimpleTokenizer below (BPE, lower-cased, truncated)
        image_features = model.encode_image(images)               :1056  -> nets.build_clip_visual (dcr_net executor)
        text_features  = model.encode_text(caps)                  :1057  -> nets.build_clip_text + end-of-text row selection
        normalise both, sims = (img * txt).sum(-1)                :1058-1062
    return np.mean(scores)                                        :1066

The `clip` package (openai/CLIP) is an un-vendored, unpinned dependency of the reference and is not installed here; its
published tokenizer algorithm and model architecture are restated.  The BPE merges file (`bpe_simple_vocab_16e6.txt.gz`,
shipped inside the clip package) and the ViT-B/16 weights cannot be downloaded in this environment: both are inputs.
"""
from __future__ import annotations

import gzip
import html
from functools import lru_cache
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .nets import DcrNet
from .retrieval import extract_features


@lru_cache()
def _byte_symbols() -> Dict[int, str]:
    """Reversible byte -> printable unicode symbol table of GPT-2 / CLIP BPE: printable latin-1 bytes map to themselves,
    the remaining 68 byte values to code points from 256 upwards."""
    keep = list(range(ord("!"), ord("~") + 1)) + list(range(0xA1, 0xAC + 1)) + list(range(0xAE, 0xFF + 1))
    table, extra = {}, 0
    for b in range(256):
        if b in keep:
            table[b] = chr(b)
        else:
            table[b] = chr(256 + extra)
            extra += 1
    return table


def _symbol_order() -> List[str]:
    """Vocabulary order of the single-byte symbols: the 188 printable bytes first, then the 68 remapped ones."""
    keep = list(range(ord("!"), ord("~") + 1)) + list(range(0xA1, 0xAC + 1)) + list(range(0xAE, 0xFF + 1))
    rest = [b for b in range(256) if b not in keep]
    sym = _byte_symbols()
    return [sym[b] for b in keep + rest]


class SimpleTokenizer:
    """CLIP's byte-level BPE.  Vocabulary = 256 byte symbols, the same 256 with the end-of-word mark `</w>`, one entry per
    merge (the first 48894 lines after the header of the merges file), `<|startoftext|>`, `<|endoftext|>` -> 49408 ids."""

    SOT, EOT = "<|startoftext|>", "<|endoftext|>"

    def __init__(self, bpe_path: str, n_merges: int = 49152 - 256 - 2):
        import regex
        opener = gzip.open if bpe_path.endswith(".gz") else open
        with opener(bpe_path, "rb") as f:
            lines = f.read().decode("utf-8").split("\n")
        merges = [tuple(m.split()) for m in lines[1:1 + n_merges] if m.strip()]
        vocab = _symbol_order()
        vocab = vocab + [v + "</w>" for v in vocab] + ["".join(m) for m in merges] + [self.SOT, self.EOT]
        self.encoder = {tok: i for i, tok in enumerate(vocab)}
        self.decoder = {i: tok for tok, i in self.encoder.items()}
        self.ranks = {m: i for i, m in enumerate(merges)}
        self.cache = {self.SOT: self.SOT, self.EOT: self.EOT}
        self.pat = regex.compile(r"<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+",
                                 regex.IGNORECASE)
        self._regex = regex

    def _bpe(self, token: str) -> str:
        if token in self.cache:
            return self.cache[token]
        word = list(token[:-1]) + [token[-1] + "</w>"]
        while len(word) > 1:
            pairs = {(word[i], word[i + 1]) for i in range(len(word) - 1)}
            best = min(pairs, key=lambda p: self.ranks.get(p, float("inf")))
            if best not in self.ranks:
                break
            a, b = best
            merged, i = [], 0
            while i < len(word):
                if i + 1 < len(word) and word[i] == a and word[i + 1] == b:
                    merged.append(a + b)
                    i += 2
                else:
                    merged.append(word[i])
                    i += 1
            word = merged
        out = " ".join(word)
        self.cache[token] = out
        return out

    def encode(self, text: str) -> List[int]:
        try:                                   # the package cleans mojibake with ftfy when it is installed
            import ftfy
            text = ftfy.fix_text(text)
        except ImportError:
            pass
        text = html.unescape(html.unescape(text)).strip()
        text = self._regex.sub(r"\s+", " ", text).strip().lower()
        sym = _byte_symbols()
        ids: List[int] = []
        for tok in self.pat.findall(text):
            tok = "".join(sym[b] for b in tok.encode("utf-8"))
            ids.extend(self.encoder[t] for t in self._bpe(tok).split(" "))
        return ids

    def tokenize(self, texts, context_length: int = 77, truncate: bool = False) -> torch.Tensor:
        """clip.tokenize: [SOT] + BPE ids + [EOT], zero padded to `context_length`; too long -> cut and end with EOT when
        `truncate` (what utils_ret.py:1055 asks for), RuntimeError otherwise."""
        if isinstance(texts, str):
            texts = [texts]
        sot, eot = self.encoder[self.SOT], self.encoder[self.EOT]
        out = torch.zeros((len(texts), context_length), dtype=torch.int32)
        for i, t in enumerate(texts):
            ids = [sot] + self.encode(t) + [eot]
            if len(ids) > context_length:
                if not truncate:
                    raise RuntimeError(f"Input {t} is too long for context length {context_length}")
                ids = ids[:context_length]
                ids[-1] = eot
            out[i, :len(ids)] = torch.tensor(ids, dtype=torch.int32)
        return out


class ClipScorer:
    """`gen_clipscore` with the model held by the object.  state_dict: the tensors of clip.load("ViT-B/16")[0].state_dict()
    (openai/CLIP names: visual.*, transformer.*, token_embedding.weight, positional_embedding, ln_final.*, text_projection)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], tokenizer: Optional[SimpleTokenizer] = None, max_batch: int = 64,
                 precision: str = "fast", mean: Sequence[float] = (0.5, 0.5, 0.5), std: Sequence[float] = (0.5, 0.5, 0.5)):
        from . import nets
        self.visual = nets.build_clip_visual(state_dict, max_batch=max_batch, precision=precision, mean=mean, std=std)
        self.text = nets.build_clip_text(state_dict, max_batch=max_batch, precision=precision)
        self.tokenizer = tokenizer

    @torch.no_grad()
    def encode_image(self, images: torch.Tensor) -> torch.Tensor:
        """uint8 [n,256,256,3] (host or device) or the transformed float32 [n,3,224,224] -> float32 [n, 512] on the GPU."""
        if images.dtype == torch.uint8:
            return extract_features(self.visual, images)
        return self.visual(images.cuda().float().contiguous())

    @torch.no_grad()
    def encode_text(self, tokens: torch.Tensor) -> torch.Tensor:
        """tokens [n, 77] -> float32 [n, 512]: projected, layer-normed state at the end-of-text position (the arg-max id)."""
        tok = tokens.to(self.text.device)
        per_token = self.text.forward_tokens(tok).view(tok.shape[0], self.text.context_length, self.text.embed_dim)
        return per_token[torch.arange(tok.shape[0], device=tok.device), tok.argmax(dim=-1)]

    @torch.no_grad()
    def pair_scores(self, images: torch.Tensor, captions) -> torch.Tensor:
        if isinstance(captions, torch.Tensor):
            tokens = captions
        else:
            if self.tokenizer is None:
                raise _lib.DcrError("captions given as text need a SimpleTokenizer (pass the clip package's merges file)")
            tokens = self.tokenizer.tokenize(list(captions), 77, True)                      # utils_ret.py:1055
        a, b = self.encode_image(images), self.encode_text(tokens)
        a = a / torch.linalg.norm(a, dim=-1, keepdim=True)                                 # :1058-1061
        b = b / torch.linalg.norm(b, dim=-1, keepdim=True)
        return (a * b).sum(dim=-1)                                                         # :1062

    def score(self, batches: Iterable[Tuple[torch.Tensor, Sequence[str]]]) -> float:
        """np.mean over every (image, caption) pair of the loader (utils_ret.py:1053-1066)."""
        scores: List[float] = []
        for images, caps in batches:
            scores += list(self.pair_scores(images, caps).cpu().numpy())
        return float(np.mean(scores))


def gen_clipscore(dataloader, state_dict, bpe_path: str, precision: str = "fast") -> float:
    """Drop-in for utils_ret.gen_clipscore(dataloader): batches of (images, captions, index) as SynthDataset yields them
    (diff_retrieval.py:102-111)."""
    scorer = ClipScorer(state_dict, SimpleTokenizer(bpe_path), precision=precision)
    return scorer.score((images, caps) for images, caps, _ in dataloader)
