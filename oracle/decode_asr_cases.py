"""TEST INFRASTRUCTURE (oracle/): random inputs for the token-ids -> text / chunks post-processing, and the checker side of the
comparison: the installed `WhisperTokenizer._decode_asr` (TF/models/whisper/tokenization_whisper.py) with the seam merge the reference
installs over transformers' (REF thestage_speechkit/__init__.py:137-139) -- the real one when the reference is importable (golden
minting, oracle/make_golden.py --only decode_asr), else its restatement oracle/hf_ref.lcs_merge (pinned to the real one by
tests/golden/lcs_cases.json).  Only tests/ and oracle/make_golden.py import this file.

The cases are built on the synthetic tokenizer (thewhisper_b200/synthetic.py): ids 0..255 are the single bytes (so multi-byte UTF-8
characters, split and broken sequences can be composed at will), 256.. are " w<i>" words, then the large-v3 special / language /
timestamp layout.
"""
from __future__ import annotations

import contextlib
from typing import List

import numpy as np

from thewhisper_b200 import synthetic as S

TB = S.TIMESTAMP_BEGIN
LANGS = ["en", "zh", "ja", "es", "th", "de"]


_TOK = {}


def special_tokenizer():
    """The synthetic tokenizer with its control tokens registered as SPECIAL tokens, as released Whisper checkpoints have them
    (`all_special_ids` = <|endoftext|> ... <|notimestamps|>): with thewhisper_b200.synthetic.make_tokenizer() only <|endoftext|> is special, so
    `_decode_asr` never takes its language branches there.  Same ids."""
    if "special" in _TOK:
        return _TOK["special"]
    from tokenizers import AddedToken
    from transformers import WhisperTokenizer

    b2u = S._bytes_to_unicode()
    vocab = {}
    for b in range(256):
        vocab[b2u[b]] = len(vocab)
    i = 0
    while len(vocab) < S.EOS:
        vocab[f"\u0120w{i}"] = len(vocab)
        i += 1
    specials = ["<|startoftranscript|>"] + [f"<|{c}|>" for c in S.LANG_CODES] + ["<|translate|>", "<|transcribe|>", "<|startoflm|>", "<|startofprev|>",
                                                                                 "<|nospeech|>", "<|notimestamps|>"]
    tok = WhisperTokenizer(vocab=vocab, merges=[], pad_token="<|endoftext|>", extra_special_tokens=specials)
    tok.add_tokens([AddedToken("<|%.2f|>" % (k * 0.02), special=False, normalized=False) for k in range(1501)])
    assert len(tok) == S.VOCAB and tok.all_special_ids[-1] == S.NOTIMESTAMPS and len(tok.all_special_ids) == S.NOTIMESTAMPS - S.EOS + 1
    assert tok.convert_tokens_to_ids(["<|startoftranscript|>", "<|en|>", "<|0.00|>"]) == [S.SOT, S.LANG_EN, S.TIMESTAMP_BEGIN]
    _TOK["special"] = tok
    return tok


def tokenizer_of(kind: str):
    return special_tokenizer() if kind == "special" else S.make_tokenizer()


def _b(text: str) -> List[int]:
    return list(text.encode("utf-8"))


_SNIPPETS = [" hello", " world", ",", ".", " (", ")", " \"", "\"", "!", "?", " -", "-", " é", "é", " naïve", "中", "文", " 日本", "語", " \U0001f600", "ß", " ¿", "¡",
             "。", "，", " “", "”", "'s", " n't", " .", " ,", "  ", " ", "\n", " <|1.23|>", "<|0.5|", "<|\u0661\u0662.\u0663|>", " <|\uff11.5|>x", "<|1.\u0e52|", "<|12.|>", " a", "b", "c", " 12", ".5", " :", ":", " [", "]", " {", "}"]


def random_text_tokens(rng, n: int) -> List[int]:
    out: List[int] = []
    while len(out) < n:
        r = rng.rand()
        if r < 0.45:
            out.append(int(256 + rng.randint(0, 3000)))  # " w<i>"
        elif r < 0.85:
            out += _b(_SNIPPETS[rng.randint(len(_SNIPPETS))])
        elif r < 0.93:
            s = _b(_SNIPPETS[rng.randint(len(_SNIPPETS))])  # a broken sequence: drop a byte of a multi-byte character
            if len(s) > 1:
                del s[rng.randint(len(s))]
            out += s
        else:
            out.append(int(rng.randint(0x80, 0x100)))  # a stray high byte
    return out[:n]


def random_case(rng, tokenizer) -> dict:
    """One call of `_decode_asr`: {"model_outputs": [...], "return_timestamps": None | True | "word", "return_language": bool,
    "time_precision": float}.  Arrays are plain lists (JSON-able); as_model_outputs() turns them into what the pipeline passes."""
    mode = [None, True, "word"][rng.randint(3)]
    return_language = bool(rng.rand() < 0.4)
    time_precision = 0.02
    n_win = int(rng.choice([1, 1, 2, 3, 4]))
    strided = n_win > 1 or rng.rand() < 0.3
    chunk_len, stride = (30.0, 5.0) if rng.rand() < 0.7 else (10.0, 10.0 / 6)
    lang = LANGS[rng.randint(len(LANGS))]
    lang_id = tokenizer.convert_tokens_to_ids(f"<|{lang}|>")
    outs = []
    carry: List[int] = []  # text tokens shared with the next window (the overlap the seam merge has to find)
    for w in range(n_win):
        ids: List[int] = []
        if rng.rand() < 0.1:
            ids += [tokenizer.convert_tokens_to_ids("<|startofprev|>")] + random_text_tokens(rng, int(rng.randint(1, 5)))
        ids.append(S.SOT)
        if rng.rand() < 0.9:
            ids.append(lang_id)
        ids.append(S.TRANSCRIBE)
        if mode is None and rng.rand() < 0.7:
            ids.append(S.NOTIMESTAMPS)
        use_ts = mode is not None or rng.rand() < 0.3
        t = 0
        body = list(carry)
        body += random_text_tokens(rng, int(rng.randint(0, 14)))
        carry = body[-int(rng.randint(2, 7)):] if (len(body) > 3 and rng.rand() < 0.8) else []
        if mode is None and rng.rand() < 0.15:  # a language switch in mid-stream
            other = tokenizer.convert_tokens_to_ids(f"<|{LANGS[rng.randint(len(LANGS))]}|>")
            body.insert(int(rng.randint(0, len(body) + 1)), other)
        if use_ts:
            pos = 0
            limit = int(chunk_len / time_precision)
            while pos < len(body) or rng.rand() < 0.15:
                seg = body[pos: pos + int(rng.randint(1, 7))]
                pos += len(seg)
                if rng.rand() < 0.9:
                    ids.append(TB + min(t, limit))
                ids += seg
                t += int(rng.randint(1, 250))
                if rng.rand() < 0.9:
                    ids.append(TB + min(t, limit))
                if rng.rand() < 0.08:
                    t = int(rng.randint(0, 40))  # a new generate() segment: times start again
                if pos >= len(body) and rng.rand() < 0.7:
                    break
        else:
            ids += body
        if rng.rand() < 0.5:
            ids.append(S.EOS)
        o = {"tokens": [ids]}
        if mode == "word":
            tt = np.cumsum(rng.rand(len(ids)) * 0.4).astype(np.float32)
            if rng.rand() < 0.05 and len(tt) > 2:
                tt = tt[:-1]  # too short: the original raises IndexError when it gets that far
            o["token_timestamps"] = [tt.tolist()]
        if strided:
            sl = 0.0 if w == 0 else stride
            sr = 0.0 if w == n_win - 1 else stride
            ln = chunk_len if w < n_win - 1 else float(np.round(rng.uniform(sl + 0.5, chunk_len), 2))
            o["stride"] = [ln, sl, sr]
        outs.append(o)
    return {"model_outputs": outs, "return_timestamps": mode, "return_language": return_language, "time_precision": time_precision}


def as_model_outputs(case: dict) -> list:
    outs = []
    for o in case["model_outputs"]:
        d = {"tokens": np.asarray(o["tokens"], dtype=np.int64)}
        if "token_timestamps" in o:
            d["token_timestamps"] = np.asarray(o["token_timestamps"], dtype=np.float32)
        if "stride" in o:
            d["stride"] = tuple(o["stride"])
        outs.append(d)
    return outs


@contextlib.contextmanager
def seam_merge(fn):
    """Run with `fn` installed as the tokenizer module's seam merge (what `import thestage_speechkit` does with its own)."""
    import transformers.models.whisper.tokenization_whisper as tw

    saved = tw._find_longest_common_sequence
    tw._find_longest_common_sequence = fn
    try:
        yield
    finally:
        tw._find_longest_common_sequence = saved


def reference_result(case: dict, tokenizer, merge_fn):
    """(text, optional) of the installed tokenizer, or {"raises": "<ExceptionType>"}."""
    with seam_merge(merge_fn):
        try:
            text, opt = tokenizer._decode_asr(as_model_outputs(case), return_timestamps=case["return_timestamps"],
                                              return_language=case["return_language"], time_precision=case["time_precision"])
        except (IndexError, KeyError, TypeError, ValueError, RuntimeError) as e:
            return {"raises": type(e).__name__}
    return {"text": text, "optional": jsonable(opt)}


def jsonable(o):
    if isinstance(o, dict):
        return {k: jsonable(v) for k, v in o.items()}
    if isinstance(o, (list, tuple)):
        return [jsonable(v) for v in o]
    if isinstance(o, (np.floating, np.integer)):
        return o.item()
    return o
