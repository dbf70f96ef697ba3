"""sdwui prompt syntax: emphasis weights, BREAK, and prompts longer than 75 tokens as several 77-token chunks.

What a remote sdwui does with `prompt` / `negative_prompt` before its text encoder, with its defaults (emphasis mode
"Original", comma_padding_backtrack 20):
  * parse_prompt_attention: `(text)` multiplies the weight of `text` by 1.1, `[text]` divides it by 1.1, `(text:w)`
    multiplies it by w; `\\(`, `\\)`, `\\[`, `\\]` and `\\\\` are literal characters; the word BREAK becomes a segment of
    its own with weight -1.
  * chunk_tokens: the segments' tokens are packed into chunks of 75 (FrozenCLIPEmbedderWithCustomWordsBase.tokenize_line),
    each framed as [BOS] + tokens + [EOS] padding + [EOS], with one multiplier per token.

Not interpreted (as text they reach the tokenizer unchanged): prompt editing `[a:b:when]`, alternation `[a|b]`,
composable `AND`, textual-inversion embeddings and extra-network tags.
"""
import re
from typing import Callable, List, Optional, Sequence, Tuple

ROUND = 1.1          # weight factor of ( )
SQUARE = 1 / 1.1     # weight factor of [ ]
CHUNK_TOKENS = 75    # prompt tokens per chunk; with BOS and EOS a chunk is 77 ids
COMMA_BACKTRACK = 20  # sdwui comma_padding_backtrack default

_TOKEN = re.compile(r"""
\\\(|\\\)|\\\[|\\\]|\\\\|\\|   # escapes (and a lone backslash)
\(|\[|                         # openers
:\s*([+-]?[.\d]+)\s*\)|        # ':weight)' closes a round bracket with an explicit weight
\)|\]|                         # closers
[^\\()\[\]:]+|                 # plain text
:                              # a colon that closes nothing
""", re.X)
_BREAK = re.compile(r"\s*\bBREAK\b\s*", re.S)


def parse_prompt_attention(text: str) -> List[Tuple[str, float]]:
    """Prompt text -> [(segment, weight)] with neighbouring equal weights merged; BREAK -> ("BREAK", -1).
    An opener without its closer applies up to the end of the text; a closer without an opener is literal text."""
    res: List[list] = []
    round_open: List[int] = []
    square_open: List[int] = []

    def scale(start: int, factor: float):
        for seg in res[start:]:
            seg[1] *= factor

    for m in _TOKEN.finditer(text):
        tok, weight = m.group(0), m.group(1)
        if tok.startswith("\\"):
            res.append([tok[1:], 1.0])
        elif tok == "(":
            round_open.append(len(res))
        elif tok == "[":
            square_open.append(len(res))
        elif weight is not None and round_open:
            scale(round_open.pop(), float(weight))
        elif tok == ")" and round_open:
            scale(round_open.pop(), ROUND)
        elif tok == "]" and square_open:
            scale(square_open.pop(), SQUARE)
        else:
            for i, part in enumerate(_BREAK.split(tok)):
                if i:
                    res.append(["BREAK", -1.0])
                res.append([part, 1.0])
    for start in round_open:
        scale(start, ROUND)
    for start in square_open:
        scale(start, SQUARE)
    if not res:
        return [("", 1.0)]
    merged = [res[0]]
    for seg in res[1:]:
        if seg[1] == merged[-1][1]:
            merged[-1][0] += seg[0]
        else:
            merged.append(seg)
    return [(t, w) for t, w in merged]


def chunk_tokens(segments: Sequence[Tuple[Sequence[int], float, bool]], bos: int, eos: int,
                 comma: Optional[int] = None, backtrack: int = COMMA_BACKTRACK) -> Tuple[List[List[int]], List[List[float]]]:
    """[(token ids, weight, is_break)] -> (chunks of 77 ids, their 77 multipliers), sdwui's tokenize_line.
    A chunk takes 75 tokens.  When a full chunk is followed by a non-comma token and the chunk's last comma is within its
    last `backtrack` tokens, the tokens after that comma move to the next chunk.  BREAK closes the current chunk (an empty
    one too).  An empty prompt is one chunk."""
    chunks: List[List[int]] = []
    mults: List[List[float]] = []
    cur: List[int] = []
    cur_m: List[float] = []
    last_comma = -1

    def close(tokens, weights):
        nonlocal last_comma
        pad = CHUNK_TOKENS - len(tokens)
        chunks.append([bos] + tokens + [eos] * pad + [eos])
        mults.append([1.0] + weights + [1.0] * pad + [1.0])
        last_comma = -1

    for ids, weight, is_break in segments:
        if is_break:
            close(cur, cur_m)
            cur, cur_m = [], []
            continue
        for t in ids:
            if comma is not None and t == comma:
                last_comma = len(cur)
            elif (backtrack and len(cur) == CHUNK_TOKENS and last_comma != -1
                  and len(cur) - last_comma <= backtrack):
                keep = last_comma + 1
                moved, moved_m = cur[keep:], cur_m[keep:]
                close(cur[:keep], cur_m[:keep])
                cur, cur_m = moved, moved_m
            if len(cur) == CHUNK_TOKENS:
                close(cur, cur_m)
                cur, cur_m = [], []
            cur.append(t)
            cur_m.append(weight)
    if cur or not chunks:
        close(cur, cur_m)
    return chunks, mults


def tokenize_prompt(text: str, tokenize: Callable[[str], List[int]], bos: int, eos: int,
                    comma: Optional[int] = None) -> Tuple[List[List[int]], List[List[float]]]:
    """one prompt -> (chunks of 77 ids, multipliers); `tokenize` maps a segment's text to ids without BOS / EOS"""
    segs = [((), w, True) if (t == "BREAK" and w == -1) else (tokenize(t), w, False)
            for t, w in parse_prompt_attention(text)]
    return chunk_tokens(segs, bos, eos, comma)
