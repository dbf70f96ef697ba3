"""sdwui prompt syntax: emphasis weights, BREAK, and prompts longer than 75 tokens as several 77-token chunks.

What a remote sdwui does with `prompt` / `negative_prompt` before its text encoder, with its defaults (emphasis mode
"Original", comma_padding_backtrack 20):
  * parse_prompt_attention: `(text)` multiplies the weight of `text` by 1.1, `[text]` divides it by 1.1, `(text:w)`
    multiplies it by w; `\\(`, `\\)`, `\\[`, `\\]` and `\\\\` are literal characters; the word BREAK becomes a segment of
    its own with weight -1.
  * chunk_tokens: the segments' tokens are packed into chunks of 75 (FrozenCLIPEmbedderWithCustomWordsBase.tokenize_line),
    each framed as [BOS] + tokens + [EOS] padding + [EOS], with one multiplier per token.  A tower whose pad id is not EOS
    (SD 2.x's OpenCLIP: 0) gets that id after the first EOS of every chunk (process_tokens).

Prompt editing `[from:to:when]` and alternation `[a|b]` (prompt_parser.get_learned_conditioning_prompt_schedules):
prompt_schedule turns a prompt into [(end_at_step, text)]; the engine encodes each text once and switches the
cross-attention context per model evaluation (schedule_index: sdwui's reconstruct_cond_batch).  Known parity gap: sdwui
parses with lark's Earley parser, which resolves the ambiguity between a group and a run of two or more stray bracket or
colon characters right after its closer in a way that depends on the rest of the prompt (`x [b:c:4]]] y` and
`[a:b:5]):` stay literal text there, `[a:1]:` does not); prompt_schedule always parses such a group.

Extra-network tags (`<lora:name:0.8>`, sdwui extra_networks.parse_prompt) are cut out of the positive prompt before any
of this by b200sd.lora.parse_prompt, which also turns lora / lyco tags into the networks merged for the request.

Not interpreted (as text they reach the tokenizer unchanged): composable `AND` and textual-inversion embeddings.
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
                 comma: Optional[int] = None, backtrack: int = COMMA_BACKTRACK,
                 pad: Optional[int] = None) -> Tuple[List[List[int]], List[List[float]]]:
    """[(token ids, weight, is_break)] -> (chunks of 77 ids, their 77 multipliers), sdwui's tokenize_line.
    A chunk takes 75 tokens.  When a full chunk is followed by a non-comma token and the chunk's last comma is within its
    last `backtrack` tokens, the tokens after that comma move to the next chunk.  BREAK closes the current chunk (an empty
    one too).  An empty prompt is one chunk.  pad: the id after the first EOS of a chunk (None: EOS)."""
    chunks: List[List[int]] = []
    mults: List[List[float]] = []
    cur: List[int] = []
    cur_m: List[float] = []
    last_comma = -1

    def close(tokens, weights):
        nonlocal last_comma
        n_pad = CHUNK_TOKENS - len(tokens)
        chunks.append([bos] + tokens + [eos] + [eos if pad is None else pad] * n_pad)
        mults.append([1.0] + weights + [1.0] * n_pad + [1.0])
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
                    comma: Optional[int] = None, pad: Optional[int] = None) -> Tuple[List[List[int]], List[List[float]]]:
    """one prompt -> (chunks of 77 ids, multipliers); `tokenize` maps a segment's text to ids without BOS / EOS; pad:
    the id after each chunk's first EOS (None: EOS)"""
    segs = [((), w, True) if (t == "BREAK" and w == -1) else (tokenize(t), w, False)
            for t, w in parse_prompt_attention(text)]
    return chunk_tokens(segs, bos, eos, comma, pad=pad)


# ------------------------------------------------------------------------------------------------ prompt editing
# sdwui's schedule grammar (prompt_parser.schedule_parser):
#   start: (prompt | stray "[", "]", "(", ")", ":")*     prompt: (emphasized | scheduled | alternate | plain | space)*
#   emphasized: "(" prompt ")" | "(" prompt ":" prompt ")" | "[" prompt "]"
#   scheduled: "[" [prompt ":"] prompt ":" [space] NUMBER [space] "]"      alternate: "[" prompt ("|" [prompt])+ "]"
# A prompt holds no stray bracket, colon or bar, so every group is closed by the nearest matching closer; an opener
# whose group is not one of the forms above is a stray character of the top level.  A bar outside an alternation, or a
# backslash that escapes nothing, makes the prompt unparseable: it is then used as it is for every step.
_NUMBER = re.compile(r"\s*([+-]?(?:[0-9]+(?:\.[0-9]*)?|\.[0-9]+)(?:[eE][+-]?[0-9]+)?)\s*")
_PLAIN = re.compile(r"[^\\\[\]():|]+")


class _Unparsable(Exception):
    pass


def _escape(s: str, j: int) -> str:
    if j + 1 >= len(s) or s[j + 1] == "\n":
        raise _Unparsable
    return s[j:j + 2]


def _group(s: str, i: int):
    """s[i] is "[" or "(": (nodes of the group, index after its closer), or None if s[i] opens none of the grammar's
    forms.  Nodes: text, ("edit", before nodes or None, after nodes, number text), ("alt", [nodes per option])."""
    close = "]" if s[i] == "[" else ")"
    segs: List[list] = [[]]
    seps: List[str] = []
    j = i + 1
    while j < len(s):
        c = s[j]
        if c == "\\":
            segs[-1].append(_escape(s, j))
            j += 2
        elif c in "[(":
            r = _group(s, j)
            if r is None:
                return None
            segs[-1].extend(r[0])
            j = r[1]
        elif c == close:
            break
        elif c in ")]":
            return None
        elif c in ":|":
            seps.append(c)
            segs.append([])
            j += 1
        else:
            m = _PLAIN.match(s, j)
            segs[-1].append(m.group(0))
            j = m.end()
    else:
        return None
    end = j + 1
    if not seps or (close == ")" and seps == [":"]):   # emphasis: the brackets stay text for parse_prompt_attention
        out = [s[i]]
        for k, seg in enumerate(segs):
            out += ([":"] if k else []) + seg
        return out + [close], end
    if close == ")":
        return None
    if all(c == "|" for c in seps):
        return [("alt", segs)], end
    if all(c == ":" for c in seps) and len(seps) <= 2 and all(isinstance(t, str) for t in segs[-1]):
        m = _NUMBER.fullmatch("".join(segs[-1]))
        if m:
            return [("edit", segs[0] if len(seps) == 2 else None, segs[-2], m.group(1))], end
    return None


def _parse_schedule(s: str) -> list:
    nodes: list = []
    j = 0
    while j < len(s):
        c = s[j]
        if c == "\\":
            nodes.append(_escape(s, j))
            j += 2
        elif c == "|":
            raise _Unparsable
        elif c in "[(" and (r := _group(s, j)) is not None:
            nodes.extend(r[0])
            j = r[1]
        elif c in "[]():":
            nodes.append(c)
            j += 1
        else:
            m = _PLAIN.match(s, j)
            nodes.append(m.group(0))
            j = m.end()
    return nodes


def prompt_schedule(text: str, steps: int, hires_steps: Optional[int] = None,
                    use_old_scheduling: bool = False) -> List[Tuple[int, str]]:
    """sdwui prompt_parser.get_learned_conditioning_prompt_schedules for one prompt: [(end_at_step, text)] in step
    order, the last entry ending at the run's steps.  `[from:to:when]` is `from` up to step `when` and `to` after it
    (`[to:when]`: nothing, then `to`); `[a|b|...]` takes option (step - 1) % n at every step.  `when` with a "." is a
    fraction of the steps, without one an absolute step; for the hires pass (hires_steps: its steps, `steps`: the
    first pass's) a fraction counts from 1.0 and a step from `steps`.  use_old_scheduling: `when` < 1 is a fraction,
    anything else a step, and no hires offsets."""
    try:
        nodes = _parse_schedule(text)
    except _Unparsable:
        return [(hires_steps if hires_steps is not None and not use_old_scheduling else steps, text)]
    if hires_steps is None or use_old_scheduling:
        int_offset, flt_offset = 0, 0.0
    else:
        int_offset, flt_offset, steps = steps, 1.0, hires_steps
    bounds = {steps}

    def when(num: str) -> int:
        v = float(num)
        if use_old_scheduling:
            v = v * steps if v < 1 else v
        elif "." in num:
            v = (v - flt_offset) * steps
        else:
            v = v - int_offset
        return steps if v >= steps else int(v)

    def resolve(ns):   # number text -> clamped step; collects the boundaries
        out = []
        for n in ns:
            if isinstance(n, str):
                out.append(n)
            elif n[0] == "edit":
                w = when(n[3])
                if w >= 1:
                    bounds.add(w)
                out.append(("edit", None if n[1] is None else resolve(n[1]), resolve(n[2]), w))
            else:
                bounds.update(range(1, steps + 1))
                out.append(("alt", [resolve(o) for o in n[1]]))
        return out

    def render(ns, step: int) -> str:
        parts = []
        for n in ns:
            if isinstance(n, str):
                parts.append(n)
            elif n[0] == "edit":
                if step <= n[3]:
                    parts.append("" if n[1] is None else render(n[1], step))
                else:
                    parts.append(render(n[2], step))
            else:
                parts.append(render(n[1][(step - 1) % len(n[1])], step))
        return "".join(parts)

    tree = resolve(nodes)
    return [(t, render(tree, t)) for t in sorted(bounds)]


def schedule_index(schedule: Sequence[Tuple[int, str]], step: int) -> int:
    """the entry model evaluation `step` (from 0) uses: the first whose end_at_step >= step, entry 0 if none
    (sdwui prompt_parser.reconstruct_cond_batch)"""
    for i, (end, _) in enumerate(schedule):
        if step <= end:
            return i
    return 0
