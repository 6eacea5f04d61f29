"""Structured outputs: decoding constrained to a fixed set of strings (``choice``) or to a regular expression (``regex``), vLLM's
``StructuredOutputsParams``.  This module is the host half: it compiles the constraint into a byte DFA, lists the bytes of every token
of the tokenizer, and keeps both on the device; the per-step work is three kernels of csrc/structured.cu.

    regex  -> Thompson NFA -> subset construction -> trim     choice -> the byte trie of the UTF-8 choices

The DFA reads UTF-8 bytes and always matches the WHOLE output.  Every state that cannot reach an accepting state is trimmed, so a
token whose bytes can be walked from a state never leads into a dead end.  Supported regex subset (Python ``re`` on bytes decides
the same strings):
  * literals, any UTF-8 text (matched as its bytes; a quantifier after a multi-byte character repeats the whole character),
  * escapes ``\\d \\w \\s \\D \\W \\S`` (ASCII: [0-9], [A-Za-z0-9_], [ \\t\\n\\r\\f\\v]; the complements include every byte >= 0x80),
    ``\\n \\t \\r \\f \\v`` and any escaped ASCII punctuation,
  * ``.`` (any byte except ``\\n``), ASCII classes ``[...]`` / ``[^...]`` with ranges and the escapes above,
  * ``* + ? {m} {m,} {,n} {m,n}`` (a trailing ``?`` -- lazy -- accepts the same strings under a full match), ``|``, ``( )``, ``(?: )``,
  * a leading ``^`` and a trailing ``$``, which a full match makes redundant.
Anything else raises ValueError naming the construct: backreferences, lookaround, named groups and inline flags, anchors inside the
pattern, non-ASCII characters inside a class, possessive quantifiers.

Size: at most MAX_STATES (4096) DFA states, and repeat counts up to MAX_REPEAT; beyond either, ValueError.  Each state costs
ceil(V / 32) words of allowed bits on the device: 19 KB at V = 152 064, 78 MB at the cap.

Token bytes: ``SimpleTokenizer`` (and no tokenizer): ids < 256 are their own byte.  A Hugging Face byte-level BPE tokenizer (or a
``tokenizers.Tokenizer``): each token string through the GPT-2 byte decoder.  Special and added tokens, tokens that are not byte-level
and embedding rows past the tokenizer have no bytes and are never allowed -- except the call's stop ids, which are allowed exactly in
accepting states and end the output there.
"""
import re
from collections import OrderedDict
from dataclasses import dataclass
from functools import lru_cache

import numpy as np
import torch

MAX_STATES = 4096
MAX_REPEAT = 1000
MAX_NFA_STATES = 200_000
MAX_STOP_IDS = 64                        # cts_struct_mask_build / cts_struct_advance take at most 64 stop ids


@dataclass
class StructuredOutputsParams:
    """vLLM's StructuredOutputsParams: at most one field set.  ``choice`` (a list of strings) and ``regex`` are supported; ``json``,
    ``grammar`` and ``json_object`` raise ValueError."""
    choice: list = None
    regex: str = None
    json: object = None
    grammar: str = None
    json_object: bool = None

    def __post_init__(self):
        named = [n for n in ("choice", "regex", "json", "grammar", "json_object") if getattr(self, n) not in (None, False)]
        if len(named) > 1:
            raise ValueError(f"structured_outputs: at most one of choice / regex / json / grammar / json_object, got {named}")
        for n in ("json", "grammar", "json_object"):
            if getattr(self, n) not in (None, False):
                raise ValueError(f"structured_outputs.{n} is not supported (choice and regex are)")
        if self.choice is not None:
            if isinstance(self.choice, str) or not isinstance(self.choice, (list, tuple)) or not self.choice \
                    or not all(isinstance(c, str) for c in self.choice):
                raise ValueError("structured_outputs.choice must be a non-empty list of strings")
            self.choice = list(self.choice)
        if self.regex is not None and not isinstance(self.regex, str):
            raise ValueError("structured_outputs.regex must be a string")

    def key(self):
        """(kind, pattern) of the constraint, None when no field is set."""
        if self.choice is not None:
            return ("choice", tuple(self.choice))
        if self.regex is not None:
            return ("regex", self.regex)
        return None


def resolve(spec):
    """StructuredOutputsParams, a dict of its fields, or None -> a validated StructuredOutputsParams, or None when nothing is set."""
    if spec is None:
        return None
    if isinstance(spec, dict):
        unknown = set(spec) - {"choice", "regex", "json", "grammar", "json_object"}
        if unknown:
            raise ValueError(f"structured_outputs: unknown fields {sorted(unknown)}")
        spec = StructuredOutputsParams(**spec)
    elif not isinstance(spec, StructuredOutputsParams):
        raise ValueError(f"structured_outputs must be StructuredOutputsParams or a dict, not {type(spec).__name__}")
    return spec if spec.key() is not None else None


# ------------------------------------------------------------------------------------------------------------------------ DFA
@dataclass
class ByteDFA:
    """trans int32 [S, 256] (-1: no transition), accept bool [S]; state 0 is the start.  Trimmed: every state reaches an accepting one."""
    trans: np.ndarray
    accept: np.ndarray

    @property
    def num_states(self):
        return self.trans.shape[0]

    def walk(self, data, state=0):
        """The state reached by reading ``data`` (bytes) from ``state``; -1 once a byte has no transition."""
        for b in data:
            if state < 0:
                break
            state = int(self.trans[state, b])
        return state

    def fullmatch(self, data):
        s = self.walk(data)
        return s >= 0 and bool(self.accept[s])


_ALL = frozenset(range(256))
_DIGIT = frozenset(range(0x30, 0x3A))
_WORD = frozenset(b"0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz_")
_SPACE = frozenset(b" \t\n\r\f\v")
_CLASS_ESCAPES = {"d": _DIGIT, "w": _WORD, "s": _SPACE, "D": _ALL - _DIGIT, "W": _ALL - _WORD, "S": _ALL - _SPACE}
_CHAR_ESCAPES = {"n": 10, "t": 9, "r": 13, "f": 12, "v": 11}
_BRACE = re.compile(r"\{(\d*)(?:(,)(\d*))?\}")


class _Parser:
    """Recursive descent over the supported subset -> AST of ("set", frozenset) / ("cat", [..]) / ("alt", [..]) / ("rep", node, m, n)."""

    def __init__(self, pattern):
        self.p, self.i = pattern, 0

    def parse(self):
        node = self.alt()
        if self.i < len(self.p):                          # only an unbalanced ')' stops the top-level alternation early
            raise ValueError(f"regex: unbalanced ')' at position {self.i}")
        return node

    def peek(self):
        return self.p[self.i] if self.i < len(self.p) else None

    def alt(self):
        branches = [self.cat()]
        while self.peek() == "|":
            self.i += 1
            branches.append(self.cat())
        return branches[0] if len(branches) == 1 else ("alt", branches)

    def cat(self):
        items = []
        while self.peek() is not None and self.peek() not in "|)":
            items.append(self.repeat())
        return ("cat", items)

    def brace(self):
        """(m, n) of a {..} quantifier at the cursor (advanced past it), or None when the brace is a literal (as in Python)."""
        m = _BRACE.match(self.p, self.i)
        if not m or (m.group(1) == "" and m.group(2) is None):
            return None
        lo = int(m.group(1) or 0)
        hi = lo if m.group(2) is None else (int(m.group(3)) if m.group(3) else None)
        if hi is not None and hi < lo:
            raise ValueError(f"regex: min repeat greater than max repeat in {m.group(0)}")
        if max(lo, hi or 0) > MAX_REPEAT:
            raise ValueError(f"regex: repeat count in {m.group(0)} exceeds {MAX_REPEAT}")
        self.i = m.end()
        return lo, hi

    def repeat(self):
        node = self.atom()
        quantified = False
        while True:
            c = self.peek()
            if c is not None and c in "*+?":
                q = {"*": (0, None), "+": (1, None), "?": (0, 1)}[c]
                self.i += 1
            elif c == "{" and _BRACE.match(self.p, self.i):
                q = self.brace()
                if q is None:
                    break
            else:
                break
            if quantified:
                raise ValueError(f"regex: repeated or possessive quantifier at position {self.i - 1}")
            node, quantified = ("rep", node, q[0], q[1]), True
            if self.peek() == "?":                        # lazy: the same strings under a full match
                self.i += 1
        return node

    def atom(self):
        p, i = self.p, self.i
        c = p[i]
        if c == "(":
            if p.startswith("(?:", i):
                self.i += 3
            elif p.startswith("(?", i):
                what = ("lookahead" if p.startswith(("(?=", "(?!"), i) else "lookbehind" if p.startswith(("(?<=", "(?<!"), i)
                        else "named group" if p.startswith(("(?P", "(?<"), i) else "inline flags / group extension")
                raise ValueError(f"regex: {what} at position {i} is not supported")
            else:
                self.i += 1
            node = self.alt()
            if self.peek() != ")":
                raise ValueError(f"regex: missing ')' for the group at position {i}")
            self.i += 1
            return node
        if c in "*+?" or (c == "{" and self.brace_is_quantifier()):
            raise ValueError(f"regex: nothing to repeat at position {i}")
        self.i += 1
        if c == "[":
            return ("set", self.char_class(i))
        if c == ".":
            return ("set", _ALL - {10})
        if c == "^":
            if i == 0:
                return ("cat", [])
            raise ValueError(f"regex: anchor '^' inside the pattern (position {i}) is not supported")
        if c == "$":
            if i == len(p) - 1:
                return ("cat", [])
            raise ValueError(f"regex: anchor '$' inside the pattern (position {i}) is not supported")
        if c == "\\":
            return ("set", self.escape(in_class=False))
        data = c.encode("utf-8")
        return ("set", frozenset(data)) if len(data) == 1 else ("cat", [("set", frozenset([b])) for b in data])

    def brace_is_quantifier(self):
        m = _BRACE.match(self.p, self.i)
        return bool(m) and not (m.group(1) == "" and m.group(2) is None)

    def escape(self, in_class):
        """Escape after the backslash (the cursor is past it) -> its byte set."""
        if self.i >= len(self.p):
            raise ValueError("regex: trailing backslash")
        e = self.p[self.i]
        self.i += 1
        if e in _CLASS_ESCAPES:
            return _CLASS_ESCAPES[e]
        if e in _CHAR_ESCAPES:
            return frozenset([_CHAR_ESCAPES[e]])
        if in_class and e == "b":
            return frozenset([8])                         # backspace inside a class, as in Python
        if e.isdigit():
            raise ValueError(f"regex: backreference or octal escape \\{e} is not supported")
        if e in "bBAZ":
            raise ValueError(f"regex: anchor \\{e} is not supported")
        if ord(e) < 128 and not e.isalnum():
            return frozenset([ord(e)])
        raise ValueError(f"regex: escape \\{e} is not supported")

    def class_item(self):
        c = self.p[self.i]
        if c == "\\":
            self.i += 1
            s = self.escape(in_class=True)
            return next(iter(s)) if len(s) == 1 else s
        if ord(c) >= 128:
            raise ValueError(f"regex: non-ASCII character {c!r} inside a character class is not supported")
        self.i += 1
        return ord(c)

    def char_class(self, start):
        p = self.p
        neg = self.peek() == "^"
        if neg:
            self.i += 1
        items, first = set(), True
        while True:
            if self.i >= len(p):
                raise ValueError(f"regex: unterminated character class at position {start}")
            if p[self.i] == "]" and not first:
                self.i += 1
                break
            first = False
            lo = self.class_item()
            if isinstance(lo, frozenset):
                items |= lo
                continue
            if self.peek() == "-" and self.i + 1 < len(p) and p[self.i + 1] != "]":
                self.i += 1
                hi = self.class_item()
                if isinstance(hi, frozenset) or hi < lo:
                    raise ValueError(f"regex: bad character range in the class at position {start}")
                items |= set(range(lo, hi + 1))
            else:
                items.add(lo)
        return frozenset(_ALL - items if neg else items)


class _NFA:
    """Thompson NFA: each state has epsilon edges and at most one byte-set edge."""

    def __init__(self):
        self.eps, self.sym, self.out = [], [], []

    def new(self):
        if len(self.eps) >= MAX_NFA_STATES:
            raise ValueError(f"regex: the automaton would exceed {MAX_NFA_STATES} NFA states")
        self.eps.append([])
        self.sym.append(None)
        self.out.append(-1)
        return len(self.eps) - 1

    def build(self, node):
        """(start, end) of the fragment of ``node``."""
        kind = node[0]
        if kind == "set":
            s, e = self.new(), self.new()
            self.sym[s], self.out[s] = tuple(sorted(node[1])), e
            return s, e
        if kind == "cat":
            s = e = self.new()
            for item in node[1]:
                a, b = self.build(item)
                self.eps[e].append(a)
                e = b
            return s, e
        if kind == "alt":
            s, e = self.new(), self.new()
            for item in node[1]:
                a, b = self.build(item)
                self.eps[s].append(a)
                self.eps[b].append(e)
            return s, e
        _, sub, m, n = node
        s = e = self.new()
        for _ in range(m):
            a, b = self.build(sub)
            self.eps[e].append(a)
            e = b
        if n is None:                                     # sub*
            a, b = self.build(sub)
            end = self.new()
            self.eps[e] += [a, end]
            self.eps[b] += [a, end]
            return s, end
        end = self.new()
        for _ in range(n - m):                            # up to n - m optional copies
            self.eps[e].append(end)
            a, b = self.build(sub)
            self.eps[e].append(a)
            e = b
        self.eps[e].append(end)
        return s, end

    def closure(self, states):
        seen, stack = set(states), list(states)
        while stack:
            for t in self.eps[stack.pop()]:
                if t not in seen:
                    seen.add(t)
                    stack.append(t)
        return frozenset(seen)


def _trim(trans, accept):
    """Drops every state that cannot reach an accepting state and renumbers the rest breadth-first from the start (state 0)."""
    S = len(trans)
    rev = [[] for _ in range(S)]
    for s in range(S):
        for t in set(trans[s]):
            if t >= 0:
                rev[t].append(s)
    live = {s for s in range(S) if accept[s]}
    stack = list(live)
    while stack:
        for u in rev[stack.pop()]:
            if u not in live:
                live.add(u)
                stack.append(u)
    if 0 not in live:
        raise ValueError("structured output: the pattern matches no string")
    order, index = [0], {0: 0}
    for s in order:
        for t in trans[s]:
            if t in live and t not in index:
                index[t] = len(order)
                order.append(t)
    out = np.full((len(order), 256), -1, dtype=np.int32)
    for new, s in enumerate(order):
        for b, t in enumerate(trans[s]):
            if t in index:
                out[new, b] = index[t]
    return ByteDFA(out, np.array([bool(accept[s]) for s in order]))


@lru_cache(maxsize=256)
def compile_regex(pattern):
    """Full-match byte DFA of ``pattern`` (the subset in the module docstring), trimmed; ValueError beyond MAX_STATES states."""
    nfa = _NFA()
    start, final = nfa.build(_Parser(pattern).parse())
    ids = {}
    sets = [nfa.closure([start])]
    ids[sets[0]] = 0
    trans, accept = [], []
    for cur in sets:                                      # `sets` grows while it is walked: breadth-first subset construction
        nxt = {}
        for s in cur:
            if nfa.sym[s] is not None:
                t = nfa.out[s]
                for b in nfa.sym[s]:
                    nxt.setdefault(b, set()).add(t)
        row = [-1] * 256
        by_targets = {}
        for b, ts in nxt.items():
            key = frozenset(ts)
            d = by_targets.get(key)
            if d is None:
                cl = nfa.closure(ts)
                d = ids.get(cl)
                if d is None:
                    if len(sets) >= MAX_STATES:
                        raise ValueError(f"structured output: the pattern needs more than {MAX_STATES} automaton states")
                    d = ids[cl] = len(sets)
                    sets.append(cl)
                by_targets[key] = d
            row[b] = d
        trans.append(row)
        accept.append(final in cur)
    return _trim(trans, accept)


@lru_cache(maxsize=256)
def compile_choice(choices):
    """Byte trie of the UTF-8 choices (a tuple of str): every node is live, so no trimming is needed."""
    trans, accept = [[-1] * 256], [False]
    for c in choices:
        s = 0
        for b in c.encode("utf-8"):
            if trans[s][b] < 0:
                if len(trans) >= MAX_STATES:
                    raise ValueError(f"structured output: the choices need more than {MAX_STATES} automaton states")
                trans[s][b] = len(trans)
                trans.append([-1] * 256)
                accept.append(False)
            s = trans[s][b]
        accept[s] = True
    return ByteDFA(np.array(trans, dtype=np.int32), np.array(accept))


def compile_params(params):
    kind, pattern = params.key()
    return compile_choice(pattern) if kind == "choice" else compile_regex(pattern)


# ------------------------------------------------------------------------------------------------------------------- token bytes
@lru_cache(maxsize=1)
def _gpt2_byte_decoder():
    """The inverse of GPT-2's bytes_to_unicode: printable bytes map to themselves, the others to U+0100 upwards in byte order."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs, n = bs[:], 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return {chr(c): b for b, c in zip(bs, cs)}


def token_bytes(tokenizer, vocab):
    """CSR of the bytes of every token id < vocab: (offsets int64 [vocab + 1], data uint8).  Ids without bytes get an empty range."""
    from .processor import SimpleTokenizer
    pieces = [b""] * vocab
    if tokenizer is None or isinstance(tokenizer, SimpleTokenizer):
        for t in range(min(256, vocab)):
            pieces[t] = bytes([t])
    else:
        dec = _gpt2_byte_decoder()
        if hasattr(tokenizer, "convert_ids_to_tokens"):                        # transformers tokenizer
            n = min(len(tokenizer), vocab)
            strs = tokenizer.convert_ids_to_tokens(list(range(n)))
            special = set(getattr(tokenizer, "all_special_ids", []) or [])
            special |= set((getattr(tokenizer, "added_tokens_decoder", None) or {}).keys())
        elif hasattr(tokenizer, "id_to_token"):                                # tokenizers.Tokenizer
            n = min(tokenizer.get_vocab_size(with_added_tokens=True), vocab)
            strs = [tokenizer.id_to_token(t) for t in range(n)]
            special = set(tokenizer.get_added_tokens_decoder().keys()) if hasattr(tokenizer, "get_added_tokens_decoder") else set()
        else:
            raise ValueError(f"structured outputs: cannot read the token bytes of a {type(tokenizer).__name__}")
        for t, s in enumerate(strs):
            if t in special or not s:
                continue
            try:
                pieces[t] = bytes(dec[ch] for ch in s)
            except KeyError:                                                   # not a byte-level token: never allowed
                pass
    lens = np.fromiter((len(p) for p in pieces), dtype=np.int64, count=vocab)
    offsets = np.zeros(vocab + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    data = np.frombuffer(b"".join(pieces) or b"\0", dtype=np.uint8).copy()
    return offsets, data


# ------------------------------------------------------------------------------------------------------------ device automata
class DeviceAutomaton:
    """One compiled constraint on the device: trans int32 [S, 256], accept uint8 [S], allowed bits int32 [S, ceil(V / 32)] and the
    stop ids, with the token bytes it was built from (offsets, data)."""

    def __init__(self, ctx, dfa, offsets, data, stops, vocab, device):
        self.dfa, self.offsets, self.data, self.stops = dfa, offsets, data, stops
        self.trans = torch.from_numpy(dfa.trans).to(device)
        self.accept = torch.from_numpy(dfa.accept.astype(np.uint8)).to(device)
        self.allowed = torch.empty(dfa.num_states, (vocab + 31) // 32, dtype=torch.int32, device=device)
        ctx.struct_mask_build(self.trans, self.accept, offsets, data, stops, self.allowed)

    def mask_apply(self, ctx, logits, batch, state):
        ctx.struct_mask_apply(logits, batch, state, self.allowed)

    def advance(self, ctx, cur_ids, batch, state):
        ctx.struct_advance(cur_ids, batch, state, self.trans, self.offsets, self.data, self.stops)


class AutomatonCache:
    """Compiled automata per (kind, pattern, tokenizer, vocab, stop ids), least recently used first out; token bytes per tokenizer."""

    def __init__(self, ctx, device, capacity=16):
        self.ctx, self.device, self.capacity = ctx, device, capacity
        self.tables, self.automata = {}, OrderedDict()

    def _tok_key(self, tokenizer):
        from .processor import SimpleTokenizer
        return "bytes" if tokenizer is None or isinstance(tokenizer, SimpleTokenizer) else id(tokenizer)

    def get(self, params, tokenizer, vocab, stop_ids):
        stops = sorted({int(t) for t in stop_ids if 0 <= int(t) < vocab})
        if len(stops) > MAX_STOP_IDS:
            raise ValueError(f"structured outputs take at most {MAX_STOP_IDS} stop ids, got {len(stops)}")
        tk = self._tok_key(tokenizer)
        key = (params.key(), tk, vocab, tuple(stops))
        hit = self.automata.get(key)
        if hit is not None:
            self.automata.move_to_end(key)
            return hit
        dfa = compile_params(params)
        tab = self.tables.get((tk, vocab))
        if tab is None:
            off, data = token_bytes(tokenizer, vocab)
            # the tokenizer is held with its table, so its id cannot be reused by another object while the entry lives
            tab = self.tables[(tk, vocab)] = (torch.from_numpy(off).to(self.device), torch.from_numpy(data).to(self.device), tokenizer)
        st = torch.tensor(stops, dtype=torch.int32, device=self.device)
        auto = DeviceAutomaton(self.ctx, dfa, tab[0], tab[1], st, vocab, self.device)
        self.automata[key] = auto
        while len(self.automata) > self.capacity:
            self.automata.popitem(last=False)
        return auto
