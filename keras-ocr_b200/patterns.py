"""Regular expressions over a recognizer's alphabet, compiled to the minimal DFA that ``b2o_ctc_beam_pattern_decode``
walks (DESIGN.md section 1, "Patterns").

The syntax is a strict subset of Python's ``re`` with full-match semantics, so a pattern accepts a reading exactly when
``re.fullmatch(pattern, reading)`` does:

* a literal character of the alphabet, or ``\\`` and any ASCII punctuation character (that character);
* ``.`` (every alphabet character but a newline) and ``\\d`` (the alphabet characters ``re`` matches with ``\\d``);
* classes ``[...]`` with ranges and ``^`` negation: the alphabet characters whose code point the class covers;
* groups ``( )`` and ``(?: )``, alternation ``|``;
* one quantifier per atom: ``?``, ``*``, ``+``, ``{m}``, ``{m,}``, ``{m,n}`` with m <= n <= 48.

Anything else -- anchors, backreferences, lookaround, flags, lazy or possessive quantifiers, other escapes, unbalanced
parentheses, bad ranges, a class without an alphabet character, a literal outside the alphabet -- raises ``ValueError``
naming its position.

``compile_pattern`` runs Thompson's construction, the subset construction over the labels 0 .. K-2, Moore's partition
refinement, trimming to the states that are reachable and co-reachable, and a breadth-first numbering from the start
state with labels in ascending order; every step is deterministic, so a pattern always gives the same tables.
"""
import collections
import re

import numpy as np

MAX_REPEAT = 48                # the decoder's 48 steps: no reading is longer
MAX_NFA_STATES = 1 << 17       # Thompson states, after the counted quantifiers are expanded
MAX_SUBSET_STATES = 1 << 16    # DFA states before minimisation
MAX_STATES = 4096              # B2O_MAX_PATTERN_STATES in include/b2ocr.h
_META = set(".^$*+?{}[]\\|()")


class _Parser:
    """Recursive descent over the pattern; nodes are ("set", mask, pos), ("cat", [nodes]), ("alt", [nodes]) and
    ("rep", node, m, n or None, pos), a mask being a Python int with bit c set for label c."""

    def __init__(self, text, alphabet):
        self.s, self.i, self.alphabet = text, 0, alphabet
        self.index = {ch: i for i, ch in enumerate(alphabet)}
        self.all = sum(1 << i for i, ch in enumerate(alphabet) if ch != "\n")
        self.digits = sum(1 << i for i, ch in enumerate(alphabet) if re.fullmatch(r"\d", ch))

    def error(self, msg, pos=None):
        pos = self.i if pos is None else pos
        raise ValueError(f"pattern {self.s!r}, position {pos}: {msg}")

    def peek(self):
        return self.s[self.i] if self.i < len(self.s) else None

    def parse(self):
        node = self.alternation()
        if self.i < len(self.s):
            self.error("unbalanced parenthesis ')'")
        return node

    def alternation(self):
        branches = [self.concatenation()]
        while self.peek() == "|":
            self.i += 1
            branches.append(self.concatenation())
        return branches[0] if len(branches) == 1 else ("alt", branches)

    def concatenation(self):
        items = []
        while self.peek() is not None and self.peek() not in "|)":
            items.append(self.repetition())
        return ("cat", items)

    def repetition(self):
        ch = self.peek()
        if ch in ("*", "+", "?") or (ch == "{" and self._counted() is not None):
            self.error(f"nothing to repeat before {ch!r}")
        node = self.atom()
        at = self.i
        ch = self.peek()
        if ch in ("*", "+", "?"):
            self.i += 1
            m, n = {"*": (0, None), "+": (1, None), "?": (0, 1)}[ch]
        elif ch == "{":
            q = self._counted()
            if q is None:
                self.error("'{' must start a quantifier {m}, {m,} or {m,n}")
            m, n, self.i = q
            if m > MAX_REPEAT or (n is not None and n > MAX_REPEAT):
                self.error(f"a counted repeat may not exceed {MAX_REPEAT}", at)
            if n is not None and m > n:
                self.error(f"bad repeat interval {{{m},{n}}}", at)
        else:
            return node
        nxt = self.peek()
        if nxt in ("?", "+"):
            self.error("lazy and possessive quantifiers are not supported")
        if nxt in ("*", "{") and (nxt == "*" or self._counted() is not None):
            self.error("multiple repeat")
        return ("rep", node, m, n, at)

    def _counted(self):
        """(m, n or None, end) of a {m} / {m,} / {m,n} at the cursor, or None."""
        mt = re.compile(r"\{(\d+)(,(\d*))?\}").match(self.s, self.i)
        if not mt:
            return None
        m = int(mt.group(1))
        if mt.group(2) is None:
            return m, m, mt.end()
        return m, (int(mt.group(3)) if mt.group(3) else None), mt.end()

    def atom(self):
        at, ch = self.i, self.peek()
        if ch == "(":
            self.i += 1
            if self.s.startswith("?:", self.i):
                self.i += 2
            elif self.peek() == "?":
                self.error("only the non-capturing group '(?:' is supported: no flags, lookaround or named groups")
            node = self.alternation()
            if self.peek() != ")":
                self.error("missing ')', unterminated subpattern", at)
            self.i += 1
            return node
        if ch in ("^", "$"):
            self.error("anchors are not supported: a pattern always matches the whole reading")
        if ch == ".":
            self.i += 1
            return ("set", self._nonempty(self.all, at), at)
        if ch == "[":
            return ("set", self._klass(), at)
        if ch == "\\":
            mask = self._escape(in_class=False)
            return ("set", self._nonempty(mask, at), at)
        if ch == "{":
            self.error("'{' must start a quantifier {m}, {m,} or {m,n}")
        self.i += 1
        return ("set", self._literal(ch, at), at)

    def _nonempty(self, mask, at):
        if not mask:
            self.error("matches no character of the alphabet", at)
        return mask

    def _literal(self, ch, at):
        if ch not in self.index:
            self.error(f"{ch!r} is not in the alphabet", at)
        return 1 << self.index[ch]

    def _escape(self, in_class):
        """The mask of the escape at the cursor (a backslash); a literal's mask is its code point wrapped as -cp - 1
        inside a class, so that ranges can use it."""
        at = self.i
        if self.i + 1 >= len(self.s):
            self.error("bad escape (end of pattern)")
        ch = self.s[self.i + 1]
        self.i += 2
        if ch == "d":
            return self.digits
        if ch.isascii() and not ch.isalnum() and ch.isprintable():
            return -ord(ch) - 1 if in_class else self._literal(ch, at)
        what = "backreferences are" if ch.isdigit() else f"the escape \\{ch} is"
        self.error(f"{what} not supported", at)

    def _klass(self):
        at = self.i
        self.i += 1
        negate = self.peek() == "^"
        if negate:
            self.i += 1
        points, mask, first = set(), 0, True

        def item():
            """A code point (int >= 0) or a mask (\\d: ("mask", m))."""
            c = self.peek()
            if c is None:
                self.error("unterminated character set", at)
            if c == "\\":
                v = self._escape(in_class=True)
                return -v - 1 if v < 0 else ("mask", v)
            if c == "[" and self.s.startswith(("[:", "[=", "[."), self.i):
                self.error("POSIX classes are not supported")
            self.i += 1
            return ord(c)

        while True:
            c = self.peek()
            if c is None:
                self.error("unterminated character set", at)
            if c == "]" and not first:
                self.i += 1
                break
            first = False
            pos = self.i
            lo = item()
            if self.peek() == "-" and self.i + 1 < len(self.s) and self.s[self.i + 1] != "]":
                self.i += 1
                hi = item()
                if isinstance(lo, tuple) or isinstance(hi, tuple):
                    self.error("bad character range", pos)
                if hi < lo:
                    self.error(f"bad character range {chr(lo)}-{chr(hi)}", pos)
                points.update(i for i, ch in enumerate(self.alphabet) if lo <= ord(ch) <= hi)
            elif isinstance(lo, tuple):
                mask |= lo[1]
            else:
                points.update(i for i, ch in enumerate(self.alphabet) if ord(ch) == lo)
        mask |= sum(1 << i for i in points)
        if negate:
            mask = sum(1 << i for i in range(len(self.alphabet))) & ~mask
        return self._nonempty(mask, at)


class _Nfa:
    """Thompson's construction: per state a list of epsilon targets and a list of (mask, target) edges."""

    def __init__(self, text):
        self.text, self.eps, self.edges = text, [], []

    def state(self):
        self.eps.append([])
        self.edges.append([])
        return len(self.eps) - 1

    def build(self, node):
        """(start, end) of a fragment for ``node``."""
        kind = node[0]
        if kind == "set":
            a, b = self.state(), self.state()
            self.edges[a].append((node[1], b))
            return a, b
        if kind == "cat":
            a = b = self.state()
            for item in node[1]:
                s, e = self.build(item)
                self.eps[b].append(s)
                b = e
            return a, b
        if kind == "alt":
            a, b = self.state(), self.state()
            for item in node[1]:
                s, e = self.build(item)
                self.eps[a].append(s)
                self.eps[e].append(b)
            return a, b
        _, sub, m, n, at = node
        a = b = self.state()
        for _ in range(m):
            s, e = self.build(sub)
            self.eps[b].append(s)
            b = e
            self._cap(at)
        if n is None:                                          # sub*: a loop through one more copy
            s, e = self.build(sub)
            end = self.state()
            self.eps[b] += [s, end]
            self.eps[e] += [s, end]
            b = end
        else:
            for _ in range(n - m):                             # (sub(sub(...)?)?)?
                s, e = self.build(sub)
                self.eps[b].append(s)
                end = self.state()
                self.eps[b].append(end)
                self.eps[e].append(end)
                b = end
                self._cap(at)
        self._cap(at)
        return a, b

    def _cap(self, at):
        if len(self.eps) > MAX_NFA_STATES:
            raise ValueError(f"pattern {self.text!r}, position {at}: the repeat expands past {MAX_NFA_STATES} "
                             "automaton states")


def _closure(nfa, states):
    seen, stack = set(states), list(states)
    while stack:
        for t in nfa.eps[stack.pop()]:
            if t not in seen:
                seen.add(t)
                stack.append(t)
    return frozenset(seen)


def _whole(text, msg):
    return ValueError(f"pattern {text!r}, positions 0 to {len(text)}: {msg}")


def compile_pattern(text, alphabet):
    """``text`` over ``alphabet`` -> (trans (n, K-1) int16 with -1 for no transition, dist (n,) uint8, start = 0).
    dist[q] is the fewest labels from q to an accepting state (0: q accepts), saturated at 255."""
    if not isinstance(text, str):
        raise ValueError(f"a pattern is a str, got {type(text).__name__}")
    k1 = len(alphabet)
    tree = _Parser(text, alphabet).parse()
    nfa = _Nfa(text)
    s0, accept = nfa.build(tree)

    # subset construction, states numbered in discovery order, labels ascending
    first = _closure(nfa, [s0])
    ids, sets, rows = {first: 0}, [first], []
    queue = collections.deque([first])
    while queue:
        cur = queue.popleft()
        moves = collections.defaultdict(set)
        for s in sorted(cur):
            for mask, t in nfa.edges[s]:
                while mask:
                    low = mask & -mask
                    moves[low.bit_length() - 1].add(t)
                    mask ^= low
        row = np.full(k1, -1, np.int64)
        for c in sorted(moves):
            nxt = _closure(nfa, moves[c])
            if nxt not in ids:
                if len(sets) >= MAX_SUBSET_STATES:
                    raise _whole(text, f"the subset construction exceeds {MAX_SUBSET_STATES} states")
                ids[nxt] = len(sets)
                sets.append(nxt)
                queue.append(nxt)
            row[c] = ids[nxt]
        rows.append(row)
    trans = np.stack(rows)
    final = np.array([accept in st for st in sets])

    # Moore refinement: split classes by (class, class of every successor) until nothing splits
    cls = final.astype(np.int64)
    count = len(np.unique(cls))
    while True:
        succ = np.where(trans >= 0, cls[np.maximum(trans, 0)], -1)
        _, cls = np.unique(np.concatenate([cls[:, None], succ], 1), axis=0, return_inverse=True)
        cls = cls.reshape(-1)
        if cls.max() + 1 == count:
            break
        count = int(cls.max()) + 1
    rep = np.unique(cls, return_index=True)[1]                  # the first state of every class
    trans = np.where(trans[rep] >= 0, cls[np.maximum(trans[rep], 0)], -1)
    final, start = final[rep], int(cls[0])

    # trimming: states co-reachable from an accepting state, then reachable from the start
    n = len(trans)
    dist = _dist(trans, final)
    live = dist < np.iinfo(np.int64).max
    if not live[start]:
        raise _whole(text, "the pattern accepts no reading")
    trans = np.where((trans >= 0) & live[np.maximum(trans, 0)], trans, -1)

    # canonical numbering: breadth first from the start state, labels ascending
    order, at = [start], {start: 0}
    for q in order:
        for c in range(k1):
            t = int(trans[q, c])
            if t >= 0 and t not in at:
                at[t] = len(order)
                order.append(t)
    n = len(order)
    if n > MAX_STATES:
        raise _whole(text, f"the minimal automaton has {n} states; at most {MAX_STATES} are supported")
    old = np.array(order)
    remap = np.full(len(trans), -1, np.int64)
    remap[old] = np.arange(n)
    trans = np.where(trans[old] >= 0, remap[np.maximum(trans[old], 0)], -1)
    dist = dist[old]
    if dist[0] > MAX_REPEAT:
        raise _whole(text, f"every accepted reading is longer than {MAX_REPEAT} characters (the shortest has "
                           f"{int(dist[0])})")
    return trans.astype(np.int16), np.minimum(dist, 255).astype(np.uint8), 0


def _dist(trans, final):
    """Fewest labels from every state to an accepting one (int64 max: none), by breadth-first search backwards."""
    n = len(trans)
    inf = np.iinfo(np.int64).max
    dist = np.full(n, inf, np.int64)
    preds = [[] for _ in range(n)]
    for q, c in zip(*np.nonzero(trans >= 0)):
        preds[int(trans[q, c])].append(int(q))
    queue = collections.deque(np.nonzero(final)[0].tolist())
    dist[final] = 0
    while queue:
        q = queue.popleft()
        for p in preds[q]:
            if dist[p] == inf:
                dist[p] = dist[q] + 1
                queue.append(p)
    return dist
